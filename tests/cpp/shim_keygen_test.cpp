// tests/cpp/shim_keygen_test.cpp -- seal_b200::KeyGenerator (include/seal_b200/keygenerator.hpp) against
// seal::KeyGenerator(context, secret_key) when the parameters carry a seeded Blake2xbPRNGFactory or Shake256PRNGFactory: every
// key of every create_* overload with a destination object must equal the reference's word for word, metadata included, and save
// to the same bytes; the error cases must raise the same exception type and text.  Built by oracle/keygen.mk into
// oracle/_ref/bin/shim_keygen_test (it links the reference library); run by tests/test_gpu_keygen.py.
#include "seal/seal.h"
#include "seal_b200/keygenerator.hpp"
#include <cstdio>
#include <cstring>
#include <functional>
#include <sstream>
#include <string>
#include <vector>

using namespace seal;

static int g_checks = 0, g_fail = 0;
#define CHECK(cond)                                                        \
    do                                                                     \
    {                                                                      \
        g_checks++;                                                        \
        if (!(cond))                                                       \
        {                                                                  \
            g_fail++;                                                      \
            std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond);    \
        }                                                                  \
    } while (0)

template <class T>
static std::string saved(const T &obj)
{
    std::stringstream ss;
    obj.save(ss, compr_mode_type::none);
    return ss.str();
}

// "ok" or the exception's type and text
static std::string outcome(const std::function<void()> &f)
{
    try
    {
        f();
        return "ok";
    }
    catch (const std::invalid_argument &e)
    {
        return std::string("invalid_argument: ") + e.what();
    }
    catch (const std::logic_error &e)
    {
        return std::string("logic_error: ") + e.what();
    }
    catch (const std::exception &e)
    {
        return std::string("exception: ") + e.what();
    }
}

static bool same_words(const Ciphertext &x, const Ciphertext &y)
{
    return x.dyn_array().size() == y.dyn_array().size() &&
           std::memcmp(x.data(), y.data(), x.dyn_array().size() * sizeof(uint64_t)) == 0;
}

static bool same_kswitch(const KSwitchKeys &a, const KSwitchKeys &b)
{
    if (a.parms_id() != b.parms_id() || a.data().size() != b.data().size())
        return false;
    for (size_t i = 0; i < a.data().size(); i++)
    {
        if (a.data()[i].size() != b.data()[i].size())
            return false;
        for (size_t j = 0; j < a.data()[i].size(); j++)
        {
            const Ciphertext &x = a.data()[i][j].data(), &y = b.data()[i][j].data();
            if (x.parms_id() != y.parms_id() || x.size() != y.size() || x.is_ntt_form() != y.is_ntt_form() ||
                x.scale() != y.scale() || x.correction_factor() != y.correction_factor() || !same_words(x, y))
                return false;
        }
    }
    return saved(a) == saved(b);
}

static void compare(scheme_type scheme, size_t n, const std::vector<int> &bits, uint64_t t, bool shake)
{
    EncryptionParameters parms(scheme);
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::Create(n, bits));
    if (scheme != scheme_type::ckks)
        parms.set_plain_modulus(t);
    prng_seed_type seed{};
    seed[0] = 0x6B657967656E;
    if (shake)
        parms.set_random_generator(std::make_shared<Shake256PRNGFactory>(seed));
    else
        parms.set_random_generator(std::make_shared<Blake2xbPRNGFactory>(seed));
    SEALContext context(parms, true, sec_level_type::none);
    seal::KeyGenerator sampler(context); // the secret key comes from the reference
    const SecretKey &sk = sampler.secret_key();
    seal::KeyGenerator rgen(context, sk);
    seal_b200::Evaluator ev(context);
    seal_b200::KeyGenerator ggen(context, sk, ev);
    CHECK(ggen.secret_key().data() == sk.data());

    PublicKey rpk, gpk;
    rgen.create_public_key(rpk);
    ggen.create_public_key(gpk);
    CHECK(rpk.parms_id() == gpk.parms_id() && same_words(rpk.data(), gpk.data()) && saved(rpk) == saved(gpk));

    const bool ks = context.using_keyswitching();
    RelinKeys rrk, grk;
    const std::string rr = outcome([&] { rgen.create_relin_keys(rrk); }), gr = outcome([&] { ggen.create_relin_keys(grk); });
    CHECK(rr == gr);
    if (ks)
        CHECK(rr == "ok" && same_kswitch(rrk, grk));

    const uint32_t m = static_cast<uint32_t>(2 * n);
    auto galois = [&](const std::function<void(seal::KeyGenerator &, GaloisKeys &)> &r,
                      const std::function<void(seal_b200::KeyGenerator &, GaloisKeys &)> &g) {
        GaloisKeys rk, gk;
        const std::string ro = outcome([&] { r(rgen, rk); }), go = outcome([&] { g(ggen, gk); });
        if (ro != go)
            std::printf("  reference: %s\n  device:    %s\n", ro.c_str(), go.c_str());
        CHECK(ro == go);
        if (ro == "ok")
            CHECK(same_kswitch(rk, gk));
        return ro;
    };
    // elements: a positive step, a negative step, the column / conjugate element, duplicates in the list
    const std::vector<uint32_t> elts{ 3, m - 1, 3, 5, m - 1, 3 };
    galois([&](seal::KeyGenerator &k, GaloisKeys &d) { k.create_galois_keys(elts, d); },
           [&](seal_b200::KeyGenerator &k, GaloisKeys &d) { k.create_galois_keys(elts, d); });
    // steps (needs batching), the default set
    const std::vector<int> steps{ 1, -2, 1 };
    galois([&](seal::KeyGenerator &k, GaloisKeys &d) { k.create_galois_keys(steps, d); },
           [&](seal_b200::KeyGenerator &k, GaloisKeys &d) { k.create_galois_keys(steps, d); });
    const std::string all = galois([&](seal::KeyGenerator &k, GaloisKeys &d) { k.create_galois_keys(d); },
                                   [&](seal_b200::KeyGenerator &k, GaloisKeys &d) { k.create_galois_keys(d); });
    CHECK((all == "ok") == ks);
    // invalid elements: even, too large, after a valid one
    for (const std::vector<uint32_t> bad : { std::vector<uint32_t>{ 4 }, std::vector<uint32_t>{ m + 1 }, std::vector<uint32_t>{ 3, m } })
    {
        const std::string o = galois([&](seal::KeyGenerator &k, GaloisKeys &d) { k.create_galois_keys(bad, d); },
                                     [&](seal_b200::KeyGenerator &k, GaloisKeys &d) { k.create_galois_keys(bad, d); });
        CHECK(o == "invalid_argument: Galois element is not valid" || (!ks && bad.size() == 2));
    }
}

int main()
{
    try
    {
        for (bool shake : { false, true })
        {
            compare(scheme_type::ckks, 4096, { 40, 30, 30, 40 }, 0, shake);
            compare(scheme_type::bfv, 4096, { 36, 36, 37 }, PlainModulus::Batching(4096, 20).value(), shake);
            compare(scheme_type::bgv, 2048, { 30, 30, 30 }, PlainModulus::Batching(2048, 17).value(), shake);
            compare(scheme_type::bfv, 8192, { 60, 60, 60, 60, 60 }, PlainModulus::Batching(8192, 20).value(), shake);
        }
        // no batching (plain modulus not 1 mod 2n): the step overload raises "encryption parameters do not support batching"
        compare(scheme_type::bfv, 2048, { 30, 30, 30 }, 1024, false);
        // one prime: no key switching, every key-switching key raises the reference's logic_error
        compare(scheme_type::bgv, 2048, { 40 }, PlainModulus::Batching(2048, 17).value(), true);
        compare(scheme_type::ckks, 1024, { 40 }, 0, false);
    }
    catch (const std::exception &e)
    {
        std::printf("FAIL: unexpected exception: %s\n", e.what());
        return 2;
    }
    std::printf("%s: %d checks, %d failed\n", g_fail ? "FAIL" : "PASS", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
