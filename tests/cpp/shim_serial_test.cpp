// tests/cpp/shim_serial_test.cpp -- the Serializable overloads of seal_b200::KeyGenerator and seal_b200::Encryptor
// (include/seal_b200/{keygenerator,encryptor,serializable}.hpp) against those of seal::KeyGenerator / seal::Encryptor when the
// parameters carry a seeded Blake2xbPRNGFactory or Shake256PRNGFactory: save with compr_mode_type::none and zlib, into a stream and
// into a buffer, and save_size in both modes must equal the reference's byte for byte; the reference must load the result; the error
// cases must raise the same exception type and text.  Built by oracle/serial.mk into oracle/_ref/bin/shim_serial_test (it links the
// reference library); run by tests/test_gpu_serializable.py.
#include "seal/seal.h"
#include "seal_b200/encryptor.hpp"
#include "seal_b200/keygenerator.hpp"
#include <cstdio>
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

template <class S>
static std::string saved(const S &obj, compr_mode_type mode)
{
    std::stringstream ss;
    obj.save(ss, mode);
    return ss.str();
}
template <class S>
static std::string saved_buffer(const S &obj, compr_mode_type mode)
{
    std::vector<seal_byte> buf(static_cast<size_t>(obj.save_size(mode)));
    const auto len = obj.save(buf.data(), buf.size(), mode);
    return std::string(reinterpret_cast<const char *>(buf.data()), static_cast<size_t>(len));
}

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

// the two objects save to the same bytes in every mode and through both save overloads, report the same save_size, and the
// reference loads the device's stream into a T that saves to the reference's unseeded bytes
template <class T, class R, class G>
static void same(const SEALContext &context, const R &ref, const G &dev, const char *what)
{
    bool ok = true;
    for (const compr_mode_type mode : { compr_mode_type::none, compr_mode_type::zlib })
    {
        ok &= ref.save_size(mode) == dev.save_size(mode);
        ok &= saved(ref, mode) == saved(dev, mode);
        ok &= saved_buffer(ref, mode) == saved_buffer(dev, mode);
    }
    T a, b;
    std::stringstream ra(saved(ref, compr_mode_type::none)), db(saved(dev, compr_mode_type::zlib));
    a.load(context, ra);
    b.load(context, db);
    ok &= saved(a, compr_mode_type::none) == saved(b, compr_mode_type::none);
    if (!ok)
        std::printf("mismatch: %s\n", what);
    CHECK(ok);
}

static void compare(scheme_type scheme, size_t n, const std::vector<int> &bits, uint64_t t, bool shake)
{
    EncryptionParameters parms(scheme);
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::Create(n, bits));
    if (scheme != scheme_type::ckks)
        parms.set_plain_modulus(t);
    prng_seed_type seed{};
    seed[0] = 0x73657269616C;
    if (shake)
        parms.set_random_generator(std::make_shared<Shake256PRNGFactory>(seed));
    else
        parms.set_random_generator(std::make_shared<Blake2xbPRNGFactory>(seed));
    SEALContext context(parms, true, sec_level_type::none);
    seal::KeyGenerator sampler(context);
    const SecretKey &sk = sampler.secret_key();
    seal::KeyGenerator rgen(context, sk);
    seal_b200::Evaluator ev(context);
    seal_b200::KeyGenerator ggen(context, sk, ev);

    same<PublicKey>(context, rgen.create_public_key(), ggen.create_public_key(), "create_public_key");
    same<RelinKeys>(context, rgen.create_relin_keys(), ggen.create_relin_keys(), "create_relin_keys");
    const std::vector<uint32_t> elts = { 2 * static_cast<uint32_t>(n) - 1, 3, 5, 3 }; // unordered, one duplicate
    same<GaloisKeys>(context, rgen.create_galois_keys(elts), ggen.create_galois_keys(elts), "create_galois_keys(elts)");
    same<GaloisKeys>(context, rgen.create_galois_keys(std::vector<uint32_t>{}), ggen.create_galois_keys(std::vector<uint32_t>{}),
                     "create_galois_keys({})");
    if (n <= 4096)
        same<GaloisKeys>(context, rgen.create_galois_keys(), ggen.create_galois_keys(), "create_galois_keys()");
    if (scheme != scheme_type::ckks)
        same<GaloisKeys>(context, rgen.create_galois_keys(std::vector<int>{ 1, -2 }), ggen.create_galois_keys(std::vector<int>{ 1, -2 }),
                         "create_galois_keys(steps)");
    CHECK(outcome([&] { (void)rgen.create_galois_keys(std::vector<uint32_t>{ 3, 2 }); }) ==
          outcome([&] { (void)ggen.create_galois_keys(std::vector<uint32_t>{ 3, 2 }); }));
    CHECK(outcome([&] { (void)rgen.create_galois_keys(std::vector<uint32_t>{ 0 }); }) ==
          outcome([&] { (void)ggen.create_galois_keys(std::vector<uint32_t>{ 0 }); }));

    PublicKey pk;
    rgen.create_public_key(pk);
    seal::Encryptor renc(context, pk, sk);
    seal_b200::Encryptor genc(context, pk, sk, ev);
    Plaintext plain;
    if (scheme == scheme_type::ckks)
    {
        CKKSEncoder enc(context);
        std::vector<double> v(n / 2);
        for (size_t i = 0; i < v.size(); i++)
            v[i] = 0.001 * static_cast<double>(i % 997) - 0.4;
        enc.encode(v, std::pow(2.0, 30), plain);
    }
    else
    {
        BatchEncoder enc(context);
        std::vector<uint64_t> v(n);
        for (size_t i = 0; i < n; i++)
            v[i] = (i * 7919 + 13) % t;
        enc.encode(v, plain);
    }
    same<Ciphertext>(context, renc.encrypt_symmetric(plain), genc.encrypt_symmetric(plain), "encrypt_symmetric");
    same<Ciphertext>(context, renc.encrypt_zero_symmetric(), genc.encrypt_zero_symmetric(), "encrypt_zero_symmetric()");
    const parms_id_type next = context.first_context_data()->next_context_data() ? context.first_context_data()->next_context_data()->parms_id()
                                                                                  : context.first_parms_id();
    same<Ciphertext>(context, renc.encrypt_zero_symmetric(next), genc.encrypt_zero_symmetric(next), "encrypt_zero_symmetric(next)");
    same<Ciphertext>(context, renc.encrypt(plain), genc.encrypt(plain), "encrypt");
    same<Ciphertext>(context, renc.encrypt_zero(), genc.encrypt_zero(), "encrypt_zero()");
    same<Ciphertext>(context, renc.encrypt_zero(next), genc.encrypt_zero(next), "encrypt_zero(next)");
    Plaintext wrong = plain;
    wrong.parms_id() = parms_id_zero;
    CHECK(outcome([&] { (void)renc.encrypt_symmetric(wrong); }) == outcome([&] { (void)genc.encrypt_symmetric(wrong); }));
    CHECK(outcome([&] { (void)renc.encrypt_zero_symmetric(parms_id_zero); }) ==
          outcome([&] { (void)genc.encrypt_zero_symmetric(parms_id_zero); }));
}

int main()
{
    for (const bool shake : { false, true })
    {
        compare(scheme_type::ckks, 4096, { 40, 30, 30, 40 }, 0, shake);
        compare(scheme_type::bfv, 4096, { 36, 36, 37 }, PlainModulus::Batching(4096, 20).value(), shake);
        compare(scheme_type::bgv, 8192, { 50, 50, 50, 60 }, PlainModulus::Batching(8192, 20).value(), shake);
    }
    std::printf("%d checks, %d failed\n", g_checks, g_fail);
    if (g_fail)
        return 1;
    std::printf("PASS\n");
    return 0;
}
