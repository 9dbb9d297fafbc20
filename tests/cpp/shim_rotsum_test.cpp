// tests/cpp/shim_rotsum_test.cpp -- seal_b200::Evaluator::apply_galois_add_inplace and rotate_sum_inplace on CiphertextBatch
// (include/seal_b200/evaluator.hpp) against the reference's chains on the same seal::Ciphertexts (oracle/ref_rotsum.cpp): words
// and metadata (parms_id, NTT form, scale bits, correction factor, size) of every member, and exception types and messages in the
// chain's order.  Covers CKKS, BFV and BGV, both key types, a destination that is the input, BGV correction factors that differ
// (the chain path), the NAF fallback, a key cache limit below the chain's keys, and the full slot sum of a BFV batch.
// Built by oracle/rotsum.mk into oracle/_ref/bin/shim_rotsum_test; run by tests/test_gpu_rotate_sum.py.
#include "seal/seal.h"
#include "seal_b200/evaluator.hpp"
#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <random>
#include <string>
#include <typeinfo>
#include <vector>

using namespace seal;

void ref_apply_galois_add(const seal::Evaluator &ev, Ciphertext &destination, const Ciphertext &encrypted, uint32_t galois_elt,
                          const GaloisKeys &galois_keys);
void ref_rotate_sum(const seal::Evaluator &ev, bool ckks, Ciphertext &encrypted, int step, size_t count, const GaloisKeys &galois_keys);

static int g_checks = 0, g_fail = 0;

static void fail(const std::string &what)
{
    g_fail++;
    std::printf("FAIL %s\n", what.c_str());
}

static std::string caught(const std::function<void()> &f, std::string *msg)
{
    try
    {
        f();
    }
    catch (const std::exception &e)
    {
        *msg = e.what();
        return typeid(e).name();
    }
    return "none";
}

static void same_throw(const std::function<void()> &ours, const std::function<void()> &theirs, const std::string &what)
{
    std::string m1, m2;
    const std::string t1 = caught(ours, &m1), t2 = caught(theirs, &m2);
    g_checks++;
    if (t1 != t2 || m1 != m2 || t1 == "none")
        fail(what + ": ours " + t1 + " '" + m1 + "', reference " + t2 + " '" + m2 + "'");
}

static bool same_ct(const Ciphertext &a, const Ciphertext &b)
{
    const double s1 = a.scale(), s2 = b.scale();
    return a.parms_id() == b.parms_id() && a.size() == b.size() && a.is_ntt_form() == b.is_ntt_form() &&
           a.correction_factor() == b.correction_factor() && std::memcmp(&s1, &s2, sizeof(double)) == 0 &&
           a.dyn_array().size() == b.dyn_array().size() && std::memcmp(a.data(), b.data(), a.dyn_array().size() * sizeof(uint64_t)) == 0;
}

struct Setup
{
    SEALContext context;
    KeyGenerator keygen;
    PublicKey pk;
    GaloisKeys gk;
    Encryptor enc;
    seal::Evaluator rev;
    seal_b200::Evaluator ev;
    seal_b200::DeviceGaloisKeys dgk;
    explicit Setup(const EncryptionParameters &parms)
        : context(parms, true, sec_level_type::none), keygen(context), pk(make_pk(keygen)), gk(make_gk(keygen)), enc(context, pk), rev(context),
          ev(context)
    {
        ev.upload(gk, dgk);
    }
    static PublicKey make_pk(KeyGenerator &k)
    {
        PublicKey p;
        k.create_public_key(p);
        return p;
    }
    static GaloisKeys make_gk(KeyGenerator &k)
    {
        GaloisKeys g;
        k.create_galois_keys(g); // every power-of-two step, both directions, and the column swap
        return g;
    }
    bool ckks() const { return context.first_context_data()->parms().scheme() == scheme_type::ckks; }
    // B encryptions of random slots at the top level
    std::vector<Ciphertext> encrypt(size_t B, std::mt19937_64 &rng)
    {
        std::vector<Ciphertext> out(B);
        const size_t n = context.first_context_data()->parms().poly_modulus_degree();
        for (auto &c : out)
        {
            Plaintext p;
            if (ckks())
            {
                CKKSEncoder e(context);
                std::vector<double> v(e.slot_count());
                for (auto &x : v)
                    x = static_cast<double>(rng() % 2000) / 1000.0 - 1.0;
                e.encode(v, std::pow(2.0, 30), p);
            }
            else
            {
                BatchEncoder e(context);
                const uint64_t t = context.first_context_data()->parms().plain_modulus().value();
                std::vector<uint64_t> v(n);
                for (auto &x : v)
                    x = rng() % t;
                e.encode(v, p);
            }
            enc.encrypt(p, c);
        }
        return out;
    }
};

static void compare(Setup &s, const seal_b200::CiphertextBatch &got, const std::vector<Ciphertext> &want, const std::string &what)
{
    std::vector<Ciphertext> h;
    s.ev.download(got, h);
    g_checks++;
    if (h.size() != want.size())
        return fail(what + ": batch size");
    for (size_t b = 0; b < want.size(); b++)
    {
        g_checks++;
        if (!same_ct(h[b], want[b]))
            fail(what + ": member " + std::to_string(b) + " differs");
    }
}

// apply_galois_add_inplace(destination, encrypted) with both key types, and with destination = encrypted, against the chain
template <class Keys>
static void check_add(Setup &s, const std::vector<Ciphertext> &dst, const std::vector<Ciphertext> &src, uint32_t elt, const Keys &keys,
                      const std::string &what)
{
    seal_b200::CiphertextBatch d, e;
    s.ev.upload(dst, d);
    s.ev.upload(src, e);
    s.ev.apply_galois_add_inplace(d, e, elt, keys);
    std::vector<Ciphertext> want = dst;
    for (size_t b = 0; b < want.size(); b++)
        ref_apply_galois_add(s.rev, want[b], src[b], elt, s.gk);
    compare(s, d, want, what);
    compare(s, e, src, what + " (input unchanged)");
    s.ev.apply_galois_add_inplace(e, e, elt, keys);
    std::vector<Ciphertext> self = src;
    for (auto &c : self)
    {
        const Ciphertext x = c;
        ref_apply_galois_add(s.rev, c, x, elt, s.gk);
    }
    compare(s, e, self, what + " (destination = encrypted)");
}

template <class Keys>
static void check_sum(Setup &s, const std::vector<Ciphertext> &x, int step, size_t count, const Keys &keys, const GaloisKeys &ref_keys,
                      const std::string &what)
{
    seal_b200::CiphertextBatch y;
    s.ev.upload(x, y);
    s.ev.rotate_sum_inplace(y, step, count, keys);
    std::vector<Ciphertext> want = x;
    for (auto &c : want)
        ref_rotate_sum(s.rev, s.ckks(), c, step, count, ref_keys);
    compare(s, y, want, what);
}

// the first failing call of the chain decides the exception, for ours and for the reference (member 0); ours writes nothing
static void check_sum_throw(Setup &s, const std::vector<Ciphertext> &x, int step, size_t count, const GaloisKeys &keys, const std::string &what)
{
    seal_b200::CiphertextBatch y;
    s.ev.upload(x, y);
    Ciphertext r = x[0];
    same_throw([&] { s.ev.rotate_sum_inplace(y, step, count, keys); }, [&] { ref_rotate_sum(s.rev, s.ckks(), r, step, count, keys); }, what);
    compare(s, y, x, what + " (batch unchanged)");
}

static void check_add_throw(Setup &s, const std::vector<Ciphertext> &dst, const std::vector<Ciphertext> &src, uint32_t elt,
                            const GaloisKeys &keys, const std::string &what)
{
    seal_b200::CiphertextBatch d, e;
    s.ev.upload(dst, d);
    s.ev.upload(src, e);
    Ciphertext r = dst[0];
    same_throw([&] { s.ev.apply_galois_add_inplace(d, e, elt, keys); }, [&] { ref_apply_galois_add(s.rev, r, src[0], elt, keys); }, what);
    compare(s, d, dst, what + " (destination unchanged)");
}

static EncryptionParameters parms_of(scheme_type scheme, size_t n, uint64_t t)
{
    EncryptionParameters p(scheme);
    p.set_poly_modulus_degree(n);
    p.set_coeff_modulus(CoeffModulus::Create(n, { 40, 30, 30, 40 }));
    if (scheme != scheme_type::ckks)
        p.set_plain_modulus(t);
    return p;
}

static void scheme_checks(scheme_type scheme, const std::string &name)
{
    const size_t n = 4096;
    Setup s(parms_of(scheme, n, PlainModulus::Batching(n, 20).value()));
    std::mt19937_64 rng(0x5EA1 + static_cast<int>(scheme));
    const std::vector<Ciphertext> x = s.encrypt(3, rng), y = s.encrypt(3, rng);
    const auto elt = [&](int step) { return s.context.first_context_data()->galois_tool()->get_elt_from_step(step); };
    for (int step : { 1, -1, 8 })
    {
        check_add(s, y, x, elt(step), s.gk, name + " apply_galois_add step " + std::to_string(step) + " (GaloisKeys)");
        check_add(s, y, x, elt(step), s.dgk, name + " apply_galois_add step " + std::to_string(step) + " (DeviceGaloisKeys)");
    }
    check_add(s, y, x, static_cast<uint32_t>(2 * n - 1), s.dgk, name + " apply_galois_add element 2n - 1");
    // a lower level
    std::vector<Ciphertext> xl = x, yl = y;
    for (auto &c : xl)
        s.rev.mod_switch_to_next_inplace(c);
    for (auto &c : yl)
        s.rev.mod_switch_to_next_inplace(c);
    check_add(s, yl, xl, elt(1), s.gk, name + " apply_galois_add below the top level");
    for (size_t count : { size_t(1), size_t(2), size_t(8) })
    {
        check_sum(s, x, 1, count, s.gk, s.gk, name + " rotate_sum step 1 count " + std::to_string(count) + " (GaloisKeys)");
        check_sum(s, x, -2, count, s.dgk, s.gk, name + " rotate_sum step -2 count " + std::to_string(count) + " (DeviceGaloisKeys)");
    }
    check_sum(s, xl, 4, 4, s.dgk, s.gk, name + " rotate_sum below the top level");
    // the NAF fallback: keys for 1, -1, 2, -2, 4, 8 only; steps 3 = 4 - 1 and 6 = 8 - 2 have no key of their own
    GaloisKeys naf;
    s.keygen.create_galois_keys(std::vector<int>{ 1, -1, 2, -2, 4, 8 }, naf);
    check_sum(s, x, 3, 2, naf, naf, name + " rotate_sum NAF fallback");
    check_sum(s, x, 1, 8, naf, naf, name + " rotate_sum with a partial key set");
    // a key cache below the chain's keys: every key of the call stays cached while it runs
    s.ev.set_key_cache_limit(1);
    check_sum(s, x, 1, 16, s.gk, s.gk, name + " rotate_sum with a key cache of one byte");
    check_add(s, y, x, elt(2), s.gk, name + " apply_galois_add with a key cache of one byte");
    s.ev.set_key_cache_limit(std::size_t(24) << 30);
    // errors, in the chain's order
    GaloisKeys one;
    s.keygen.create_galois_keys(std::vector<int>{ 1 }, one);
    check_sum_throw(s, x, 1, 4, one, name + " rotate_sum missing key");
    check_sum_throw(s, x, static_cast<int>(n / 4 + 1), 4, s.gk, name + " rotate_sum step count too large");
    check_add_throw(s, y, x, elt(3), one, name + " apply_galois_add missing key");
    check_add_throw(s, yl, x, elt(1), s.gk, name + " apply_galois_add level mismatch");
    {
        seal_b200::CiphertextBatch b;
        s.ev.upload(x, b);
        std::string m;
        g_checks++;
        if (caught([&] { s.ev.rotate_sum_inplace(b, 0, 4, s.gk); }, &m) != typeid(std::invalid_argument).name())
            fail(name + " rotate_sum step 0");
        g_checks++;
        if (caught([&] { s.ev.rotate_sum_inplace(b, 1, 3, s.gk); }, &m) != typeid(std::invalid_argument).name())
            fail(name + " rotate_sum count 3");
        compare(s, b, x, name + " rotate_sum argument errors (batch unchanged)");
    }
    if (scheme == scheme_type::ckks)
    {
        std::vector<Ciphertext> sc = y;
        for (auto &c : sc)
            c.scale() *= 2;
        check_add_throw(s, sc, x, elt(1), s.gk, name + " apply_galois_add scale mismatch");
    }
    if (scheme == scheme_type::bgv)
    {
        // correction factors that differ: a fresh encryption at the next level against mod-switched ones (the chain path)
        std::vector<Ciphertext> fresh(3);
        for (auto &c : fresh)
            s.enc.encrypt_zero(s.context.first_context_data()->next_context_data()->parms_id(), c);
        check_add(s, fresh, xl, elt(1), s.gk, name + " apply_galois_add with differing correction factors");
    }
    if (scheme == scheme_type::bfv)
    {
        // every slot: each row summed, then the other row added by the column swap
        seal_b200::CiphertextBatch b;
        s.ev.upload(x, b);
        s.ev.rotate_sum_inplace(b, 1, n / 2, s.gk);
        s.ev.apply_galois_add_inplace(b, b, static_cast<uint32_t>(2 * n - 1), s.gk);
        std::vector<Ciphertext> want = x;
        for (auto &c : want)
        {
            ref_rotate_sum(s.rev, s.ckks(), c, 1, n / 2, s.gk);
            const Ciphertext t = c;
            ref_apply_galois_add(s.rev, c, t, static_cast<uint32_t>(2 * n - 1), s.gk);
        }
        compare(s, b, want, name + " slot sum of every slot");
        // batching unsupported: a plain modulus that is not 1 mod 2n
        Setup nb(parms_of(scheme, n, 1024));
        std::vector<Ciphertext> z(1);
        nb.enc.encrypt_zero(z[0]);
        check_sum_throw(nb, z, 1, 2, nb.gk, name + " rotate_sum without batching");
    }
}

int main()
{
    scheme_checks(scheme_type::ckks, "CKKS");
    scheme_checks(scheme_type::bfv, "BFV");
    scheme_checks(scheme_type::bgv, "BGV");
    std::printf("%d checks, %d failures\n", g_checks, g_fail);
    if (g_fail)
        return 1;
    std::printf("shim_rotsum_test ok\n");
    return 0;
}
