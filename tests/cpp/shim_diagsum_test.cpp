// tests/cpp/shim_diagsum_test.cpp -- seal_b200::Evaluator::apply_galois_multiply_plain_add_inplace and diagonal_sum on
// CiphertextBatch (include/seal_b200/evaluator.hpp) against the reference's chains on the same seal::Ciphertexts
// (oracle/ref_diagsum.cpp): words and metadata (parms_id, NTT form, scale bits, correction factor, size) of every member, and
// exception types and messages in the chain's order.  Covers CKKS, BFV and BGV, both key types, shared and per-member diagonals,
// NTT-form and coefficient-form diagonals, a destination that is the input, BGV correction factors that differ (the chain path),
// the NAF fallback, a key cache of one byte, and "scale mismatch" between CKKS diagonals of different scales.
// Built by oracle/diagsum.mk into oracle/_ref/bin/shim_diagsum_test; run by tests/test_gpu_diagonal_sum.py.
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

void ref_apply_galois_multiply_plain_add(const seal::Evaluator &ev, Ciphertext &destination, const Ciphertext &encrypted, uint32_t galois_elt,
                                         const Plaintext &plain, const GaloisKeys &galois_keys);
void ref_diagonal_sum(const seal::Evaluator &ev, bool ckks, const Ciphertext &encrypted, const std::vector<int> &steps,
                      const std::vector<Plaintext> &diagonals, const GaloisKeys &galois_keys, Ciphertext &destination);

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


// one diagonal per member (or one for the batch): random slot values at the level of `level`, NTT form for CKKS (scale 2^30 or
// `scale`), coefficient form for BFV / BGV unless ntt (BGV: transform_to_ntt_inplace)
static std::vector<Plaintext> diagonals(Setup &s, size_t count, const parms_id_type &level, std::mt19937_64 &rng, bool ntt = false,
                                        double scale = 0)
{
    std::vector<Plaintext> out(count);
    const size_t n = s.context.first_context_data()->parms().poly_modulus_degree();
    for (auto &p : out)
    {
        if (s.ckks())
        {
            CKKSEncoder e(s.context);
            std::vector<double> v(e.slot_count());
            for (auto &x : v)
                x = static_cast<double>(rng() % 2000) / 1000.0 - 1.0;
            e.encode(v, level, scale ? scale : std::pow(2.0, 30), p);
        }
        else
        {
            BatchEncoder e(s.context);
            const uint64_t t = s.context.first_context_data()->parms().plain_modulus().value();
            std::vector<uint64_t> v(n);
            for (auto &x : v)
                x = rng() % t;
            e.encode(v, p);
            if (ntt)
                s.rev.transform_to_ntt_inplace(p, level);
        }
    }
    return out;
}

static seal_b200::PlaintextBatch upload_plains(Setup &s, const std::vector<Plaintext> &p)
{
    seal_b200::PlaintextBatch b;
    s.ev.upload(p, b);
    return b;
}

// member b's plaintext of a diagonal that holds one plaintext (shared) or one per member
static const Plaintext &member(const std::vector<Plaintext> &d, size_t b) { return d.size() == 1 ? d[0] : d[b]; }

template <class Keys>
static void check_mpa(Setup &s, const std::vector<Ciphertext> &dst, const std::vector<Ciphertext> &src, uint32_t elt,
                      const std::vector<Plaintext> &plain, const Keys &keys, const std::string &what)
{
    seal_b200::CiphertextBatch d, e;
    s.ev.upload(dst, d);
    s.ev.upload(src, e);
    const seal_b200::PlaintextBatch p = upload_plains(s, plain);
    s.ev.apply_galois_multiply_plain_add_inplace(d, e, elt, p, keys);
    std::vector<Ciphertext> want = dst;
    for (size_t b = 0; b < want.size(); b++)
        ref_apply_galois_multiply_plain_add(s.rev, want[b], src[b], elt, member(plain, b), s.gk);
    compare(s, d, want, what);
    compare(s, e, src, what + " (input unchanged)");
    if (s.ckks()) // destination = encrypted: its scale is not the product's
        return;
    s.ev.apply_galois_multiply_plain_add_inplace(e, e, elt, p, keys);
    std::vector<Ciphertext> self = src;
    for (size_t b = 0; b < self.size(); b++)
    {
        const Ciphertext x = self[b];
        ref_apply_galois_multiply_plain_add(s.rev, self[b], x, elt, member(plain, b), s.gk);
    }
    compare(s, e, self, what + " (destination = encrypted)");
}

template <class Keys>
static void check_diag(Setup &s, const std::vector<Ciphertext> &x, const std::vector<int> &steps, const std::vector<std::vector<Plaintext>> &diags,
                       const Keys &keys, const GaloisKeys &ref_keys, const std::string &what)
{
    seal_b200::CiphertextBatch e, y;
    s.ev.upload(x, e);
    std::vector<seal_b200::PlaintextBatch> d;
    for (auto &p : diags)
        d.push_back(upload_plains(s, p));
    s.ev.diagonal_sum(e, steps, d, keys, y);
    std::vector<Ciphertext> want(x.size());
    for (size_t b = 0; b < x.size(); b++)
    {
        std::vector<Plaintext> db;
        for (auto &p : diags)
            db.push_back(member(p, b));
        ref_diagonal_sum(s.rev, s.ckks(), x[b], steps, db, ref_keys, want[b]);
    }
    compare(s, y, want, what);
    compare(s, e, x, what + " (input unchanged)");
}

// the first failing call of the chain decides the exception, for ours and for the reference (member 0); ours writes nothing
static void check_diag_throw(Setup &s, const std::vector<Ciphertext> &x, const std::vector<int> &steps,
                             const std::vector<std::vector<Plaintext>> &diags, const GaloisKeys &keys, const std::string &what)
{
    seal_b200::CiphertextBatch e, y;
    s.ev.upload(x, e);
    s.ev.upload(x, y);
    std::vector<seal_b200::PlaintextBatch> d;
    for (auto &p : diags)
        d.push_back(upload_plains(s, p));
    std::vector<Plaintext> d0;
    for (auto &p : diags)
        d0.push_back(p[0]);
    Ciphertext r;
    same_throw([&] { s.ev.diagonal_sum(e, steps, d, keys, y); }, [&] { ref_diagonal_sum(s.rev, s.ckks(), x[0], steps, d0, keys, r); }, what);
    compare(s, y, x, what + " (destination unchanged)");
}

static void check_mpa_throw(Setup &s, const std::vector<Ciphertext> &dst, const std::vector<Ciphertext> &src, uint32_t elt,
                            const std::vector<Plaintext> &plain, const GaloisKeys &keys, const std::string &what)
{
    seal_b200::CiphertextBatch d, e;
    s.ev.upload(dst, d);
    s.ev.upload(src, e);
    const seal_b200::PlaintextBatch p = upload_plains(s, plain);
    Ciphertext r = dst[0];
    same_throw([&] { s.ev.apply_galois_multiply_plain_add_inplace(d, e, elt, p, keys); },
               [&] { ref_apply_galois_multiply_plain_add(s.rev, r, src[0], elt, plain[0], keys); }, what);
    compare(s, d, dst, what + " (destination unchanged)");
}

static EncryptionParameters parms_of(scheme_type scheme, size_t n, uint64_t t)
{
    EncryptionParameters p(scheme);
    p.set_poly_modulus_degree(n);
    p.set_coeff_modulus(CoeffModulus::Create(n, { 50, 40, 40, 50 }));
    if (scheme != scheme_type::ckks)
        p.set_plain_modulus(t);
    return p;
}

static void scheme_checks(scheme_type scheme, const std::string &name)
{
    const size_t n = 4096, B = 3;
    Setup s(parms_of(scheme, n, PlainModulus::Batching(n, 20).value()));
    std::mt19937_64 rng(0xD1A6 + static_cast<int>(scheme));
    const std::vector<Ciphertext> x = s.encrypt(B, rng), y0 = s.encrypt(B, rng);
    const parms_id_type top = x[0].parms_id();
    const auto elt = [&](int step) { return s.context.first_context_data()->galois_tool()->get_elt_from_step(step); };
    const bool bgv = scheme == scheme_type::bgv;
    // the fused single term takes NTT-form plaintexts (CKKS's own; BGV's transformed); BFV's coefficient-form one takes the chain.
    const std::vector<Plaintext> p1 = diagonals(s, 1, top, rng, bgv), pB = diagonals(s, B, top, rng, bgv);
    // CKKS: the destination at the product's scale 2^60 (add_inplace's scale check); its words are any ciphertext's
    std::vector<Ciphertext> y = y0;
    if (s.ckks())
        for (auto &c : y)
            c.scale() *= std::pow(2.0, 30);
    for (int step : { 1, -1, 8 })
    {
        check_mpa(s, y, x, elt(step), p1, s.gk, name + " apply_galois_multiply_plain_add step " + std::to_string(step) + " (GaloisKeys)");
        check_mpa(s, y, x, elt(step), pB, s.dgk, name + " apply_galois_multiply_plain_add step " + std::to_string(step) + " per member (DeviceGaloisKeys)");
    }
    check_mpa(s, y, x, static_cast<uint32_t>(2 * n - 1), pB, s.dgk, name + " apply_galois_multiply_plain_add element 2n - 1");
    // diagonal sums: identity first, in the middle, absent; shared and per-member mixed; both keys; BGV in both plaintext forms
    std::vector<std::vector<Plaintext>> d4 = { diagonals(s, 1, top, rng), diagonals(s, B, top, rng), diagonals(s, 1, top, rng),
                                               diagonals(s, B, top, rng) };
    check_diag(s, x, { 0, 1, -1, 4 }, d4, s.gk, s.gk, name + " diagonal_sum identity first (GaloisKeys)");
    check_diag(s, x, { 1, 0, -1, 4 }, d4, s.dgk, s.gk, name + " diagonal_sum identity in the middle (DeviceGaloisKeys)");
    check_diag(s, x, { 2, -2, 1, 1 }, d4, s.gk, s.gk, name + " diagonal_sum no identity, a repeated step");
    check_diag(s, x, { 0 }, { d4[1] }, s.gk, s.gk, name + " diagonal_sum identity only");
    if (bgv)
    {
        std::vector<std::vector<Plaintext>> dn = { diagonals(s, 1, top, rng, true), diagonals(s, B, top, rng, true) };
        check_diag(s, x, { 0, 1 }, dn, s.dgk, s.gk, name + " diagonal_sum NTT-form diagonals");
        check_diag(s, x, { 0, 1 }, { d4[0], dn[1] }, s.dgk, s.gk, name + " diagonal_sum mixed forms (the chain)");
    }
    // a lower level
    std::vector<Ciphertext> xl = x;
    for (auto &c : xl)
        s.rev.mod_switch_to_next_inplace(c);
    const parms_id_type low = xl[0].parms_id();
    check_diag(s, xl, { 0, 1, 8 }, { diagonals(s, 1, low, rng), diagonals(s, B, low, rng), diagonals(s, 1, low, rng) }, s.dgk, s.gk,
               name + " diagonal_sum below the top level");
    // the NAF fallback: keys for 1, -1, 2, -2, 4, 8 only; step 3 = 4 - 1 has no key of its own
    GaloisKeys naf;
    s.keygen.create_galois_keys(std::vector<int>{ 1, -1, 2, -2, 4, 8 }, naf);
    check_diag(s, x, { 0, 3, 1 }, { d4[0], d4[1], d4[2] }, naf, naf, name + " diagonal_sum NAF fallback");
    // a key cache below the call's keys: every key of the call stays cached while it runs
    s.ev.set_key_cache_limit(1);
    check_diag(s, x, { 1, 2, 4, 8 }, d4, s.gk, s.gk, name + " diagonal_sum with a key cache of one byte");
    check_mpa(s, y, x, elt(4), p1, s.gk, name + " apply_galois_multiply_plain_add with a key cache of one byte");
    s.ev.set_key_cache_limit(std::size_t(24) << 30);
    // errors, in the chain's order
    GaloisKeys one;
    s.keygen.create_galois_keys(std::vector<int>{ 1 }, one);
    check_diag_throw(s, x, { 0, 1, 2 }, { d4[0], d4[1], d4[2] }, one, name + " diagonal_sum missing key");
    check_diag_throw(s, x, { 0, static_cast<int>(n) }, { d4[0], d4[1] }, s.gk, name + " diagonal_sum step count too large");
    check_mpa_throw(s, y, x, elt(3), p1, one, name + " apply_galois_multiply_plain_add missing key");
    if (s.ckks())
    {
        check_diag_throw(s, x, { 0, 1 }, { d4[0], diagonals(s, 1, top, rng, false, std::pow(2.0, 31)) }, s.gk,
                         name + " diagonal_sum scale mismatch");
        check_diag_throw(s, x, { 0, 1 }, { d4[0], diagonals(s, 1, low, rng) }, s.gk, name + " diagonal_sum diagonal at another level");
        check_mpa_throw(s, y, x, elt(1), diagonals(s, 1, top, rng, false, std::pow(2.0, 31)), s.gk,
                        name + " apply_galois_multiply_plain_add scale mismatch");
    }
    if (bgv)
    {
        // correction factors that differ: a fresh encryption at the next level against mod-switched ones (the chain path)
        std::vector<Ciphertext> fresh(B);
        for (auto &c : fresh)
            s.enc.encrypt_zero(low, c);
        check_mpa(s, fresh, xl, elt(1), diagonals(s, 1, low, rng, true), s.gk, name + " apply_galois_multiply_plain_add differing correction factors");
    }
    {
        seal_b200::CiphertextBatch e;
        s.ev.upload(x, e);
        std::string m;
        std::vector<seal_b200::PlaintextBatch> d;
        d.push_back(upload_plains(s, d4[0]));
        g_checks++;
        if (caught([&] { s.ev.diagonal_sum(e, {}, {}, s.gk, e); }, &m) != typeid(std::invalid_argument).name())
            fail(name + " diagonal_sum empty");
        g_checks++;
        if (caught([&] { s.ev.diagonal_sum(e, { 0, 1 }, d, s.gk, e); }, &m) != typeid(std::invalid_argument).name())
            fail(name + " diagonal_sum one diagonal for two steps");
        g_checks++;
        if (caught([&] { s.ev.diagonal_sum(e, { 0 }, d, s.gk, e); }, &m) != typeid(std::invalid_argument).name())
            fail(name + " diagonal_sum destination = encrypted");
        compare(s, e, x, name + " diagonal_sum argument errors (batch unchanged)");
    }
}

int main()
{
    for (auto [scheme, name] : { std::pair<scheme_type, const char *>{ scheme_type::ckks, "CKKS" }, { scheme_type::bfv, "BFV" },
                                 { scheme_type::bgv, "BGV" } })
    {
        std::string m;
        const std::string t = caught([&] { scheme_checks(scheme, name); }, &m);
        if (t != "none")
            fail(std::string(name) + ": unexpected exception " + t + " '" + m + "'");
    }
    std::printf("%d checks, %d failures\n", g_checks, g_fail);
    if (g_fail)
        return 1;
    std::printf("shim_diagsum_test ok\n");
    return 0;
}
