// tests/cpp/shim_multsum_test.cpp -- seal_b200::Evaluator::multiply_sum and multiply_relinearize_sum on CiphertextBatch
// (include/seal_b200/evaluator.hpp) against the reference's chain on the same seal::Ciphertexts (oracle/ref_multsum.cpp:
// multiply_inplace of every term, add_many, then relinearize_inplace): words and metadata (scale, correction factor, size,
// parms_id, NTT form) of every member of every output, and exception types and messages in the chain's order.  Covers CKKS, BFV
// and BGV (with correction factors that differ between terms and between outputs), M = 1 and M > 1, both key types, squares, and
// a size-3 operand (the chain path).
// Built by oracle/multsum.mk into oracle/_ref/bin/shim_multsum_test; run by tests/test_gpu_multiply_sum.py.
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

std::vector<Ciphertext> ref_multiply_sum(const seal::Evaluator &ev, const std::vector<Ciphertext> &lhs, const std::vector<Ciphertext> &rhs,
                                         const RelinKeys *relin_keys);

static int g_checks = 0, g_fail = 0;

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
    {
        g_fail++;
        std::printf("FAIL %s: ours %s '%s', reference %s '%s'\n", what.c_str(), t1.c_str(), m1.c_str(), t2.c_str(), m2.c_str());
    }
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
    RelinKeys rk;
    Encryptor enc;
    seal::Evaluator rev;
    seal_b200::Evaluator ev;
    seal_b200::DeviceRelinKeys drk;
    explicit Setup(const EncryptionParameters &parms)
        : context(parms, true, sec_level_type::none), keygen(context), pk(make_pk(keygen)), rk(make_rk(keygen)), enc(context, pk), rev(context),
          ev(context)
    {
        ev.upload(rk, drk);
    }
    static PublicKey make_pk(KeyGenerator &k)
    {
        PublicKey p;
        k.create_public_key(p);
        return p;
    }
    static RelinKeys make_rk(KeyGenerator &k)
    {
        RelinKeys r;
        k.create_relin_keys(r);
        return r;
    }
};

using Batches = std::vector<std::vector<Ciphertext>>; // [operand][member]

static std::vector<seal_b200::CiphertextBatch> upload(Setup &s, const Batches &x)
{
    std::vector<seal_b200::CiphertextBatch> out(x.size());
    for (size_t i = 0; i < x.size(); i++)
        s.ev.upload(x[i], out[i]);
    return out;
}

// got [M] batches against the reference chain, member by member (relin: 0 none, otherwise relinearized by the chain)
static void compare(Setup &s, std::vector<seal_b200::CiphertextBatch> &got, const Batches &lhs, const Batches &rhs, bool relin,
                    const std::string &what)
{
    const size_t K = rhs.size(), M = lhs.size() / K, B = rhs[0].size();
    g_checks++;
    if (got.size() != M)
    {
        g_fail++;
        std::printf("FAIL %s: %zu outputs\n", what.c_str(), got.size());
        return;
    }
    std::vector<std::vector<Ciphertext>> h(M);
    for (size_t j = 0; j < M; j++)
        s.ev.download(got[j], h[j]);
    for (size_t b = 0; b < B; b++)
    {
        std::vector<Ciphertext> l, r;
        for (auto &v : lhs)
            l.push_back(v[b]);
        for (auto &v : rhs)
            r.push_back(v[b]);
        const std::vector<Ciphertext> want = ref_multiply_sum(s.rev, l, r, relin ? &s.rk : nullptr);
        for (size_t j = 0; j < M; j++)
        {
            g_checks++;
            if (!same_ct(h[j][b], want[j]))
            {
                g_fail++;
                std::printf("FAIL %s: output %zu member %zu differs\n", what.c_str(), j, b);
            }
        }
    }
}

// every overload on lhs [M K] x rhs [K]: multiply_sum (M outputs, and the single-destination form on row 0), and
// multiply_relinearize_sum with both key types (relin: the sums have size 3, which one relinearization key reduces)
static void check_sum(Setup &s, const Batches &lhs, const Batches &rhs, const std::string &what, bool relin = true)
{
    const size_t K = rhs.size();
    std::vector<seal_b200::CiphertextBatch> l = upload(s, lhs), r = upload(s, rhs), outs;
    s.ev.multiply_sum(l, r, outs);
    compare(s, outs, lhs, rhs, false, what + " multiply_sum");
    if (!relin)
        return;
    std::vector<seal_b200::CiphertextBatch> rl(2);
    s.ev.multiply_relinearize_sum(l, r, s.rk, rl);
    compare(s, rl, lhs, rhs, true, what + " multiply_relinearize_sum (RelinKeys)");
    s.ev.multiply_relinearize_sum(l, r, s.drk, rl);
    compare(s, rl, lhs, rhs, true, what + " multiply_relinearize_sum (DeviceRelinKeys)");
    // the single-destination overloads on the first K left operands
    const Batches lhs0(lhs.begin(), lhs.begin() + static_cast<long>(K));
    std::vector<seal_b200::CiphertextBatch> l0 = upload(s, lhs0), one(1), rone(1);
    s.ev.multiply_sum(l0, r, one[0]);
    compare(s, one, lhs0, rhs, false, what + " multiply_sum (one destination)");
    s.ev.multiply_relinearize_sum(l0, r, s.drk, rone[0]);
    compare(s, rone, lhs0, rhs, true, what + " multiply_relinearize_sum (one destination)");
}

// squares: the same batches on both sides, sum_i x_i^2
static void check_squares(Setup &s, const Batches &x, const std::string &what)
{
    std::vector<seal_b200::CiphertextBatch> v = upload(s, x), one(1);
    s.ev.multiply_relinearize_sum(v, v, s.rk, one[0]);
    compare(s, one, x, x, true, what + " squares");
}

// the first failing call of the chain decides the exception, for ours and for the reference (member 0); the destination stays empty
static void check_throw(Setup &s, const Batches &lhs, const Batches &rhs, bool relin, const std::string &what)
{
    std::vector<seal_b200::CiphertextBatch> l = upload(s, lhs), r = upload(s, rhs), outs(1);
    std::vector<Ciphertext> l0, r0;
    for (auto &v : lhs)
        l0.push_back(v[0]);
    for (auto &v : rhs)
        r0.push_back(v[0]);
    same_throw(
        [&] {
            if (relin)
                s.ev.multiply_relinearize_sum(l, r, s.rk, outs);
            else
                s.ev.multiply_sum(l, r, outs);
        },
        [&] { ref_multiply_sum(s.rev, l0, r0, relin ? &s.rk : nullptr); }, what);
    g_checks++;
    if (outs.size() != 1 || outs[0].batch_size() != 0)
    {
        g_fail++;
        std::printf("FAIL %s: destinations changed\n", what.c_str());
    }
}

static std::vector<Ciphertext> encrypt_ckks(Setup &s, CKKSEncoder &enc, size_t B, double scale, std::mt19937_64 &rng)
{
    std::vector<Ciphertext> out(B);
    for (auto &c : out)
    {
        std::vector<double> v(enc.slot_count());
        for (auto &x : v)
            x = static_cast<double>(rng() % 2000) / 1000.0 - 1.0;
        Plaintext p;
        enc.encode(v, scale, p);
        s.enc.encrypt(p, c);
    }
    return out;
}

static void ckks_checks()
{
    EncryptionParameters parms(scheme_type::ckks);
    const size_t n = 8192;
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::Create(n, { 60, 40, 40, 60 }));
    Setup s(parms);
    CKKSEncoder enc(s.context);
    std::mt19937_64 rng(21);
    const double scale = std::pow(2.0, 40);
    const size_t B = 3, K = 3, M = 2;
    Batches lhs, rhs;
    for (size_t x = 0; x < M * K; x++)
        lhs.push_back(encrypt_ckks(s, enc, B, scale, rng));
    for (size_t i = 0; i < K; i++)
        rhs.push_back(encrypt_ckks(s, enc, B, scale, rng));
    check_sum(s, lhs, rhs, "CKKS K=3 M=2");
    check_squares(s, rhs, "CKKS");

    // a size-3 left operand takes the chain path (scale 2^40 so that its product matches the others' 2^80)
    Batches big = lhs;
    for (auto &c : big[1])
    {
        Ciphertext y = c;
        s.rev.multiply_inplace(c, y);
        c.scale() = scale;
    }
    check_sum(s, big, rhs, "CKKS size-3 operand", false);
    check_throw(s, big, rhs, true, "CKKS size-4 sum: not enough relinearization keys");

    // errors, the first failing call of the chain
    Batches odd = rhs;
    for (auto &c : odd[1])
        c.scale() = std::pow(2.0, 30);
    check_throw(s, lhs, odd, false, "CKKS scale mismatch of term 1 (add_many)");
    Batches low = rhs;
    for (auto &c : low[2])
        s.rev.mod_switch_to_next_inplace(c);
    check_throw(s, lhs, low, false, "CKKS parameter mismatch (multiply of term 2)");
    Batches huge = rhs;
    for (auto &c : huge[0])
        c.scale() = std::pow(2.0, 200);
    check_throw(s, lhs, huge, false, "CKKS scale out of bounds (multiply of term 0)");
    check_throw(s, lhs, low, true, "CKKS parameter mismatch before relinearization");

    // ours only: empty operands, a left list that is not M K batches, a destination among the operands
    std::vector<seal_b200::CiphertextBatch> l = upload(s, lhs), r = upload(s, rhs), outs;
    std::vector<seal_b200::CiphertextBatch> r4 = upload(s, Batches{ rhs[0], rhs[1], rhs[2], rhs[0] }); // 6 left operands are not M x 4
    std::string m;
    g_checks += 3;
    if (caught([&] { s.ev.multiply_sum(l, {}, outs); }, &m) != typeid(std::invalid_argument).name() || m != "encrypteds cannot be empty")
        g_fail++, std::printf("FAIL empty: %s\n", m.c_str());
    if (caught([&] { s.ev.multiply_sum(l, r4, outs); }, &m) != typeid(std::invalid_argument).name() ||
        m != "encrypteds1 must hold K ciphertext batches per destination")
        g_fail++, std::printf("FAIL left list: %s\n", m.c_str());
    if (caught([&] { s.ev.multiply_sum(l, r, r[0]); }, &m) != typeid(std::invalid_argument).name() || m != "encrypteds must be different from destination")
        g_fail++, std::printf("FAIL destination alias: %s\n", m.c_str());
}

static EncryptionParameters integer_parms(scheme_type scheme, size_t n)
{
    EncryptionParameters parms(scheme);
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::Create(n, { 40, 40, 40, 40 }));
    parms.set_plain_modulus(PlainModulus::Batching(n, 20));
    return parms;
}

static std::vector<Ciphertext> encrypt_int(Setup &s, size_t B, std::mt19937_64 &rng)
{
    const auto &parms = s.context.first_context_data()->parms();
    std::vector<Ciphertext> out(B);
    for (auto &c : out)
    {
        Plaintext p(parms.poly_modulus_degree());
        for (size_t i = 0; i < parms.poly_modulus_degree(); i++)
            p[i] = rng() % parms.plain_modulus().value();
        s.enc.encrypt(p, c);
    }
    return out;
}

static void integer_checks(scheme_type scheme, const char *name)
{
    Setup s(integer_parms(scheme, 4096));
    std::mt19937_64 rng(23);
    const bool bgv = scheme == scheme_type::bgv;
    const size_t B = 2, K = 3, M = 2;
    Batches lhs, rhs;
    for (size_t x = 0; x < M * K; x++)
        lhs.push_back(encrypt_int(s, B, rng));
    for (size_t i = 0; i < K; i++)
        rhs.push_back(encrypt_int(s, B, rng));
    if (bgv)
    {
        // level 2: mod switching gives correction factors other than 1; fresh zeros keep factor 1.  The factors of the products
        // differ between the terms of a row and between the rows, so the outputs take different balancing steps
        const bool fresh_l[] = { false, false, true, true, false, false }, fresh_r[] = { false, true, false };
        for (size_t x = 0; x < M * K; x++)
            for (auto &c : lhs[x])
            {
                s.rev.mod_switch_to_next_inplace(c);
                if (fresh_l[x])
                    s.enc.encrypt_zero(c.parms_id(), c);
            }
        for (size_t i = 0; i < K; i++)
            for (auto &c : rhs[i])
            {
                s.rev.mod_switch_to_next_inplace(c);
                if (fresh_r[i])
                    s.enc.encrypt_zero(c.parms_id(), c);
            }
        if (lhs[0][0].correction_factor() == lhs[2][0].correction_factor())
            g_fail++, std::printf("FAIL %s: the correction factors do not differ\n", name);
    }
    check_sum(s, lhs, rhs, std::string(name) + " K=3 M=2");
    check_squares(s, rhs, name);
    Batches big = lhs;
    for (auto &c : big[4])
    {
        Ciphertext y = c;
        s.rev.multiply_inplace(c, y);
    }
    check_sum(s, big, rhs, std::string(name) + " size-3 operand", false);
    check_throw(s, big, rhs, true, std::string(name) + " size-4 sum: not enough relinearization keys");
    if (!bgv)
    {
        Batches ntt = rhs;
        for (auto &c : ntt[1])
            s.rev.transform_to_ntt_inplace(c);
        check_throw(s, lhs, ntt, false, std::string(name) + " NTT-form operand (multiply of term 1)");
    }
}

int main()
{
    ckks_checks();
    integer_checks(scheme_type::bfv, "BFV");
    integer_checks(scheme_type::bgv, "BGV");
    std::printf("%d checks, %d failures\n", g_checks, g_fail);
    if (g_fail)
        return 1;
    std::printf("shim_multsum_test ok\n");
    return 0;
}
