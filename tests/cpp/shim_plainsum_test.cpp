// tests/cpp/shim_plainsum_test.cpp -- seal_b200::Evaluator::multiply_plain_sum on CiphertextBatch / PlaintextBatch
// (include/seal_b200/evaluator.hpp) against the reference's chain on the same seal::Ciphertexts and seal::Plaintexts
// (oracle/ref_plainsum.cpp: multiply_plain_inplace of every term, then add_many): words and metadata of every member of every
// output, and exception types and messages.  Covers CKKS (with a baby-step/giant-step-shaped case: K rotations of one ciphertext
// times an M x K matrix of diagonals), BFV in all four NTT-form combinations, BGV with differing correction factors, shared and
// per-member plaintexts and mixed sizes.
// Built by oracle/plainsum.mk into oracle/_ref/bin/shim_plainsum_test; run by tests/test_gpu_plain_sum.py.
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

std::vector<Ciphertext> ref_multiply_plain_sum(const seal::Evaluator &ev, const std::vector<Ciphertext> &encrypteds,
                                               const std::vector<const Plaintext *> &plains);

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
    Encryptor enc;
    seal::Evaluator rev;
    seal_b200::Evaluator ev;
    explicit Setup(const EncryptionParameters &parms)
        : context(parms, true, sec_level_type::none), keygen(context), pk(make_pk(keygen)), enc(context, pk), rev(context), ev(context)
    {}
    static PublicKey make_pk(KeyGenerator &k)
    {
        PublicKey p;
        k.create_public_key(p);
        return p;
    }
};

// cts [K][B]; plains [M K][count], count 1 (shared) or B.  Both overloads against the chain, member by member.
static void check_sum(Setup &s, const std::vector<std::vector<Ciphertext>> &cts, const std::vector<std::vector<Plaintext>> &plains,
                      const std::string &what)
{
    const size_t K = cts.size(), M = plains.size() / K, B = cts[0].size();
    std::vector<seal_b200::CiphertextBatch> cb(K);
    std::vector<seal_b200::PlaintextBatch> pb(M * K);
    for (size_t i = 0; i < K; i++)
        s.ev.upload(cts[i], cb[i]);
    for (size_t x = 0; x < M * K; x++)
        s.ev.upload(plains[x], pb[x]);
    std::vector<seal_b200::CiphertextBatch> outs;
    s.ev.multiply_plain_sum(cb, pb, outs);
    g_checks++;
    if (outs.size() != M)
    {
        g_fail++;
        std::printf("FAIL %s: %zu outputs\n", what.c_str(), outs.size());
        return;
    }
    std::vector<std::vector<Ciphertext>> got(M);
    for (size_t j = 0; j < M; j++)
        s.ev.download(outs[j], got[j]);
    for (size_t b = 0; b < B; b++)
    {
        std::vector<Ciphertext> col;
        std::vector<const Plaintext *> ps;
        for (size_t i = 0; i < K; i++)
            col.push_back(cts[i][b]);
        for (size_t x = 0; x < M * K; x++)
            ps.push_back(&plains[x][plains[x].size() == 1 ? 0 : b]);
        const std::vector<Ciphertext> want = ref_multiply_plain_sum(s.rev, col, ps);
        for (size_t j = 0; j < M; j++)
        {
            g_checks++;
            if (!same_ct(got[j][b], want[j]))
            {
                g_fail++;
                std::printf("FAIL %s: output %zu member %zu differs\n", what.c_str(), j, b);
            }
        }
    }
    // the single-destination overload gives output 0's words and metadata
    std::vector<seal_b200::PlaintextBatch> first(K);
    for (size_t i = 0; i < K; i++)
        s.ev.upload(plains[i], first[i]);
    seal_b200::CiphertextBatch one;
    s.ev.multiply_plain_sum(cb, first, one);
    std::vector<Ciphertext> g1;
    s.ev.download(one, g1);
    for (size_t b = 0; b < B; b++)
    {
        g_checks++;
        if (!same_ct(g1[b], got[0][b]))
        {
            g_fail++;
            std::printf("FAIL %s: single-destination overload, member %zu\n", what.c_str(), b);
        }
    }
}

// the first failing call of the chain decides the exception, for ours and for the reference (member 0)
static void check_throw(Setup &s, const std::vector<std::vector<Ciphertext>> &cts, const std::vector<std::vector<Plaintext>> &plains,
                        const std::string &what)
{
    const size_t K = cts.size();
    std::vector<seal_b200::CiphertextBatch> cb(K);
    std::vector<seal_b200::PlaintextBatch> pb(plains.size());
    for (size_t i = 0; i < K; i++)
        s.ev.upload(cts[i], cb[i]);
    for (size_t x = 0; x < plains.size(); x++)
        s.ev.upload(plains[x], pb[x]);
    std::vector<seal_b200::CiphertextBatch> outs(1);
    std::vector<Ciphertext> col;
    std::vector<const Plaintext *> ps;
    for (size_t i = 0; i < K; i++)
        col.push_back(cts[i][0]);
    for (auto &p : plains)
        ps.push_back(&p[0]);
    same_throw([&] { s.ev.multiply_plain_sum(cb, pb, outs); }, [&] { ref_multiply_plain_sum(s.rev, col, ps); }, what);
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

static std::vector<Plaintext> encode_ckks(CKKSEncoder &enc, size_t count, parms_id_type pid, double scale, std::mt19937_64 &rng)
{
    std::vector<Plaintext> out(count);
    for (auto &p : out)
    {
        std::vector<double> v(enc.slot_count());
        for (auto &x : v)
            x = static_cast<double>(rng() % 2000) / 1000.0 - 1.0;
        enc.encode(v, pid, scale, p);
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
    std::mt19937_64 rng(11);
    const double scale = std::pow(2.0, 40);
    const size_t B = 3, K = 3, M = 2;
    std::vector<std::vector<Ciphertext>> cts;
    for (size_t i = 0; i < K; i++)
        cts.push_back(encrypt_ckks(s, enc, B, scale, rng));
    for (auto &c : cts[1]) // a size-3 term; its scale is set so that its products match the others' (2^80) with plaintexts at 2^20
    {
        Ciphertext y = c;
        s.rev.multiply_inplace(c, y);
        c.scale() = std::pow(2.0, 60);
    }
    const parms_id_type pid = cts[0][0].parms_id();
    std::vector<std::vector<Plaintext>> plains;
    for (size_t x = 0; x < M * K; x++)
        plains.push_back(encode_ckks(enc, x % 2 ? 1 : B, pid, x % K == 1 ? std::pow(2.0, 20) : scale, rng));
    check_sum(s, cts, plains, "CKKS K=3 M=2");

    // baby-step/giant-step shape: K rotations of one ciphertext per member times an M x K matrix of diagonals
    {
        GaloisKeys gk;
        s.keygen.create_galois_keys(std::vector<int>{ 1, 2, 3 }, gk);
        const size_t KB = 4, MB = 3, BB = 2;
        const std::vector<Ciphertext> base = encrypt_ckks(s, enc, BB, scale, rng);
        std::vector<std::vector<Ciphertext>> rot(KB, std::vector<Ciphertext>(BB));
        for (size_t r = 0; r < KB; r++)
            for (size_t b = 0; b < BB; b++)
            {
                rot[r][b] = base[b];
                if (r)
                    s.rev.rotate_vector_inplace(rot[r][b], static_cast<int>(r), gk);
            }
        std::vector<std::vector<Plaintext>> diag;
        for (size_t x = 0; x < MB * KB; x++)
            diag.push_back(encode_ckks(enc, 1, base[0].parms_id(), scale, rng));
        check_sum(s, rot, diag, "CKKS baby-step/giant-step");
    }

    // errors: the first failing call of the chain
    std::vector<std::vector<Ciphertext>> two = { cts[0], cts[2] };
    check_throw(s, two, { plains[0], encode_ckks(enc, B, pid, std::pow(2.0, 30), rng) }, "CKKS scale mismatch (add_many)");
    auto next = s.context.get_context_data(pid)->next_context_data()->parms_id();
    check_throw(s, two, { plains[0], encode_ckks(enc, B, next, scale, rng) }, "CKKS parameter mismatch (multiply_plain of term 1)");
    check_throw(s, two, { encode_ckks(enc, B, pid, std::pow(2.0, 110), rng), plains[0] }, "CKKS scale out of bounds (term 0)");
    check_throw(s, { cts[0], cts[1] }, { plains[0], plains[2] }, "CKKS scale mismatch of a size-3 term");
    // ours only: empty operands, a plaintext count that is neither 1 nor B, too few plaintexts
    std::vector<seal_b200::CiphertextBatch> cb(2);
    std::vector<seal_b200::PlaintextBatch> pb(3);
    s.ev.upload(cts[0], cb[0]), s.ev.upload(cts[2], cb[1]);
    s.ev.upload(plains[0], pb[0]), s.ev.upload(plains[2], pb[1]);
    s.ev.upload(std::vector<Plaintext>(plains[0].begin(), plains[0].begin() + 2), pb[2]);
    std::vector<seal_b200::CiphertextBatch> outs;
    std::string m;
    g_checks += 3;
    if (caught([&] { s.ev.multiply_plain_sum({}, {}, outs); }, &m) != typeid(std::invalid_argument).name() || m != "encrypteds cannot be empty")
        g_fail++, std::printf("FAIL empty: %s\n", m.c_str());
    std::vector<seal_b200::PlaintextBatch> bad(2);
    s.ev.upload(plains[0], bad[0]), s.ev.upload(std::vector<Plaintext>(plains[0].begin(), plains[0].begin() + 2), bad[1]);
    if (caught([&] { s.ev.multiply_plain_sum(cb, bad, outs); }, &m) != typeid(std::invalid_argument).name() ||
        m != "plain batch size must be 1 or the ciphertext batch size")
        g_fail++, std::printf("FAIL plain count: %s\n", m.c_str());
    if (caught([&] { s.ev.multiply_plain_sum(cb, pb, outs); }, &m) != typeid(std::invalid_argument).name() ||
        m != "plains must hold K plaintext batches per destination")
        g_fail++, std::printf("FAIL plain list: %s\n", m.c_str());
}

static EncryptionParameters integer_parms(scheme_type scheme, size_t n)
{
    EncryptionParameters parms(scheme);
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::Create(n, { 40, 40, 40, 40 }));
    parms.set_plain_modulus(PlainModulus::Batching(n, 20));
    return parms;
}

static std::vector<Plaintext> coeff_plains(Setup &s, size_t count, std::mt19937_64 &rng)
{
    const auto &parms = s.context.first_context_data()->parms();
    std::vector<Plaintext> out(count);
    for (auto &p : out)
    {
        p.resize(parms.poly_modulus_degree());
        for (size_t i = 0; i < parms.poly_modulus_degree(); i++)
            p[i] = rng() % parms.plain_modulus().value();
    }
    return out;
}

static void integer_checks(scheme_type scheme, const char *name)
{
    Setup s(integer_parms(scheme, 4096));
    std::mt19937_64 rng(13);
    const bool bgv = scheme == scheme_type::bgv;
    const size_t B = 3, K = 4, M = 2;
    std::vector<std::vector<Ciphertext>> cts(K, std::vector<Ciphertext>(B));
    for (size_t i = 0; i < K; i++)
        for (size_t b = 0; b < B; b++)
        {
            std::vector<Plaintext> p = coeff_plains(s, 1, rng);
            s.enc.encrypt(p[0], cts[i][b]);
            if (i == 1) // a size-3 term
            {
                Ciphertext y = cts[i][b];
                s.rev.multiply_inplace(cts[i][b], y);
            }
            if (bgv) // level 2: mod switching gives correction factors other than 1; term 3 is a fresh zero with factor 1
            {
                s.rev.mod_switch_to_next_inplace(cts[i][b]);
                if (i == 3)
                    s.enc.encrypt_zero(cts[0][0].parms_id(), cts[i][b]);
            }
        }
    if (bgv && cts[0][0].correction_factor() == cts[3][0].correction_factor())
        g_fail++, std::printf("FAIL %s: the correction factors do not differ\n", name);
    for (int ct_ntt = 0; ct_ntt < 2; ct_ntt++)
        for (int plain_ntt = 0; plain_ntt < 2; plain_ntt++)
        {
            if (bgv && !ct_ntt)
                continue; // BGV ciphertexts are in NTT form
            std::vector<std::vector<Ciphertext>> c = cts;
            if (ct_ntt && !bgv)
                for (auto &v : c)
                    for (auto &x : v)
                        s.rev.transform_to_ntt_inplace(x);
            std::vector<std::vector<Plaintext>> plains;
            for (size_t x = 0; x < M * K; x++)
            {
                plains.push_back(coeff_plains(s, x % 3 == 1 ? 1 : B, rng));
                if (plain_ntt)
                    for (auto &p : plains.back())
                        s.rev.transform_to_ntt_inplace(p, c[0][0].parms_id());
            }
            check_sum(s, c, plains, std::string(name) + " ct_ntt=" + std::to_string(ct_ntt) + " plain_ntt=" + std::to_string(plain_ntt));
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
    std::printf("shim_plainsum_test ok\n");
    return 0;
}
