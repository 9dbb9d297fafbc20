// tests/cpp/shim_encrypt_test.cpp -- the device-resident members of seal_b200::Encryptor (PlaintextBatch -> CiphertextBatch,
// encrypt_zero into a CiphertextBatch), seal_b200::Decryptor (CiphertextBatch -> PlaintextBatch) and the encoders' decode of a
// PlaintextBatch, against seal::Encryptor / Decryptor / encoders under seeded Blake2xb and Shake256 factories: words, metadata,
// exception types, CKKS decoded doubles as bit patterns, and a CKKS and a BFV chain (encode -> encrypt -> multiply_plain ->
// multiply + relinearize -> rotate -> decrypt -> decode) kept on the device.  Built by oracle/encrypt.mk into
// oracle/_ref/bin/shim_encrypt_test; run by tests/test_gpu_encrypt_batch.py.
#include "seal/seal.h"
#include "seal_b200/batchencoder.hpp"
#include "seal_b200/ckks.hpp"
#include "seal_b200/decryptor.hpp"
#include "seal_b200/encryptor.hpp"
#include "seal_b200/evaluator.hpp"
#include <complex>
#include <cstdio>
#include <cstring>
#include <functional>
#include <memory>
#include <string>
#include <typeinfo>
#include <vector>

using namespace seal;

static int g_checks = 0, g_fail = 0;
#define CHECK(cond)                                                     \
    do                                                                  \
    {                                                                   \
        g_checks++;                                                     \
        if (!(cond))                                                    \
        {                                                               \
            g_fail++;                                                   \
            std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); \
        }                                                               \
    } while (0)

static std::string caught(const std::function<void()> &f, std::string *msg = nullptr)
{
    try
    {
        f();
    }
    catch (const std::exception &e)
    {
        if (msg)
            *msg = e.what();
        return typeid(e).name();
    }
    return "none";
}

// the exception both throw: same type, same message
static void same_throw(const std::function<void()> &ours, const std::function<void()> &theirs, const char *what)
{
    std::string m1, m2;
    const std::string t1 = caught(ours, &m1), t2 = caught(theirs, &m2);
    g_checks++;
    if (t1 != t2 || m1 != m2 || t1 == "none")
    {
        g_fail++;
        std::printf("FAIL %s: ours %s '%s', reference %s '%s'\n", what, t1.c_str(), m1.c_str(), t2.c_str(), m2.c_str());
    }
}

static bool same_ct(const Ciphertext &a, const Ciphertext &b)
{
    const double s1 = a.scale(), s2 = b.scale();
    return a.parms_id() == b.parms_id() && a.size() == b.size() && a.is_ntt_form() == b.is_ntt_form() &&
           a.correction_factor() == b.correction_factor() && std::memcmp(&s1, &s2, sizeof(double)) == 0 &&
           std::memcmp(a.data(), b.data(), a.size() * a.coeff_modulus_size() * a.poly_modulus_degree() * sizeof(std::uint64_t)) == 0;
}

static EncryptionParameters params(scheme_type scheme, std::size_t n, const std::vector<int> &bits, int prng, std::uint64_t seed0)
{
    EncryptionParameters parms(scheme);
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::Create(n, bits));
    if (scheme != scheme_type::ckks)
        parms.set_plain_modulus(PlainModulus::Batching(n, 20));
    prng_seed_type s{};
    s[0] = seed0;
    if (prng == 1)
        parms.set_random_generator(std::make_shared<Blake2xbPRNGFactory>(s));
    else
        parms.set_random_generator(std::make_shared<Shake256PRNGFactory>(s));
    return parms;
}

// One scheme under one factory type: ours and the reference each get their own context with an identically seeded factory,
// so both draw the same seeds in the same order.  Keys come from a third context (parms_id does not depend on the factory).
static void run(scheme_type scheme, int prng)
{
    const bool ckks = scheme == scheme_type::ckks;
    const std::size_t n = 8192, B = 3;
    const std::vector<int> bits = ckks ? std::vector<int>{ 60, 40, 40, 60 } : std::vector<int>{ 50, 50, 50 };
    SEALContext ours(params(scheme, n, bits, prng, 0x5EED), true, sec_level_type::none);
    SEALContext ref(params(scheme, n, bits, prng, 0x5EED), true, sec_level_type::none);
    SEALContext keyctx(params(scheme, n, bits, prng, 0xC0DE), true, sec_level_type::none);
    KeyGenerator keygen(keyctx);
    const SecretKey &sk = keygen.secret_key();
    PublicKey pk;
    keygen.create_public_key(pk);
    RelinKeys rk;
    keygen.create_relin_keys(rk);
    GaloisKeys gk;
    keygen.create_galois_keys(std::vector<int>{ 1 }, gk);

    seal_b200::Evaluator ev(ours);
    seal_b200::Encryptor enc(ours, pk, sk, ev);
    seal_b200::Decryptor dec(ours, sk, ev);
    seal::Encryptor renc(ref, pk, sk);
    seal::Decryptor rdec(ref, sk);
    seal::Evaluator rev(ref);
    const double scale = std::pow(2.0, 40);

    // plaintexts: encoded on the device (ours) and by the reference encoder (words equal: shim_plain_test)
    seal_b200::PlaintextBatch P;
    std::vector<Plaintext> rp(B);
    std::unique_ptr<seal_b200::CKKSEncoder> cenc;
    std::unique_ptr<seal_b200::BatchEncoder> benc;
    std::unique_ptr<seal::CKKSEncoder> rcenc;
    std::unique_ptr<seal::BatchEncoder> rbenc;
    std::vector<std::vector<double>> cvals(B);
    std::vector<std::vector<std::int64_t>> bvals(B);
    if (ckks)
    {
        cenc = std::make_unique<seal_b200::CKKSEncoder>(ours, ev), rcenc = std::make_unique<seal::CKKSEncoder>(ref);
        for (std::size_t b = 0; b < B; b++)
        {
            for (std::size_t i = 0; i < n / 2; i++)
                cvals[b].push_back(std::sin(0.001 * static_cast<double>(i + 7 * b)) * (b + 1));
            rcenc->encode(cvals[b], scale, rp[b]);
        }
        cenc->encode(cvals, ours.first_parms_id(), scale, P);
    }
    else
    {
        benc = std::make_unique<seal_b200::BatchEncoder>(ours, ev), rbenc = std::make_unique<seal::BatchEncoder>(ref);
        const std::int64_t t = static_cast<std::int64_t>(ref.first_context_data()->parms().plain_modulus().value());
        for (std::size_t b = 0; b < B; b++)
        {
            for (std::size_t i = 0; i < n; i++)
                bvals[b].push_back(static_cast<std::int64_t>((i * 7919 + b * 104729) % static_cast<std::size_t>(t)) - t / 2);
            rbenc->encode(bvals[b], rp[b]);
        }
        benc->encode(bvals, P);
    }

    // encrypt_symmetric, encrypt, encrypt_zero_symmetric, encrypt_zero: in this order on both sides (the factories advance alike)
    seal_b200::CiphertextBatch C1, C2, Z1, Z2;
    enc.encrypt_symmetric(P, C1);
    enc.encrypt(P, C2);
    enc.encrypt_zero_symmetric(ours.first_parms_id(), B, Z1);
    enc.encrypt_zero(ours.first_parms_id(), B, Z2);
    std::vector<Ciphertext> r1(B), r2(B), rz1(B), rz2(B);
    for (std::size_t b = 0; b < B; b++)
        renc.encrypt_symmetric(rp[b], r1[b]);
    for (std::size_t b = 0; b < B; b++)
        renc.encrypt(rp[b], r2[b]);
    for (std::size_t b = 0; b < B; b++)
        renc.encrypt_zero_symmetric(ref.first_parms_id(), rz1[b]);
    for (std::size_t b = 0; b < B; b++)
        renc.encrypt_zero(ref.first_parms_id(), rz2[b]);
    const std::pair<seal_b200::CiphertextBatch *, std::vector<Ciphertext> *> pairs[] = { { &C1, &r1 }, { &C2, &r2 }, { &Z1, &rz1 }, { &Z2, &rz2 } };
    for (auto &pr : pairs)
    {
        std::vector<Ciphertext> got;
        ev.download(*pr.first, got);
        CHECK(got.size() == B);
        for (std::size_t b = 0; b < B && b < got.size(); b++)
            CHECK(same_ct(got[b], (*pr.second)[b]));
    }

    // the vector overload (one slab upload, one encryption call, one download) under the same factory sequence
    std::vector<Ciphertext> v1, w1(B);
    enc.encrypt_symmetric(rp, v1);
    for (std::size_t b = 0; b < B; b++)
        renc.encrypt_symmetric(rp[b], w1[b]);
    for (std::size_t b = 0; b < B; b++)
        CHECK(same_ct(v1[b], w1[b]));

    // the chain, on the device between encode and decode: multiply_plain, multiply + relinearize, rotate, decrypt, decode
    ev.multiply_plain_inplace(C1, P);
    ev.relinearize_inplace(C1, rk); // size 2 stays size 2 (a no-op), as in the reference
    ev.multiply_inplace(C1, C2);
    ev.relinearize_inplace(C1, rk);
    if (ckks)
        ev.rotate_vector_inplace(C1, 1, gk);
    else
        ev.rotate_rows_inplace(C1, 1, gk);
    seal_b200::PlaintextBatch D;
    dec.decrypt(C1, D);
    for (std::size_t b = 0; b < B; b++)
    {
        rev.multiply_plain_inplace(r1[b], rp[b]);
        rev.relinearize_inplace(r1[b], rk);
        rev.multiply_inplace(r1[b], r2[b]);
        rev.relinearize_inplace(r1[b], rk);
        if (ckks)
            rev.rotate_vector_inplace(r1[b], 1, gk);
        else
            rev.rotate_rows_inplace(r1[b], 1, gk);
    }
    CHECK(D.batch_size() == B && D.is_ntt_form() == ckks && D.parms_id() == (ckks ? C1.parms_id() : parms_id_zero));
    if (ckks)
    {
        std::vector<std::vector<double>> got;
        std::vector<std::vector<std::complex<double>>> gotc;
        cenc->decode(D, got);
        cenc->decode(D, gotc);
        for (std::size_t b = 0; b < B; b++)
        {
            Plaintext pt;
            rdec.decrypt(r1[b], pt);
            CHECK(D.scale() == pt.scale());
            std::vector<double> want;
            std::vector<std::complex<double>> wantc;
            rcenc->decode(pt, want);
            rcenc->decode(pt, wantc);
            CHECK(got[b].size() == want.size() && std::memcmp(got[b].data(), want.data(), want.size() * sizeof(double)) == 0);
            CHECK(gotc[b].size() == wantc.size() && std::memcmp(gotc[b].data(), wantc.data(), wantc.size() * sizeof(wantc[0])) == 0);
        }
        seal_b200::PlaintextBatch e;
        CHECK(caught([&] { cenc->decode(e, got); }) == typeid(std::invalid_argument).name());
    }
    else
    {
        std::vector<std::vector<std::int64_t>> got;
        std::vector<std::vector<std::uint64_t>> gotu;
        benc->decode(D, got);
        benc->decode(D, gotu);
        for (std::size_t b = 0; b < B; b++)
        {
            Plaintext pt;
            rdec.decrypt(r1[b], pt);
            std::vector<std::int64_t> want;
            std::vector<std::uint64_t> wantu;
            rbenc->decode(pt, want);
            rbenc->decode(pt, wantu);
            CHECK(got[b] == want);
            CHECK(gotu[b] == wantu);
        }
        // an NTT-form plaintext batch is refused with the reference's message
        seal_b200::PlaintextBatch N;
        dec.decrypt(C2, N);
        ev.transform_to_ntt_inplace(N, ours.first_parms_id());
        Plaintext rn;
        rdec.decrypt(r2[0], rn);
        rev.transform_to_ntt_inplace(rn, ref.first_parms_id());
        same_throw([&] { benc->decode(N, gotu); }, [&] { std::vector<std::uint64_t> x; rbenc->decode(rn, x); }, "decode of an NTT-form plaintext");
        same_throw([&] { seal_b200::CiphertextBatch x; enc.encrypt(N, x); }, [&] { Ciphertext x; renc.encrypt(rn, x); }, "encrypt of an NTT-form plaintext");
    }

    // errors: the key that is not set, an empty batch, a batch of another device context
    seal_b200::Encryptor sym_only(ours, sk, ev);
    seal::Encryptor rsym_only(ref, sk);
    same_throw([&] { seal_b200::CiphertextBatch x; sym_only.encrypt(P, x); }, [&] { Ciphertext x; rsym_only.encrypt(rp[0], x); }, "public key is not set");
    seal_b200::PlaintextBatch empty;
    seal_b200::CiphertextBatch x;
    CHECK(caught([&] { enc.encrypt_symmetric(empty, x); }) == typeid(std::invalid_argument).name());
    CHECK(caught([&] { enc.encrypt_zero(ours.first_parms_id(), 0, x); }) == typeid(std::invalid_argument).name());
    seal_b200::Evaluator other(ours);
    seal_b200::Encryptor enc_other(ours, pk, sk, other);
    CHECK(caught([&] { enc_other.encrypt(P, x); }) == typeid(std::invalid_argument).name());
    seal_b200::Decryptor dec_other(ours, sk, other);
    seal_b200::PlaintextBatch y;
    CHECK(caught([&] { dec_other.decrypt(C2, y); }) == typeid(std::invalid_argument).name());
    std::printf("%s prng %d: %d checks\n", ckks ? "CKKS" : scheme == scheme_type::bfv ? "BFV" : "BGV", prng, g_checks);
}

int main()
{
    for (int prng : { 1, 2 })
    {
        run(scheme_type::ckks, prng);
        run(scheme_type::bfv, prng);
        run(scheme_type::bgv, prng);
    }
    if (g_fail)
    {
        std::printf("%d of %d checks failed\n", g_fail, g_checks);
        return 1;
    }
    std::printf("shim_encrypt_test ok: %d checks\n", g_checks);
    return 0;
}
