// tests/cpp/shim_plain_test.cpp -- seal_b200::PlaintextBatch and the plaintext members of seal_b200::Evaluator on CiphertextBatch
// (include/seal_b200/evaluator.hpp), with the device encoders (batchencoder.hpp, ckks.hpp), against seal::Evaluator on
// seal::Ciphertexts made by seal::Encryptor: words after each chain, metadata after every step, exception types and messages.
// Built by oracle/plain.mk into oracle/_ref/bin/shim_plain_test; run by tests/test_gpu_plain_batch.py.
#include "seal/seal.h"
#include "seal_b200/batchencoder.hpp"
#include "seal_b200/ckks.hpp"
#include "seal_b200/evaluator.hpp"
#include <cmath>
#include <cstdio>
#include <functional>
#include <cstring>
#include <random>
#include <string>
#include <typeinfo>
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

static bool same_meta(const seal_b200::CiphertextBatch &b, const Ciphertext &r)
{
    const double s1 = b.scale(), s2 = r.scale();
    return b.parms_id() == r.parms_id() && b.size() == r.size() && b.is_ntt_form() == r.is_ntt_form() &&
           b.correction_factor() == r.correction_factor() && std::memcmp(&s1, &s2, sizeof(double)) == 0;
}

static bool same_ct(const Ciphertext &a, const Ciphertext &b)
{
    const double s1 = a.scale(), s2 = b.scale();
    return a.parms_id() == b.parms_id() && a.size() == b.size() && a.is_ntt_form() == b.is_ntt_form() &&
           a.correction_factor() == b.correction_factor() && std::memcmp(&s1, &s2, sizeof(double)) == 0 &&
           a.dyn_array().size() == b.dyn_array().size() && std::memcmp(a.data(), b.data(), a.dyn_array().size() * sizeof(uint64_t)) == 0;
}

static bool same_plain(const Plaintext &a, const Plaintext &b)
{
    const double s1 = a.scale(), s2 = b.scale();
    return a.coeff_count() == b.coeff_count() && a.parms_id() == b.parms_id() && std::memcmp(&s1, &s2, sizeof(double)) == 0 &&
           std::memcmp(a.data(), b.data(), a.coeff_count() * sizeof(uint64_t)) == 0;
}

static void same_batch(const seal_b200::Evaluator &ev, const seal_b200::CiphertextBatch &b, const std::vector<Ciphertext> &want, const char *what)
{
    std::vector<Ciphertext> got;
    ev.download(b, got);
    CHECK(got.size() == want.size());
    for (size_t i = 0; i < got.size() && i < want.size(); i++)
        if (!same_ct(got[i], want[i]))
        {
            g_checks++, g_fail++;
            std::printf("FAIL %s: ciphertext %zu differs\n", what, i);
        }
}

static void same_plains(const seal_b200::Evaluator &ev, const seal_b200::PlaintextBatch &b, const std::vector<Plaintext> &want, const char *what)
{
    std::vector<Plaintext> got;
    ev.download(b, got);
    CHECK(got.size() == want.size());
    for (size_t i = 0; i < got.size() && i < want.size(); i++)
    {
        Plaintext w = want[i]; // coefficient-form plaintexts come back zero-padded to n words
        if (!w.is_ntt_form() && w.coeff_count() < got[i].coeff_count())
            w.resize(got[i].coeff_count());
        if (!same_plain(got[i], w))
        {
            g_checks++, g_fail++;
            std::printf("FAIL %s: plaintext %zu differs\n", what, i);
        }
    }
}

static void ckks_chain()
{
    EncryptionParameters parms(scheme_type::ckks);
    const size_t n = 8192, B = 4;
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::Create(n, { 60, 40, 40, 60 }));
    SEALContext context(parms, true, sec_level_type::none);
    KeyGenerator keygen(context);
    PublicKey pk;
    keygen.create_public_key(pk);
    GaloisKeys gk;
    keygen.create_galois_keys(std::vector<int>{ 1 }, gk);
    Encryptor encryptor(context, pk);
    seal::CKKSEncoder renc(context);
    seal::Evaluator rev(context);
    seal_b200::Evaluator ev(context);
    seal_b200::CKKSEncoder denc(context, ev);
    const double scale = std::pow(2.0, 40);
    const auto top = context.first_parms_id(), next = context.first_context_data()->next_context_data()->parms_id();
    std::mt19937_64 rng(11);
    std::uniform_real_distribution<double> u(-1.0, 1.0);
    auto vec = [&](size_t count) {
        std::vector<double> v(count);
        for (auto &x : v)
            x = u(rng);
        return v;
    };
    std::vector<Ciphertext> cts(B);
    for (auto &c : cts)
    {
        Plaintext p;
        renc.encode(vec(n / 2), scale, p);
        encryptor.encrypt(p, c);
    }
    seal_b200::CiphertextBatch cb;
    ev.upload(cts, cb);

    // one shared plaintext, encoded on the device
    const std::vector<double> w = vec(n / 2);
    seal_b200::PlaintextBatch pw;
    denc.encode(std::vector<std::vector<double>>{ w }, top, scale, pw);
    Plaintext rw;
    renc.encode(w, top, scale, rw);
    same_plains(ev, pw, { rw }, "CKKS device encode");

    // errors before anything is written: a plaintext batch of the wrong size, parms_id and scale mismatches, NTT forms
    {
        seal_b200::PlaintextBatch p3;
        denc.encode(std::vector<std::vector<double>>{ w, w, w }, top, scale, p3);
        CHECK(caught([&] { ev.multiply_plain_inplace(cb, p3); }) == typeid(std::invalid_argument).name());
        seal_b200::PlaintextBatch plow;
        Plaintext rlow;
        denc.encode(std::vector<std::vector<double>>{ w }, next, scale, plow);
        renc.encode(w, next, scale, rlow);
        Ciphertext c0 = cts[0];
        same_throw([&] { ev.multiply_plain_inplace(cb, plow); }, [&] { rev.multiply_plain_inplace(c0, rlow); }, "CKKS multiply_plain parms mismatch");
        seal_b200::PlaintextBatch pscale;
        Plaintext rscale;
        denc.encode(std::vector<std::vector<double>>{ w }, top, scale * 2, pscale);
        renc.encode(w, top, scale * 2, rscale);
        same_throw([&] { ev.add_plain_inplace(cb, pscale); }, [&] { rev.add_plain_inplace(c0, rscale); }, "CKKS add_plain scale mismatch");
        same_throw([&] { ev.add_plain_inplace(cb, plow); }, [&] { rev.add_plain_inplace(c0, rlow); }, "CKKS add_plain parms mismatch");
        Plaintext rhigh = rlow;
        same_throw([&] { ev.mod_switch_to_inplace(plow, top); }, [&] { rev.mod_switch_to_inplace(rhigh, top); }, "CKKS plaintext to a higher level");
        seal_b200::PlaintextBatch plast;
        ev.upload(std::vector<Plaintext>{ rlow }, plast);
        Plaintext rlast = rlow;
        ev.mod_switch_to_next_inplace(plast);
        rev.mod_switch_to_next_inplace(rlast);
        same_plains(ev, plast, { rlast }, "CKKS plaintext to the last level");
        same_throw([&] { ev.mod_switch_to_next_inplace(plast); }, [&] { rev.mod_switch_to_next_inplace(rlast); }, "CKKS plaintext end of chain");
    }

    ev.multiply_plain_inplace(cb, pw);
    for (auto &c : cts)
        rev.multiply_plain_inplace(c, rw);
    CHECK(same_meta(cb, cts[0]));
    ev.rescale_to_next_inplace(cb);
    for (auto &c : cts)
        rev.rescale_to_next_inplace(c);
    CHECK(same_meta(cb, cts[0]));

    // a shared plaintext at the rescaled scale, encoded at the first level and switched down on the device
    const std::vector<double> a = vec(n / 3);
    seal_b200::PlaintextBatch pa;
    Plaintext ra;
    denc.encode(std::vector<std::vector<double>>{ a }, top, cts[0].scale(), pa);
    renc.encode(a, top, cts[0].scale(), ra);
    ev.mod_switch_to_next_inplace(pa);
    rev.mod_switch_to_next_inplace(ra);
    same_plains(ev, pa, { ra }, "CKKS plaintext mod_switch_to_next");
    ev.add_plain_inplace(cb, pa);
    for (auto &c : cts)
        rev.add_plain_inplace(c, ra);
    CHECK(same_meta(cb, cts[0]));
    ev.rotate_vector_inplace(cb, 1, gk);
    for (auto &c : cts)
        rev.rotate_vector_inplace(c, 1, gk);
    CHECK(same_meta(cb, cts[0]));

    // one plaintext per ciphertext
    std::vector<std::vector<double>> vs(B);
    std::vector<Plaintext> rs(B);
    for (size_t i = 0; i < B; i++)
    {
        vs[i] = vec(n / 2 - i);
        renc.encode(vs[i], cts[0].parms_id(), cts[0].scale(), rs[i]);
    }
    seal_b200::PlaintextBatch ps;
    denc.encode(vs, cts[0].parms_id(), cts[0].scale(), ps);
    ev.sub_plain_inplace(cb, ps);
    for (size_t i = 0; i < B; i++)
        rev.sub_plain_inplace(cts[i], rs[i]);
    CHECK(same_meta(cb, cts[0]));
    same_batch(ev, cb, cts, "CKKS chain");

    // a plaintext uploaded from the host, and mod_switch_to of a plaintext batch
    seal_b200::PlaintextBatch pu;
    ev.upload(std::vector<Plaintext>{ rw }, pu);
    ev.mod_switch_to_inplace(pu, next);
    Plaintext rwn = rw;
    rev.mod_switch_to_inplace(rwn, next);
    same_plains(ev, pu, { rwn }, "CKKS plaintext mod_switch_to");
}

static void bfv_chain()
{
    EncryptionParameters parms(scheme_type::bfv);
    const size_t n = 4096, B = 3;
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::BFVDefault(n));
    parms.set_plain_modulus(PlainModulus::Batching(n, 20));
    SEALContext context(parms, true, sec_level_type::none);
    const uint64_t t = parms.plain_modulus().value();
    KeyGenerator keygen(context);
    PublicKey pk;
    keygen.create_public_key(pk);
    Encryptor encryptor(context, pk);
    seal::BatchEncoder renc(context);
    seal::Evaluator rev(context);
    seal_b200::Evaluator ev(context);
    seal_b200::BatchEncoder denc(context, ev);
    std::mt19937_64 rng(13);
    auto mat = [&]() {
        std::vector<uint64_t> v(n);
        for (auto &x : v)
            x = rng() % t;
        v[0] = 0, v[1] = t - 1, v[2] = (t + 1) / 2, v[3] = (t + 1) / 2 - 1;
        return v;
    };
    std::vector<Ciphertext> cts(B);
    for (auto &c : cts)
    {
        Plaintext p;
        renc.encode(mat(), p);
        encryptor.encrypt(p, c);
    }
    seal_b200::CiphertextBatch cb;
    ev.upload(cts, cb);
    std::vector<std::vector<uint64_t>> ms(B);
    std::vector<Plaintext> rp(B);
    for (size_t i = 0; i < B; i++)
    {
        ms[i] = mat();
        renc.encode(ms[i], rp[i]);
    }
    seal_b200::PlaintextBatch pb;
    denc.encode(ms, pb);
    same_plains(ev, pb, rp, "BFV device encode");

    ev.multiply_plain_inplace(cb, pb); // coefficient form: multiply_plain_normal
    for (size_t i = 0; i < B; i++)
        rev.multiply_plain_inplace(cts[i], rp[i]);
    CHECK(same_meta(cb, cts[0]));
    ev.transform_to_ntt_inplace(pb, cb.parms_id());
    for (auto &p : rp)
        rev.transform_to_ntt_inplace(p, cts[0].parms_id());
    same_plains(ev, pb, rp, "BFV plaintext transform_to_ntt");
    ev.transform_to_ntt_inplace(cb);
    for (auto &c : cts)
        rev.transform_to_ntt_inplace(c);
    CHECK(same_meta(cb, cts[0]));
    ev.multiply_plain_inplace(cb, pb); // both in NTT form
    for (size_t i = 0; i < B; i++)
        rev.multiply_plain_inplace(cts[i], rp[i]);
    CHECK(same_meta(cb, cts[0]));
    {
        Ciphertext c0 = cts[0];
        seal_b200::PlaintextBatch pone;
        denc.encode(std::vector<std::vector<uint64_t>>{ ms[0] }, pone);
        Plaintext rone;
        renc.encode(ms[0], rone);
        same_throw([&] { ev.add_plain_inplace(cb, pone); }, [&] { rev.add_plain_inplace(c0, rone); }, "BFV add_plain on NTT-form ciphertexts");
    }
    ev.transform_from_ntt_inplace(cb);
    for (auto &c : cts)
        rev.transform_from_ntt_inplace(c);
    {
        Ciphertext c0 = cts[0];
        same_throw([&] { ev.add_plain_inplace(cb, pb); }, [&] { rev.add_plain_inplace(c0, rp[0]); }, "BFV add_plain with an NTT-form plaintext");
    }
    std::vector<int64_t> sv(n / 2);
    for (auto &x : sv)
        x = static_cast<int64_t>(rng() % t) - static_cast<int64_t>(t / 2);
    seal_b200::PlaintextBatch pshared;
    denc.encode(std::vector<std::vector<int64_t>>{ sv }, pshared);
    Plaintext rshared;
    renc.encode(sv, rshared);
    ev.add_plain_inplace(cb, pshared);
    for (auto &c : cts)
        rev.add_plain_inplace(c, rshared);
    CHECK(same_meta(cb, cts[0]));
    same_batch(ev, cb, cts, "BFV chain");

    // an all-zero plaintext makes the result transparent: download throws where the reference's multiply_plain throws
    seal_b200::PlaintextBatch pz;
    denc.encode(std::vector<std::vector<uint64_t>>{ std::vector<uint64_t>(n, 0) }, pz);
    Plaintext rz;
    renc.encode(std::vector<uint64_t>(n, 0), rz);
    Ciphertext c0 = cts[0];
    same_throw(
        [&] {
            ev.multiply_plain_inplace(cb, pz);
            std::vector<Ciphertext> out;
            ev.download(cb, out);
        },
        [&] { rev.multiply_plain_inplace(c0, rz); }, "BFV multiply_plain by zero");
}

static void bgv_chain()
{
    EncryptionParameters parms(scheme_type::bgv);
    const size_t n = 4096, B = 3;
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::Create(n, { 50, 36, 45, 60 }));
    parms.set_plain_modulus(PlainModulus::Batching(n, 20));
    SEALContext context(parms, true, sec_level_type::none);
    const uint64_t t = parms.plain_modulus().value();
    KeyGenerator keygen(context);
    PublicKey pk;
    keygen.create_public_key(pk);
    Encryptor encryptor(context, pk);
    seal::BatchEncoder renc(context);
    seal::Evaluator rev(context);
    seal_b200::Evaluator ev(context);
    seal_b200::BatchEncoder denc(context, ev);
    std::mt19937_64 rng(17);
    auto mat = [&]() {
        std::vector<uint64_t> v(n);
        for (auto &x : v)
            x = rng() % t;
        return v;
    };
    std::vector<Ciphertext> cts(B);
    for (auto &c : cts)
    {
        Plaintext p;
        renc.encode(mat(), p);
        encryptor.encrypt(p, c);
    }
    seal_b200::CiphertextBatch cb;
    ev.upload(cts, cb);
    ev.mod_switch_to_next_inplace(cb);
    for (auto &c : cts)
        rev.mod_switch_to_next_inplace(c);
    CHECK(same_meta(cb, cts[0]));
    CHECK(cts[0].correction_factor() != 1);
    const std::vector<uint64_t> m = mat();
    seal_b200::PlaintextBatch pshared;
    denc.encode(std::vector<std::vector<uint64_t>>{ m }, pshared);
    Plaintext rshared;
    renc.encode(m, rshared);
    ev.add_plain_inplace(cb, pshared);
    for (auto &c : cts)
        rev.add_plain_inplace(c, rshared);
    CHECK(same_meta(cb, cts[0]));
    std::vector<std::vector<uint64_t>> ms(B);
    std::vector<Plaintext> rp(B);
    for (size_t i = 0; i < B; i++)
    {
        ms[i] = mat();
        renc.encode(ms[i], rp[i]);
    }
    seal_b200::PlaintextBatch pb;
    denc.encode(ms, pb);
    ev.sub_plain_inplace(cb, pb);
    for (size_t i = 0; i < B; i++)
        rev.sub_plain_inplace(cts[i], rp[i]);
    CHECK(same_meta(cb, cts[0]));
    ev.multiply_plain_inplace(cb, pshared); // coefficient-form plaintext, NTT-form ciphertexts
    for (auto &c : cts)
        rev.multiply_plain_inplace(c, rshared);
    CHECK(same_meta(cb, cts[0]));
    same_batch(ev, cb, cts, "BGV chain");
}

int main()
{
    ckks_chain();
    bfv_chain();
    bgv_chain();
    std::printf("%d checks, %d failures\n", g_checks, g_fail);
    if (g_fail)
        return 1;
    std::printf("shim_plain_test ok\n");
    return 0;
}
