// tests/cpp/shim_scalar_test.cpp -- the scalar overloads of seal_b200::CKKSEncoder (include/seal_b200/ckks.hpp) against
// seal::CKKSEncoder: the six Plaintext overloads called as the reference's examples call them (words, parms_id, scale, exception
// types and messages, the destination left alone on error), the PlaintextBatch overloads member by member, and the reference's
// example 5 (5_ckks_basics.cpp: PI*x^3 + 0.4*x + 1) in full on device-resident batches, every intermediate ciphertext word for word
// and the decoded doubles bit for bit.  Built by oracle/scalar.mk into oracle/_ref/bin/shim_scalar_test; run by
// tests/test_gpu_ckks_scalar.py.
#include "seal/seal.h"
#include "seal_b200/ckks.hpp"
#include "seal_b200/decryptor.hpp"
#include "seal_b200/encryptor.hpp"
#include "seal_b200/evaluator.hpp"
#include <cmath>
#include <complex>
#include <cstdio>
#include <cstring>
#include <functional>
#include <limits>
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

static bool same_plain(const Plaintext &a, const Plaintext &b)
{
    const double s1 = a.scale(), s2 = b.scale();
    return a.coeff_count() == b.coeff_count() && a.parms_id() == b.parms_id() && std::memcmp(&s1, &s2, sizeof(double)) == 0 &&
           std::memcmp(a.data(), b.data(), a.coeff_count() * sizeof(uint64_t)) == 0;
}

static bool same_ct(const Ciphertext &a, const Ciphertext &b)
{
    const double s1 = a.scale(), s2 = b.scale();
    return a.parms_id() == b.parms_id() && a.size() == b.size() && a.is_ntt_form() == b.is_ntt_form() &&
           a.correction_factor() == b.correction_factor() && std::memcmp(&s1, &s2, sizeof(double)) == 0 &&
           a.dyn_array().size() == b.dyn_array().size() && std::memcmp(a.data(), b.data(), a.dyn_array().size() * sizeof(uint64_t)) == 0;
}

static EncryptionParameters params(std::size_t n, const std::vector<int> &bits, std::uint64_t seed0)
{
    EncryptionParameters parms(scheme_type::ckks);
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::Create(n, bits));
    prng_seed_type s{};
    s[0] = seed0;
    parms.set_random_generator(std::make_shared<Blake2xbPRNGFactory>(s));
    return parms;
}

// every member of a device batch against the reference's ciphertexts
static bool batch_matches(const seal_b200::Evaluator &ev, const seal_b200::CiphertextBatch &batch, const std::vector<Ciphertext> &ref)
{
    std::vector<Ciphertext> got;
    ev.download(batch, got);
    if (got.size() != ref.size())
        return false;
    for (std::size_t b = 0; b < ref.size(); b++)
        if (!same_ct(got[b], ref[b]))
            return false;
    return true;
}

static bool plain_batch_matches(const seal_b200::Evaluator &ev, const seal_b200::PlaintextBatch &batch, const std::vector<Plaintext> &ref)
{
    std::vector<Plaintext> got;
    ev.download(batch, got);
    if (got.size() != ref.size())
        return false;
    for (std::size_t b = 0; b < ref.size(); b++)
        if (!same_plain(got[b], ref[b]))
            return false;
    return true;
}

// the six overloads and their errors, at the first level and below it
static void overloads()
{
    const std::size_t n = 8192;
    SEALContext ctx(params(n, { 60, 40, 40, 60 }, 1), true, sec_level_type::none);
    seal_b200::Evaluator ev(ctx);
    seal_b200::CKKSEncoder ours(ctx, ev);
    seal::CKKSEncoder ref(ctx);
    const double scale = std::pow(2.0, 40);
    const parms_id_type first = ctx.first_parms_id(), last = ctx.last_parms_id();

    // as example 5 calls them (5_ckks_basics.cpp:124-126), and example 7 (7_serialization.cpp:287-288)
    for (double v : { 3.14159265, 0.4, 1.0, 2.3, 4.5, -0.49, 0.5, -2.5, 0.0, -0.0, 1e9, -123456.789 })
    {
        Plaintext a, b;
        ours.encode(v, scale, a);
        ref.encode(v, scale, b);
        CHECK(same_plain(a, b));
        ours.encode(v, last, std::pow(2.0, 20), a);
        ref.encode(v, last, std::pow(2.0, 20), b);
        CHECK(same_plain(a, b));
    }
    for (std::complex<double> v : { std::complex<double>(1.5, -0.25), std::complex<double>(-3.0, 0.0), std::complex<double>(0.0, 7.0) })
    {
        Plaintext a, b;
        ours.encode(v, scale, a);
        ref.encode(v, scale, b);
        CHECK(same_plain(a, b));
        ours.encode(v, last, std::pow(2.0, 20), a);
        ref.encode(v, last, std::pow(2.0, 20), b);
        CHECK(same_plain(a, b));
    }
    // 8_performance.cpp:479-482: encode(i + 1, plain) with a size_t argument selects the int64 overload
    for (std::size_t i = 0; i < 5; i++)
    {
        Plaintext a, b;
        ours.encode(i + 1, a);
        ref.encode(i + 1, b);
        CHECK(same_plain(a, b));
        CHECK(a.scale() == 1.0);
    }
    for (std::int64_t v : { std::int64_t(0), std::int64_t(-1), std::int64_t(-(std::int64_t(1) << 40)), std::int64_t(1) << 50,
                            std::int64_t(-123456789) })
    {
        Plaintext a, b;
        ours.encode(v, a);
        ref.encode(v, b);
        CHECK(same_plain(a, b));
        ours.encode(v, last, a);
        ref.encode(v, last, b);
        CHECK(same_plain(a, b));
    }

    // errors: same exception type and message, and the destination left as it was
    Plaintext keep_ours, keep_ref;
    ours.encode(1.25, scale, keep_ours);
    ref.encode(1.25, scale, keep_ref);
    const Plaintext before = keep_ours;
    const double inf = std::numeric_limits<double>::infinity(), nan = std::numeric_limits<double>::quiet_NaN();
    same_throw([&] { ours.encode(1.0, parms_id_zero, scale, keep_ours); }, [&] { ref.encode(1.0, parms_id_zero, scale, keep_ref); }, "real, parms_id");
    same_throw([&] { ours.encode(std::complex<double>(1, 1), parms_id_zero, scale, keep_ours); },
               [&] { ref.encode(std::complex<double>(1, 1), parms_id_zero, scale, keep_ref); }, "complex, parms_id");
    same_throw([&] { ours.encode(std::int64_t(1), parms_id_zero, keep_ours); }, [&] { ref.encode(std::int64_t(1), parms_id_zero, keep_ref); },
               "int64, parms_id");
    same_throw([&] { ours.encode(1.0, scale, keep_ours, MemoryPoolHandle()); }, [&] { ref.encode(1.0, scale, keep_ref, MemoryPoolHandle()); },
               "real, pool");
    same_throw([&] { ours.encode(std::complex<double>(1, 1), scale, keep_ours, MemoryPoolHandle()); },
               [&] { ref.encode(std::complex<double>(1, 1), scale, keep_ref, MemoryPoolHandle()); }, "complex, pool");
    for (double s : { 0.0, -1.0, inf, nan, std::pow(2.0, 200) })
        same_throw([&] { ours.encode(1.0, s, keep_ours); }, [&] { ref.encode(1.0, s, keep_ref); }, "real, scale");
    for (double v : { inf, -inf, nan })
        same_throw([&] { ours.encode(v, scale, keep_ours); }, [&] { ref.encode(v, scale, keep_ref); }, "real, value");
    same_throw([&] { ours.encode(1e300, scale, keep_ours); }, [&] { ref.encode(1e300, scale, keep_ref); }, "real, product overflows");
    same_throw([&] { ours.encode(1e30, scale, keep_ours); }, [&] { ref.encode(1e30, scale, keep_ref); }, "real, too large");
    same_throw([&] { ours.encode(std::complex<double>(inf, 0), scale, keep_ours); }, [&] { ref.encode(std::complex<double>(inf, 0), scale, keep_ref); },
               "complex, value");
    same_throw([&] { ours.encode(std::complex<double>(1e30, 0), scale, keep_ours); },
               [&] { ref.encode(std::complex<double>(1e30, 0), scale, keep_ref); }, "complex, too large");
    same_throw([&] { ours.encode(std::complex<double>(1, 0), 5e-324, keep_ours); }, [&] { ref.encode(std::complex<double>(1, 0), 5e-324, keep_ref); },
               "complex, subnormal scale");
    same_throw([&] { ours.encode(std::numeric_limits<std::int64_t>::max(), last, keep_ours); },
               [&] { ref.encode(std::numeric_limits<std::int64_t>::max(), last, keep_ref); }, "int64, too large");
    CHECK(same_plain(keep_ours, before));
    CHECK(same_plain(keep_ours, keep_ref));
    // accepted by encode(double) only: a subnormal scale
    {
        Plaintext a, b;
        ours.encode(1.0, 5e-324, a);
        ref.encode(1.0, 5e-324, b);
        CHECK(same_plain(a, b));
    }

    // PlaintextBatch overloads: a batch of one, and one member per value
    {
        seal_b200::PlaintextBatch P;
        Plaintext r;
        ours.encode(3.14159265, first, scale, P);
        ref.encode(3.14159265, first, scale, r);
        CHECK(P.batch_size() == 1 && P.parms_id() == first && P.scale() == scale && P.is_ntt_form());
        CHECK(plain_batch_matches(ev, P, { r }));
        ours.encode(std::complex<double>(0.5, -2.0), last, scale, P);
        ref.encode(std::complex<double>(0.5, -2.0), last, scale, r);
        CHECK(plain_batch_matches(ev, P, { r }));
        ours.encode(std::int64_t(-7), first, P);
        ref.encode(std::int64_t(-7), first, r);
        CHECK(P.scale() == 1.0 && plain_batch_matches(ev, P, { r }));

        const std::vector<double> dv{ 0.4, -1.5, 2.5, 1e6 };
        const std::vector<std::complex<double>> cv{ { 1, 2 }, { -0.5, 0 }, { 0, -3 } };
        const std::vector<std::int64_t> iv{ 1, -1, 1ll << 45, -(1ll << 45), 0 };
        std::vector<Plaintext> rs;
        ours.encode_scalars(dv, first, scale, P);
        rs.assign(dv.size(), Plaintext());
        for (std::size_t b = 0; b < dv.size(); b++)
            ref.encode(dv[b], first, scale, rs[b]);
        CHECK(P.batch_size() == dv.size() && plain_batch_matches(ev, P, rs));
        ours.encode_scalars(cv, last, scale, P);
        rs.assign(cv.size(), Plaintext());
        for (std::size_t b = 0; b < cv.size(); b++)
            ref.encode(cv[b], last, scale, rs[b]);
        CHECK(P.batch_size() == cv.size() && plain_batch_matches(ev, P, rs));
        ours.encode_scalars(iv, first, P);
        rs.assign(iv.size(), Plaintext());
        for (std::size_t b = 0; b < iv.size(); b++)
            ref.encode(iv[b], first, rs[b]);
        CHECK(P.batch_size() == iv.size() && plain_batch_matches(ev, P, rs));

        // errors: the reference's message for the first failing member
        const std::vector<double> bad{ 1.0, inf, 1e300 };
        Plaintext r0;
        same_throw([&] { ours.encode_scalars(bad, first, scale, P); }, [&] {
            for (double v : bad)
                ref.encode(v, first, scale, r0);
        }, "encode_scalars, first failing member");
        same_throw([&] { ours.encode(1.0, parms_id_zero, scale, P); }, [&] { ref.encode(1.0, parms_id_zero, scale, r0); }, "batch, parms_id");
    }
}

// 5_ckks_basics.cpp on four input vectors at once: every step on device-resident batches against the reference, one ciphertext per
// input, under identically seeded Blake2xb factories
static void example5()
{
    const std::size_t n = 8192, B = 4;
    SEALContext ours_ctx(params(n, { 60, 40, 40, 60 }, 0x5EED), true, sec_level_type::none);
    SEALContext ref_ctx(params(n, { 60, 40, 40, 60 }, 0x5EED), true, sec_level_type::none);
    SEALContext key_ctx(params(n, { 60, 40, 40, 60 }, 0xC0DE), true, sec_level_type::none);
    KeyGenerator keygen(key_ctx);
    const SecretKey &sk = keygen.secret_key();
    PublicKey pk;
    keygen.create_public_key(pk);
    RelinKeys rk;
    keygen.create_relin_keys(rk);

    seal_b200::Evaluator ev(ours_ctx);
    seal_b200::Encryptor enc(ours_ctx, pk, ev);
    seal_b200::Decryptor dec(ours_ctx, sk, ev);
    seal_b200::CKKSEncoder encoder(ours_ctx, ev);
    seal::Encryptor renc(ref_ctx, pk);
    seal::Decryptor rdec(ref_ctx, sk);
    seal::Evaluator rev(ref_ctx);
    seal::CKKSEncoder rencoder(ref_ctx);
    const double scale = std::pow(2.0, 40);
    const std::size_t slots = encoder.slot_count();

    // four inputs: the example's ramp over [0, 1] and three variations of it
    std::vector<std::vector<double>> input(B);
    for (std::size_t b = 0; b < B; b++)
    {
        double curr_point = 0;
        const double step_size = 1.0 / (static_cast<double>(slots) - 1);
        for (std::size_t i = 0; i < slots; i++)
        {
            input[b].push_back(b == 0 ? curr_point : b == 1 ? 1.0 - curr_point : b == 2 ? -curr_point : std::sin(7.0 * curr_point));
            curr_point += step_size;
        }
    }

    seal_b200::PlaintextBatch plain_coeff3, plain_coeff1, plain_coeff0;
    encoder.encode(3.14159265, ours_ctx.first_parms_id(), scale, plain_coeff3);
    encoder.encode(0.4, ours_ctx.first_parms_id(), scale, plain_coeff1);
    encoder.encode(1.0, ours_ctx.first_parms_id(), scale, plain_coeff0);
    Plaintext r_coeff3, r_coeff1, r_coeff0;
    rencoder.encode(3.14159265, scale, r_coeff3);
    rencoder.encode(0.4, scale, r_coeff1);
    rencoder.encode(1.0, scale, r_coeff0);
    CHECK(plain_batch_matches(ev, plain_coeff3, { r_coeff3 }));
    CHECK(plain_batch_matches(ev, plain_coeff1, { r_coeff1 }));
    CHECK(plain_batch_matches(ev, plain_coeff0, { r_coeff0 }));

    seal_b200::PlaintextBatch x_plain;
    encoder.encode(input, ours_ctx.first_parms_id(), scale, x_plain);
    seal_b200::CiphertextBatch x1_encrypted;
    enc.encrypt(x_plain, x1_encrypted);
    std::vector<Plaintext> rx_plain(B);
    std::vector<Ciphertext> rx1(B);
    for (std::size_t b = 0; b < B; b++)
    {
        rencoder.encode(input[b], scale, rx_plain[b]);
        renc.encrypt(rx_plain[b], rx1[b]);
    }
    CHECK(plain_batch_matches(ev, x_plain, rx_plain));
    CHECK(batch_matches(ev, x1_encrypted, rx1));

    // x^2, relinearized and rescaled (the batch is copied through the host: a CiphertextBatch has no copy)
    std::vector<Ciphertext> host;
    ev.download(x1_encrypted, host);
    seal_b200::CiphertextBatch x3_encrypted;
    ev.upload(host, x3_encrypted);
    ev.square_inplace(x3_encrypted);
    std::vector<Ciphertext> rx3(B);
    for (std::size_t b = 0; b < B; b++)
        rev.square(rx1[b], rx3[b]);
    CHECK(batch_matches(ev, x3_encrypted, rx3));
    ev.relinearize_inplace(x3_encrypted, rk);
    for (auto &c : rx3)
        rev.relinearize_inplace(c, rk);
    CHECK(batch_matches(ev, x3_encrypted, rx3));
    ev.rescale_to_next_inplace(x3_encrypted);
    for (auto &c : rx3)
        rev.rescale_to_next_inplace(c);
    CHECK(batch_matches(ev, x3_encrypted, rx3));

    // PI*x, rescaled
    seal_b200::CiphertextBatch x1_encrypted_coeff3;
    ev.upload(host, x1_encrypted_coeff3);
    ev.multiply_plain_inplace(x1_encrypted_coeff3, plain_coeff3);
    std::vector<Ciphertext> rx1c3(B);
    for (std::size_t b = 0; b < B; b++)
        rev.multiply_plain(rx1[b], r_coeff3, rx1c3[b]);
    CHECK(batch_matches(ev, x1_encrypted_coeff3, rx1c3));
    ev.rescale_to_next_inplace(x1_encrypted_coeff3);
    for (auto &c : rx1c3)
        rev.rescale_to_next_inplace(c);
    CHECK(batch_matches(ev, x1_encrypted_coeff3, rx1c3));

    // PI*x^3, relinearized and rescaled
    ev.multiply_inplace(x3_encrypted, x1_encrypted_coeff3);
    for (std::size_t b = 0; b < B; b++)
        rev.multiply_inplace(rx3[b], rx1c3[b]);
    CHECK(batch_matches(ev, x3_encrypted, rx3));
    ev.relinearize_inplace(x3_encrypted, rk);
    for (auto &c : rx3)
        rev.relinearize_inplace(c, rk);
    ev.rescale_to_next_inplace(x3_encrypted);
    for (auto &c : rx3)
        rev.rescale_to_next_inplace(c);
    CHECK(batch_matches(ev, x3_encrypted, rx3));

    // 0.4*x, rescaled
    ev.multiply_plain_inplace(x1_encrypted, plain_coeff1);
    for (auto &c : rx1)
        rev.multiply_plain_inplace(c, r_coeff1);
    CHECK(batch_matches(ev, x1_encrypted, rx1));
    ev.rescale_to_next_inplace(x1_encrypted);
    for (auto &c : rx1)
        rev.rescale_to_next_inplace(c);
    CHECK(batch_matches(ev, x1_encrypted, rx1));

    // the scales set to 2^40, the levels aligned by mod_switch_to, then the sum
    x3_encrypted.scale() = std::pow(2.0, 40);
    x1_encrypted.scale() = std::pow(2.0, 40);
    for (std::size_t b = 0; b < B; b++)
        rx3[b].scale() = std::pow(2.0, 40), rx1[b].scale() = std::pow(2.0, 40);
    const parms_id_type last_parms_id = x3_encrypted.parms_id();
    CHECK(last_parms_id == rx3[0].parms_id());
    ev.mod_switch_to_inplace(x1_encrypted, last_parms_id);
    ev.mod_switch_to_inplace(plain_coeff0, last_parms_id);
    for (auto &c : rx1)
        rev.mod_switch_to_inplace(c, last_parms_id);
    rev.mod_switch_to_inplace(r_coeff0, last_parms_id);
    CHECK(batch_matches(ev, x1_encrypted, rx1));
    CHECK(plain_batch_matches(ev, plain_coeff0, { r_coeff0 }));

    ev.add_inplace(x3_encrypted, x1_encrypted); // evaluator.add(x3_encrypted, x1_encrypted, encrypted_result)
    ev.add_plain_inplace(x3_encrypted, plain_coeff0);
    std::vector<Ciphertext> rresult(B);
    for (std::size_t b = 0; b < B; b++)
    {
        rev.add(rx3[b], rx1[b], rresult[b]);
        rev.add_plain_inplace(rresult[b], r_coeff0);
    }
    CHECK(batch_matches(ev, x3_encrypted, rresult));

    // decrypt and decode: the doubles bit for bit, and close to the true result
    seal_b200::PlaintextBatch plain_result;
    dec.decrypt(x3_encrypted, plain_result);
    std::vector<std::vector<double>> result;
    encoder.decode(plain_result, result);
    CHECK(result.size() == B);
    double worst = 0;
    for (std::size_t b = 0; b < B && b < result.size(); b++)
    {
        Plaintext rp;
        rdec.decrypt(rresult[b], rp);
        std::vector<double> rr;
        rencoder.decode(rp, rr);
        CHECK(rr.size() == result[b].size() && std::memcmp(rr.data(), result[b].data(), rr.size() * sizeof(double)) == 0);
        for (std::size_t i = 0; i < slots && i < result[b].size(); i++)
        {
            const double x = input[b][i];
            worst = std::max(worst, std::fabs(result[b][i] - ((3.14159265 * x * x + 0.4) * x + 1)));
        }
    }
    CHECK(worst < 1e-3);
    std::printf("example 5 on %zu inputs: largest error against the true result %.3g\n", B, worst);
}

int main()
{
    overloads();
    example5();
    std::printf("%d checks, %d failed\n", g_checks, g_fail);
    if (g_fail)
        return 1;
    std::printf("PASS\n");
    return 0;
}
