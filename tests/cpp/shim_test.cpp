// tests/cpp/shim_test.cpp -- drop-in check of include/seal_b200/evaluator.hpp against the reference's own
// seal::Evaluator (linked from oracle/_ref/libseal.so): same inputs -> identical ciphertext words and metadata, same
// exception types; plus the reference's style of semantic tests (encrypt -> evaluate on GPU -> decrypt), cf.
// native/tests/seal/evaluator.cpp:1356 (BFVEncryptMultiplyDecrypt), :3513 (CKKSEncryptMultiplyRelinRescaleDecrypt),
// :4326 (CKKSEncryptRotateDecrypt), :5670 (BFVEncryptRotateMatrixDecrypt), :2505/:2532 (negative relinearize tests).
// TEST INFRASTRUCTURE: links the reference; oracle/Makefile builds it into oracle/_ref/bin/ where the reference sources are.
#include "seal_b200/batchencoder.hpp"
#include "seal_b200/ckks.hpp"
#include "seal_b200/encryptor.hpp"
#include "seal_b200/decryptor.hpp"
#include "seal_b200/evaluator.hpp"
#include <complex>
#include <cstdio>
#include <cstring>
#include <functional>
#include <memory>
#include <random>
#include <typeinfo>

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

static bool same_ct(const Ciphertext &a, const Ciphertext &b)
{
    if (a.parms_id() != b.parms_id() || a.size() != b.size() || a.is_ntt_form() != b.is_ntt_form() ||
        a.coeff_modulus_size() != b.coeff_modulus_size())
        return false;
    double sa = a.scale(), sb = b.scale();
    if (std::memcmp(&sa, &sb, sizeof(double)) != 0 || a.correction_factor() != b.correction_factor())
        return false;
    return std::memcmp(a.data(), b.data(), a.size() * a.coeff_modulus_size() * a.poly_modulus_degree() * 8) == 0;
}

static bool same_plain(const Plaintext &a, const Plaintext &b)
{
    double sa = a.scale(), sb = b.scale();
    return a.parms_id() == b.parms_id() && a.coeff_count() == b.coeff_count() && std::memcmp(&sa, &sb, sizeof(double)) == 0 &&
           std::memcmp(a.data(), b.data(), a.coeff_count() * 8) == 0;
}

// runs f on both evaluators; returns a tag describing the exception type (or "ok")
template <class F>
static std::string outcome(F f)
{
    try
    {
        f();
        return "ok";
    }
    catch (const std::invalid_argument &)
    {
        return "invalid_argument";
    }
    catch (const std::out_of_range &)
    {
        return "out_of_range";
    }
    catch (const std::logic_error &)
    {
        return "logic_error";
    }
    catch (const std::exception &)
    {
        return "exception";
    }
}

static void test_ckks()
{
    EncryptionParameters parms(scheme_type::ckks);
    const size_t n = 8192;
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::Create(n, { 54, 40, 40, 54 }));
    SEALContext context(parms, true, sec_level_type::none);
    KeyGenerator keygen(context);
    PublicKey pk;
    keygen.create_public_key(pk);
    RelinKeys rlk;
    keygen.create_relin_keys(rlk);
    GaloisKeys glk;
    keygen.create_galois_keys(glk); // power-of-two steps only -> step 5 goes through the NAF fallback
    Encryptor encryptor(context, pk);
    Decryptor decryptor(context, keygen.secret_key());
    CKKSEncoder encoder(context);
    seal::Evaluator ref(context);
    seal_b200::Evaluator gpu(context);

    const size_t slots = n / 2;
    std::mt19937_64 rng(0x5EA1);
    std::vector<double> x(slots), y(slots);
    for (size_t i = 0; i < slots; i++)
        x[i] = double(rng() % 2000) / 100.0 - 10.0, y[i] = double(rng() % 2000) / 100.0 - 10.0;
    const double scale = std::pow(2.0, 40);
    Plaintext px, py;
    encoder.encode(x, scale, px);
    encoder.encode(y, scale, py);
    Ciphertext cx, cy;
    encryptor.encrypt(px, cx);
    encryptor.encrypt(py, cy);

    Ciphertext r1, g1;
    ref.multiply(cx, cy, r1);
    gpu.multiply(cx, cy, g1);
    CHECK(same_ct(r1, g1));
    ref.relinearize_inplace(r1, rlk);
    gpu.relinearize_inplace(g1, rlk);
    CHECK(same_ct(r1, g1));
    ref.rescale_to_next_inplace(r1);
    gpu.rescale_to_next_inplace(g1);
    CHECK(same_ct(r1, g1));
    {
        Plaintext p;
        decryptor.decrypt(g1, p);
        std::vector<double> got;
        encoder.decode(p, got);
        double err = 0;
        for (size_t i = 0; i < slots; i++)
            err = std::max(err, std::abs(got[i] - x[i] * y[i]));
        CHECK(err < 1e-3);
    }
    {
        // Decryptor::decrypt on the device (CKKS: the NTT-form phase is the plaintext), sizes 2 and 3
        seal_b200::Decryptor gdec(context, keygen.secret_key(), gpu);
        Plaintext rp, gp;
        decryptor.decrypt(g1, rp);
        gdec.decrypt(g1, gp);
        CHECK(same_plain(rp, gp));
        Ciphertext c3;
        ref.multiply(cx, cy, c3);
        decryptor.decrypt(c3, rp);
        gdec.decrypt(c3, gp);
        CHECK(same_plain(rp, gp));
    }
    {
        // SURVEY 8(f) rank 1: square / add / sub / negate
        Ciphertext r2, g2, r3, g3;
        ref.square(cx, r2);
        gpu.square(cx, g2);
        CHECK(same_ct(r2, g2));
        ref.add(cx, cy, r3);
        gpu.add(cx, cy, g3);
        CHECK(same_ct(r3, g3));
        ref.sub_inplace(r3, cx);
        gpu.sub_inplace(g3, cx);
        CHECK(same_ct(r3, g3));
        ref.negate_inplace(r3);
        gpu.negate_inplace(g3);
        CHECK(same_ct(r3, g3));
        // operands of different sizes: the longer tail is copied (add) or negated (sub), evaluator.cpp:228-233, :336-341
        Ciphertext c3, r4, g4;
        ref.multiply(cx, cy, c3);
        c3.scale() = cx.scale();
        ref.add(cx, c3, r4);
        gpu.add(cx, c3, g4);
        CHECK(r4.size() == 3 && same_ct(r4, g4));
        ref.sub(cx, c3, r4);
        gpu.sub(cx, c3, g4);
        CHECK(same_ct(r4, g4));
        ref.sub(c3, cx, r4);
        gpu.sub(c3, cx, g4);
        CHECK(same_ct(r4, g4));
        auto a = outcome([&] { Ciphertext t = cx; t.scale() *= 2; ref.add_inplace(t, cy); });
        auto b = outcome([&] { Ciphertext t = cx; t.scale() *= 2; gpu.add_inplace(t, cy); });
        CHECK(a == b && a == "invalid_argument"); // scale mismatch
    }
    {
        // SURVEY 8(f) rank 1: multiply_plain, NTT path (CKKS plaintexts are always in NTT form)
        Ciphertext r2, g2;
        ref.multiply_plain(cx, py, r2);
        gpu.multiply_plain(cx, py, g2);
        CHECK(same_ct(r2, g2));
        ref.multiply(cx, cy, r2);
        g2 = r2; // size 3
        Plaintext pz;
        encoder.encode(y, r2.parms_id(), std::pow(2.0, 20), pz);
        ref.multiply_plain_inplace(r2, pz);
        gpu.multiply_plain_inplace(g2, pz);
        CHECK(same_ct(r2, g2));
        Plaintext low;
        encoder.encode(y, r1.parms_id(), scale, low); // one level down: parameter mismatch with cx
        auto a = outcome([&] { Ciphertext t = cx; ref.multiply_plain_inplace(t, low); });
        auto b = outcome([&] { Ciphertext t = cx; gpu.multiply_plain_inplace(t, low); });
        CHECK(a == b && a == "invalid_argument");
        Plaintext big;
        encoder.encode(y, std::pow(2.0, 120), big);
        a = outcome([&] { Ciphertext t = cx; ref.multiply_plain_inplace(t, big); });
        b = outcome([&] { Ciphertext t = cx; gpu.multiply_plain_inplace(t, big); });
        CHECK(a == b && a == "invalid_argument"); // scale out of bounds
    }
    {
        // general-size multiply (evaluator.cpp:664-700): size 3 x size 2 -> 4, and a size-3 square
        Ciphertext r2, g2, c3;
        ref.multiply(cx, cy, c3);
        Ciphertext lo = cx;
        lo.scale() = 4.0; // keep the product scale inside the level's bounds
        c3.scale() = 4.0;
        ref.multiply(c3, lo, r2);
        gpu.multiply(c3, lo, g2);
        CHECK(r2.size() == 4 && same_ct(r2, g2));
        ref.square(c3, r2);
        gpu.square(c3, g2);
        CHECK(r2.size() == 5 && same_ct(r2, g2));
    }
    {
        // add_plain / sub_plain (CKKS), add_many, mod_switch_to / rescale_to
        Ciphertext r2, g2;
        ref.add_plain(cx, py, r2);
        gpu.add_plain(cx, py, g2);
        CHECK(same_ct(r2, g2));
        ref.sub_plain_inplace(r2, px);
        gpu.sub_plain_inplace(g2, px);
        CHECK(same_ct(r2, g2));
        std::vector<Ciphertext> many{ cx, cy, r2 };
        ref.add_many(many, r2);
        gpu.add_many(many, g2);
        CHECK(same_ct(r2, g2));
        {
            // layout-only level changes: mod_reduce_to_next (ciphertext), mod_switch_to_next / mod_switch_to (NTT-form plaintext)
            Ciphertext c3, r5, g5;
            ref.multiply(cx, cy, c3); // size 3
            ref.mod_reduce_to_next(c3, r5);
            gpu.mod_reduce_to_next(c3, g5);
            CHECK(same_ct(r5, g5));
            ref.mod_reduce_to(cx, context.last_parms_id(), r5);
            gpu.mod_reduce_to(cx, context.last_parms_id(), g5);
            CHECK(same_ct(r5, g5));
            Plaintext rp, gp;
            ref.mod_switch_to_next(px, rp);
            gpu.mod_switch_to_next(px, gp);
            CHECK(rp.parms_id() == gp.parms_id() && rp.coeff_count() == gp.coeff_count() && rp.scale() == gp.scale() &&
                  std::memcmp(rp.data(), gp.data(), rp.coeff_count() * 8) == 0);
            ref.mod_switch_to(px, context.last_parms_id(), rp);
            gpu.mod_switch_to(px, context.last_parms_id(), gp);
            CHECK(rp.parms_id() == gp.parms_id() && rp.coeff_count() == gp.coeff_count() &&
                  std::memcmp(rp.data(), gp.data(), rp.coeff_count() * 8) == 0);
            auto a = outcome([&] { Plaintext t = rp; ref.mod_switch_to_next_inplace(t); });
            auto b = outcome([&] { Plaintext t = gp; gpu.mod_switch_to_next_inplace(t); });
            CHECK(a == b && a == "invalid_argument"); // end of modulus switching chain reached
        }
        auto last = context.last_parms_id();
        ref.mod_switch_to(cx, last, r2);
        gpu.mod_switch_to(cx, last, g2);
        CHECK(same_ct(r2, g2));
        Ciphertext hi = cx;
        hi.scale() = std::pow(2.0, 100);
        ref.rescale_to(hi, last, r2);
        gpu.rescale_to(hi, last, g2);
        CHECK(same_ct(r2, g2));
        auto a = outcome([&] { Ciphertext t = r2; ref.mod_switch_to_inplace(t, cx.parms_id()); });
        auto b = outcome([&] { Ciphertext t = g2; gpu.mod_switch_to_inplace(t, cx.parms_id()); });
        CHECK(a == b && a == "invalid_argument"); // cannot switch to higher level modulus
        a = outcome([&] { Ciphertext t; ref.multiply_many(many, rlk, t); });
        b = outcome([&] { Ciphertext t; gpu.multiply_many(many, rlk, t); });
        CHECK(a == b && a == "logic_error"); // BFV / BGV only
    }
    for (int step : { 1, -4, 5, 1023 })
    {
        Ciphertext r2, g2;
        ref.rotate_vector(r1, step, glk, r2);
        gpu.rotate_vector(g1, step, glk, g2);
        CHECK(same_ct(r2, g2));
    }
    {
        Ciphertext r2, g2;
        ref.complex_conjugate(cx, glk, r2);
        gpu.complex_conjugate(cx, glk, g2);
        CHECK(same_ct(r2, g2));
        ref.mod_switch_to_next_inplace(r2);
        gpu.mod_switch_to_next_inplace(g2);
        CHECK(same_ct(r2, g2));
        ref.transform_from_ntt_inplace(r2);
        gpu.transform_from_ntt_inplace(g2);
        CHECK(same_ct(r2, g2));
        ref.transform_to_ntt_inplace(r2);
        gpu.transform_to_ntt_inplace(g2);
        CHECK(same_ct(r2, g2));
    }
    // batch extension == singles
    {
        std::vector<Ciphertext> a(3, cx), b(3, cy), out;
        ref.square_inplace(a[1]);
        ref.relinearize_inplace(a[1], rlk); // a different (size-2) operand; scale 2^80 is still in bounds at level 3? use cx*cx rescaled
        ref.rescale_to_next_inplace(a[1]);
        // bring everything to the same level
        for (auto *v : { &a[0], &a[2], &b[0], &b[1], &b[2] })
            ref.mod_switch_to_next_inplace(*v);
        gpu.multiply_relinearize(a, b, rlk, out);
        for (size_t i = 0; i < 3; i++)
        {
            Ciphertext r;
            ref.multiply(a[i], b[i], r);
            ref.relinearize_inplace(r, rlk);
            CHECK(same_ct(r, out[i]));
        }
    }
    // negative tests: identical exception types
    {
        Ciphertext bad = cx;
        bad.is_ntt_form() = false; // CKKS operand not in NTT form -> evaluator.cpp:571-574
        auto a = outcome([&] { Ciphertext t; ref.multiply(bad, cy, t); });
        auto b = outcome([&] { Ciphertext t; gpu.multiply(bad, cy, t); });
        CHECK(a == b && a == "invalid_argument");
        Ciphertext last = cx;
        while (last.parms_id() != context.last_parms_id())
            ref.mod_switch_to_next_inplace(last);
        a = outcome([&] { Ciphertext t = last; ref.rescale_to_next_inplace(t); });
        b = outcome([&] { Ciphertext t = last; gpu.rescale_to_next_inplace(t); });
        CHECK(a == b && a == "invalid_argument");
        GaloisKeys few;
        keygen.create_galois_keys(std::vector<int>{ 1 }, few);
        a = outcome([&] { Ciphertext t = cx; ref.rotate_vector_inplace(t, 2, few); });
        b = outcome([&] { Ciphertext t = cx; gpu.rotate_vector_inplace(t, 2, few); });
        CHECK(a == b && a == "invalid_argument"); // "Galois key not present"
        a = outcome([&] { Ciphertext t = cx; ref.rotate_rows_inplace(t, 1, glk); });
        b = outcome([&] { Ciphertext t = cx; gpu.rotate_rows_inplace(t, 1, glk); });
        CHECK(a == b && a == "logic_error"); // wrong scheme
        // key set from another context (parms mismatch) -> relinearize_internal :1153-1156
        EncryptionParameters p2(scheme_type::ckks);
        p2.set_poly_modulus_degree(n);
        p2.set_coeff_modulus(CoeffModulus::Create(n, { 50, 50, 50 }));
        SEALContext c2(p2, true, sec_level_type::none);
        KeyGenerator kg2(c2);
        RelinKeys rlk2;
        kg2.create_relin_keys(rlk2);
        Ciphertext m3;
        ref.multiply(cx, cy, m3);
        a = outcome([&] { Ciphertext t = m3; ref.relinearize_inplace(t, rlk2); });
        b = outcome([&] { Ciphertext t = m3; gpu.relinearize_inplace(t, rlk2); });
        CHECK(a == b && a == "invalid_argument");
    }
}

static void test_bfv()
{
    EncryptionParameters parms(scheme_type::bfv);
    const size_t n = 4096; // BASELINE.json configs[0]: BFV n=4096, 3x36-bit coeff_modulus
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::BFVDefault(n));
    parms.set_plain_modulus(PlainModulus::Batching(n, 20));
    SEALContext context(parms, true, sec_level_type::none);
    KeyGenerator keygen(context);
    RelinKeys rlk;
    keygen.create_relin_keys(rlk);
    GaloisKeys glk;
    keygen.create_galois_keys(glk);
    Encryptor encryptor(context, keygen.secret_key());
    Decryptor decryptor(context, keygen.secret_key());
    BatchEncoder encoder(context);
    seal::Evaluator ref(context);
    seal_b200::Evaluator gpu(context);
    const uint64_t t = parms.plain_modulus().value();

    std::mt19937_64 rng(7);
    std::vector<uint64_t> x(n), y(n);
    for (size_t i = 0; i < n; i++)
        x[i] = rng() % 500, y[i] = rng() % 500;
    Plaintext px, py;
    encoder.encode(x, px);
    encoder.encode(y, py);
    Ciphertext cx, cy;
    encryptor.encrypt_symmetric(px, cx);
    encryptor.encrypt_symmetric(py, cy);

    Ciphertext r1, g1;
    ref.multiply(cx, cy, r1);
    gpu.multiply(cx, cy, g1);
    CHECK(same_ct(r1, g1));
    ref.relinearize_inplace(r1, rlk);
    gpu.relinearize_inplace(g1, rlk);
    CHECK(same_ct(r1, g1));
    {
        Plaintext p;
        decryptor.decrypt(g1, p);
        std::vector<uint64_t> got;
        encoder.decode(p, got);
        bool ok = true;
        for (size_t i = 0; i < n; i++)
            ok = ok && got[i] == (x[i] * y[i]) % t;
        CHECK(ok);
        CHECK(decryptor.invariant_noise_budget(g1) > 0);
    }
    for (int step : { 1, -2, 7 })
    {
        Ciphertext r2, g2;
        ref.rotate_rows(cx, step, glk, r2);
        gpu.rotate_rows(cx, step, glk, g2);
        CHECK(same_ct(r2, g2));
    }
    {
        Ciphertext r2, g2;
        ref.rotate_columns(cx, glk, r2);
        gpu.rotate_columns(cx, glk, g2);
        CHECK(same_ct(r2, g2));
        Plaintext p;
        decryptor.decrypt(g2, p);
        std::vector<uint64_t> got;
        encoder.decode(p, got);
        bool ok = true;
        for (size_t i = 0; i < n / 2; i++)
            ok = ok && got[i] == x[i + n / 2] && got[i + n / 2] == x[i];
        CHECK(ok);
        ref.mod_switch_to_next_inplace(r2);
        gpu.mod_switch_to_next_inplace(g2);
        CHECK(same_ct(r2, g2));
        ref.transform_to_ntt_inplace(r2);
        gpu.transform_to_ntt_inplace(g2);
        CHECK(same_ct(r2, g2));
    }
    {
        // general-size BFV multiply (:524-560): size 3 x size 2 -> 4; decrypts to x*y*y
        Ciphertext c3, r2, g2;
        ref.multiply(cx, cy, c3);
        ref.multiply(c3, cy, r2);
        gpu.multiply(c3, cy, g2);
        CHECK(r2.size() == 4 && same_ct(r2, g2));
        if (decryptor.invariant_noise_budget(g2) > 0)
        {
            Plaintext p;
            decryptor.decrypt(g2, p);
            std::vector<uint64_t> got;
            encoder.decode(p, got);
            bool ok = true;
            for (size_t i = 0; i < n; i++)
                ok = ok && got[i] == (x[i] * y[i] % t) * y[i] % t;
            CHECK(ok);
        }
    }
    {
        // coefficient-form plaintexts: multiply_plain_normal, add_plain / sub_plain (scaling variant), transform_to_ntt(Plaintext)
        Ciphertext r2, g2;
        ref.multiply_plain(cx, py, r2);
        gpu.multiply_plain(cx, py, g2);
        CHECK(same_ct(r2, g2));
        ref.add_plain_inplace(r2, px);
        gpu.add_plain_inplace(g2, px);
        CHECK(same_ct(r2, g2));
        ref.sub_plain_inplace(r2, py);
        gpu.sub_plain_inplace(g2, py);
        CHECK(same_ct(r2, g2));
        Plaintext p;
        decryptor.decrypt(g2, p);
        std::vector<uint64_t> got;
        encoder.decode(p, got);
        bool ok = true;
        for (size_t i = 0; i < n; i++)
            ok = ok && got[i] == (x[i] * y[i] + x[i] + t - y[i]) % t;
        CHECK(ok);
        Plaintext rp, gp;
        ref.transform_to_ntt(py, cx.parms_id(), rp);
        gpu.transform_to_ntt(py, cx.parms_id(), gp);
        CHECK(rp.parms_id() == gp.parms_id() && rp.coeff_count() == gp.coeff_count() &&
              std::memcmp(rp.data(), gp.data(), rp.coeff_count() * 8) == 0);
        Plaintext mono("3x^5"); // a short plaintext: the monomial branch of multiply_plain_normal (:2047-2092)
        ref.multiply_plain(cx, mono, r2);
        gpu.multiply_plain(cx, mono, g2);
        CHECK(same_ct(r2, g2));
        auto a = outcome([&] { Ciphertext tt = cx; ref.add_plain_inplace(tt, rp); });
        auto b = outcome([&] { Ciphertext tt = cx; gpu.add_plain_inplace(tt, gp); });
        CHECK(a == b && a == "invalid_argument"); // BFV plain cannot be in NTT form
    }
    {
        // Decryptor::decrypt on the device (BFV: phase + decrypt_scale_and_round), sizes 2 and 3
        seal_b200::Decryptor gdec(context, keygen.secret_key(), gpu);
        Plaintext rp, gp;
        decryptor.decrypt(cx, rp);
        gdec.decrypt(cx, gp);
        CHECK(same_plain(rp, gp));
        Ciphertext c3;
        ref.multiply(cx, cy, c3);
        decryptor.decrypt(c3, rp);
        gdec.decrypt(c3, gp);
        CHECK(same_plain(rp, gp));
        auto a = outcome([&] { Ciphertext tt = cx; tt.is_ntt_form() = true; Plaintext p; decryptor.decrypt(tt, p); });
        auto b = outcome([&] { Ciphertext tt = cx; tt.is_ntt_form() = true; Plaintext p; gdec.decrypt(tt, p); });
        CHECK(a == b && a == "invalid_argument");
    }
    {
        // BatchEncoder on the device: encode / decode, unsigned and signed, short inputs
        seal_b200::BatchEncoder genc(context, gpu);
        CHECK(genc.slot_count() == encoder.slot_count());
        Plaintext rp, gp;
        encoder.encode(x, rp);
        genc.encode(x, gp);
        CHECK(rp.coeff_count() == gp.coeff_count() && rp.parms_id() == gp.parms_id() &&
              std::memcmp(rp.data(), gp.data(), rp.coeff_count() * 8) == 0);
        std::vector<uint64_t> rv, gv;
        encoder.decode(px, rv);
        genc.decode(px, gv);
        CHECK(rv == gv && gv == x);
        std::vector<int64_t> sx{ -5, 7, 0, -123456, 99 }, rs, gs;
        encoder.encode(sx, rp);
        genc.encode(sx, gp);
        CHECK(rp.coeff_count() == gp.coeff_count() && std::memcmp(rp.data(), gp.data(), rp.coeff_count() * 8) == 0);
        encoder.decode(rp, rs);
        genc.decode(gp, gs);
        CHECK(rs == gs && gs[0] == -5 && gs[3] == -123456 && gs[5] == 0);
        Plaintext small("7x^2 + 1"); // fewer than n coefficients
        encoder.decode(small, rv);
        genc.decode(small, gv);
        CHECK(rv == gv);
        auto a = outcome([&] { Plaintext tt; encoder.encode(std::vector<uint64_t>(n + 1, 1), tt); });
        auto b = outcome([&] { Plaintext tt; genc.encode(std::vector<uint64_t>(n + 1, 1), tt); });
        CHECK(a == b && a == "invalid_argument");
        a = outcome([&] { Plaintext tt; encoder.encode(std::vector<uint64_t>{ t }, tt); });
        b = outcome([&] { Plaintext tt; genc.encode(std::vector<uint64_t>{ t }, tt); });
        CHECK(a == b && a == "invalid_argument");
        // whole pipeline on the device side of the boundary: encode -> multiply_plain -> decrypt (reference) -> decode
        Ciphertext g2;
        gpu.multiply_plain(cx, gp, g2); // gp = encode(sx)
        Plaintext dp;
        decryptor.decrypt(g2, dp);
        genc.decode(dp, gs);
        CHECK(gs[0] == static_cast<int64_t>((t - 5 * x[0] % t) % t > t / 2 ? (t - 5 * x[0] % t) % t - t : (t - 5 * x[0] % t) % t));
    }
    {
        // multiply_many / exponentiate (evaluator.cpp:1649-1757)
        std::vector<Ciphertext> many{ cx, cy, cx };
        Ciphertext r2, g2;
        ref.multiply_many(many, rlk, r2);
        gpu.multiply_many(many, rlk, g2);
        CHECK(same_ct(r2, g2));
        ref.exponentiate(cx, 3, rlk, r2);
        gpu.exponentiate(cx, 3, rlk, g2);
        CHECK(same_ct(r2, g2));
        auto a = outcome([&] { Ciphertext t = cx; ref.exponentiate_inplace(t, 0, rlk); });
        auto b = outcome([&] { Ciphertext t = cx; gpu.exponentiate_inplace(t, 0, rlk); });
        CHECK(a == b && a == "invalid_argument");
        ref.mod_switch_to(cx, context.last_parms_id(), r2);
        gpu.mod_switch_to(cx, context.last_parms_id(), g2);
        CHECK(same_ct(r2, g2));
    }
    {
        // multiply_plain with an NTT-form plaintext: ciphertext in NTT form (:1991-1994) and in coefficient form (:2006-2011)
        Plaintext pn = py;
        ref.transform_to_ntt_inplace(pn, cx.parms_id());
        Ciphertext r2, g2;
        ref.multiply_plain(cx, pn, r2);
        gpu.multiply_plain(cx, pn, g2);
        CHECK(same_ct(r2, g2));
        Plaintext p;
        decryptor.decrypt(g2, p);
        std::vector<uint64_t> got;
        encoder.decode(p, got);
        bool ok = true;
        for (size_t i = 0; i < n; i++)
            ok = ok && got[i] == (x[i] * y[i]) % t;
        CHECK(ok);
        Ciphertext rn, gn;
        ref.transform_to_ntt(cx, rn);
        gn = rn;
        ref.multiply_plain_inplace(rn, pn);
        gpu.multiply_plain_inplace(gn, pn);
        CHECK(same_ct(rn, gn));
    }
    {
        Ciphertext bad = cx;
        bad.is_ntt_form() = true; // evaluator.cpp:397-400
        auto a = outcome([&] { Ciphertext tt; ref.multiply(bad, cy, tt); });
        auto b = outcome([&] { Ciphertext tt; gpu.multiply(bad, cy, tt); });
        CHECK(a == b && a == "invalid_argument");
        a = outcome([&] { Ciphertext tt = cx; ref.rescale_to_next_inplace(tt); });
        b = outcome([&] { Ciphertext tt = cx; gpu.rescale_to_next_inplace(tt); });
        CHECK(a == b && a == "invalid_argument"); // unsupported operation for scheme type
        a = outcome([&] { Ciphertext tt = cx; ref.apply_galois_inplace(tt, 4, glk); });
        b = outcome([&] { Ciphertext tt = cx; gpu.apply_galois_inplace(tt, 4, glk); });
        CHECK(a == b && a == "invalid_argument"); // even Galois element: no such key
    }
}

// SURVEY 8(f) rank 2: BGV -- NTT-form ciphertexts, correction factors, plain-modulus-aware mod-down
static void test_bgv()
{
    EncryptionParameters parms(scheme_type::bgv);
    const size_t n = 8192;
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::BFVDefault(n));
    parms.set_plain_modulus(PlainModulus::Batching(n, 20));
    SEALContext context(parms, true, sec_level_type::none);
    KeyGenerator keygen(context);
    RelinKeys rlk;
    keygen.create_relin_keys(rlk);
    GaloisKeys glk;
    keygen.create_galois_keys(glk);
    Encryptor encryptor(context, keygen.secret_key());
    Decryptor decryptor(context, keygen.secret_key());
    BatchEncoder encoder(context);
    seal::Evaluator ref(context);
    seal_b200::Evaluator gpu(context);
    const uint64_t t = parms.plain_modulus().value();

    std::mt19937_64 rng(11);
    std::vector<uint64_t> x(n), y(n);
    for (size_t i = 0; i < n; i++)
        x[i] = rng() % 500, y[i] = rng() % 500;
    Plaintext px, py;
    encoder.encode(x, px);
    encoder.encode(y, py);
    Ciphertext cx, cy;
    encryptor.encrypt_symmetric(px, cx);
    encryptor.encrypt_symmetric(py, cy);
    CHECK(cx.is_ntt_form());

    Ciphertext r1, g1;
    ref.multiply(cx, cy, r1);
    gpu.multiply(cx, cy, g1);
    CHECK(same_ct(r1, g1));
    ref.relinearize_inplace(r1, rlk);
    gpu.relinearize_inplace(g1, rlk);
    CHECK(same_ct(r1, g1));
    ref.mod_switch_to_next_inplace(r1);
    gpu.mod_switch_to_next_inplace(g1);
    CHECK(same_ct(r1, g1));
    CHECK(g1.correction_factor() != 1); // q_last^-1 mod t entered the metadata (evaluator.cpp:1288-1293)
    {
        // Decryptor::decrypt on the device (BGV: phase, INTT, exact base conversion, inverse correction factor)
        seal_b200::Decryptor gdec(context, keygen.secret_key(), gpu);
        Plaintext rp, gp;
        decryptor.decrypt(g1, rp);
        gdec.decrypt(g1, gp);
        CHECK(same_plain(rp, gp));
        decryptor.decrypt(cx, rp);
        gdec.decrypt(cx, gp);
        CHECK(same_plain(rp, gp));
    }
    {
        Plaintext p;
        decryptor.decrypt(g1, p);
        std::vector<uint64_t> got;
        encoder.decode(p, got);
        bool ok = true;
        for (size_t i = 0; i < n; i++)
            ok = ok && got[i] == (x[i] * y[i]) % t;
        CHECK(ok);
        CHECK(decryptor.invariant_noise_budget(g1) > 0);
    }
    {
        // a second level: square of the switched product, relinearize, switch again
        Ciphertext r2, g2;
        ref.square(r1, r2);
        gpu.square(g1, g2);
        CHECK(same_ct(r2, g2));
        ref.relinearize_inplace(r2, rlk);
        gpu.relinearize_inplace(g2, rlk);
        ref.mod_switch_to_next_inplace(r2);
        gpu.mod_switch_to_next_inplace(g2);
        CHECK(same_ct(r2, g2));
        Plaintext p;
        decryptor.decrypt(g2, p);
        std::vector<uint64_t> got;
        encoder.decode(p, got);
        bool ok = true;
        for (size_t i = 0; i < n; i++)
            ok = ok && got[i] == ((x[i] * y[i]) % t) * ((x[i] * y[i]) % t) % t;
        CHECK(ok);
    }
    for (int step : { 1, -3 })
    {
        Ciphertext r2, g2;
        ref.rotate_rows(r1, step, glk, r2);
        gpu.rotate_rows(g1, step, glk, g2);
        CHECK(same_ct(r2, g2));
    }
    {
        Ciphertext r2, g2;
        ref.rotate_columns(cx, glk, r2);
        gpu.rotate_columns(cx, glk, g2);
        CHECK(same_ct(r2, g2));
        std::vector<std::vector<Ciphertext>> out(1);
        std::vector<Ciphertext> a(2, cx), b(2, cy);
        gpu.multiply_relinearize(a, b, rlk, out[0]);
        Ciphertext r;
        ref.multiply(cx, cy, r);
        ref.relinearize_inplace(r, rlk);
        CHECK(same_ct(r, out[0][0]) && same_ct(r, out[0][1]));
    }
    {
        // add / sub across different correction factors (evaluator.cpp:50-118, :188-209): u = x two levels down,
        // w = x*y one level down, multiplied and switched once more
        Ciphertext u = cx, v = cy, w;
        ref.mod_switch_to_next_inplace(u);
        ref.mod_switch_to_next_inplace(v);
        ref.multiply(u, v, w);
        ref.relinearize_inplace(w, rlk);
        ref.mod_switch_to_next_inplace(w);
        ref.mod_switch_to_next_inplace(u);
        CHECK(u.correction_factor() != w.correction_factor());
        Ciphertext r2, g2;
        ref.add(u, w, r2);
        gpu.add(u, w, g2);
        CHECK(same_ct(r2, g2));
        Plaintext p;
        decryptor.decrypt(g2, p);
        std::vector<uint64_t> got;
        encoder.decode(p, got);
        bool ok = true;
        for (size_t i = 0; i < n; i++)
            ok = ok && got[i] == (x[i] + x[i] * y[i]) % t;
        CHECK(ok);
        ref.sub(w, u, r2);
        gpu.sub(w, u, g2);
        CHECK(same_ct(r2, g2));
        // add_plain / sub_plain / multiply_plain with a coefficient-form plaintext on a ciphertext whose correction factor is not 1
        {
            Ciphertext r3 = w, g3 = w;
            ref.add_plain_inplace(r3, py);
            gpu.add_plain_inplace(g3, py);
            CHECK(same_ct(r3, g3));
            ref.multiply_plain_inplace(r3, px);
            gpu.multiply_plain_inplace(g3, px);
            CHECK(same_ct(r3, g3));
            ref.sub_plain_inplace(r3, px);
            gpu.sub_plain_inplace(g3, px);
            CHECK(same_ct(r3, g3));
            Plaintext pp;
            decryptor.decrypt(g3, pp);
            std::vector<uint64_t> gg;
            encoder.decode(pp, gg);
            bool fine = true;
            for (size_t i = 0; i < n; i++)
                fine = fine && gg[i] == ((x[i] * y[i] + y[i]) % t * x[i] + t - x[i]) % t;
            CHECK(fine);
        }
        Ciphertext odd = u;
        odd.correction_factor() = 12345; // arbitrary factors take the same path
        ref.add(odd, w, r2);
        gpu.add(odd, w, g2);
        CHECK(same_ct(r2, g2));
    }
    {
        auto a = outcome([&] { Ciphertext tt = cx; ref.rescale_to_next_inplace(tt); });
        auto b = outcome([&] { Ciphertext tt = cx; gpu.rescale_to_next_inplace(tt); });
        CHECK(a == b && a == "invalid_argument"); // unsupported operation for scheme type
        Ciphertext bad = cx;
        bad.is_ntt_form() = false;
        a = outcome([&] { Ciphertext tt; ref.multiply(bad, cy, tt); });
        b = outcome([&] { Ciphertext tt; gpu.multiply(bad, cy, tt); });
        CHECK(a == b && a == "invalid_argument"); // :712-715
        a = outcome([&] { Ciphertext tt = bad; ref.mod_switch_to_next_inplace(tt); });
        b = outcome([&] { Ciphertext tt = bad; gpu.mod_switch_to_next_inplace(tt); });
        CHECK(a == b && a == "invalid_argument"); // BGV encrypted must be in NTT form
        a = outcome([&] { Ciphertext tt = cx; ref.rotate_vector_inplace(tt, 1, glk); });
        b = outcome([&] { Ciphertext tt = cx; gpu.rotate_vector_inplace(tt, 1, glk); });
        CHECK(a == b && a == "logic_error");
    }
}

// Device-resident batches (seal_b200::CiphertextBatch): a chain of operations that leaves the GPU once, checked against the
// reference evaluator ciphertext by ciphertext (words and metadata); the reference's usage pattern is the chain
// multiply -> relinearize -> rescale of native/tests/seal/evaluator.cpp:3513-3780.
static void test_batches_and_keys()
{
    EncryptionParameters parms(scheme_type::ckks);
    const size_t n = 8192;
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::Create(n, { 50, 40, 40, 40, 50 }));
    SEALContext context(parms, true, sec_level_type::none);
    KeyGenerator keygen(context);
    PublicKey pk;
    keygen.create_public_key(pk);
    RelinKeys rlk;
    keygen.create_relin_keys(rlk);
    GaloisKeys glk;
    keygen.create_galois_keys(std::vector<int>{ 1, 2, 4, -1 }, glk); // 3 = 4 - 1 goes through the NAF fallback
    Encryptor encryptor(context, pk);
    CKKSEncoder encoder(context);
    seal::Evaluator ref(context);
    seal_b200::Evaluator gpu(context);
    const double scale = std::pow(2.0, 40);
    const size_t B = 5;
    std::mt19937_64 rng(11);
    std::vector<Ciphertext> a(B), b(B);
    for (size_t i = 0; i < B; i++)
    {
        std::vector<double> x(n / 2), y(n / 2);
        for (auto &v : x)
            v = double(rng() % 1000) / 100.0;
        for (auto &v : y)
            v = double(rng() % 1000) / 100.0;
        Plaintext px, py;
        encoder.encode(x, scale, px);
        encoder.encode(y, scale, py);
        encryptor.encrypt(px, a[i]);
        encryptor.encrypt(py, b[i]);
    }
    // depth-2 chain on the device: a <- rescale(relin(a*b)); b <- mod_switch_to_next(b)   (SURVEY 8d, cfg3's chain)
    seal_b200::CiphertextBatch da, db;
    gpu.upload(a, da);
    gpu.upload(b, db);
    std::vector<Ciphertext> ra = a, rb = b;
    for (int depth = 0; depth < 2; depth++)
    {
        gpu.multiply_relinearize_inplace(da, db, rlk);
        gpu.rescale_to_next_inplace(da);
        gpu.mod_switch_to_next_inplace(db);
        // keep the scales aligned the way a user would (the reference does the same below)
        db.scale() = da.scale();
        for (size_t i = 0; i < B; i++)
        {
            ref.multiply_inplace(ra[i], rb[i]);
            ref.relinearize_inplace(ra[i], rlk);
            ref.rescale_to_next_inplace(ra[i]);
            ref.mod_switch_to_next_inplace(rb[i]);
            rb[i].scale() = ra[i].scale();
        }
    }
    gpu.rotate_vector_inplace(da, 3, glk); // NAF fallback: -1, then 4
    gpu.add_inplace(da, db);
    gpu.negate_inplace(da);
    std::vector<Ciphertext> ga, gb;
    gpu.download(da, ga);
    gpu.download(db, gb);
    CHECK(ga.size() == B && gb.size() == B);
    for (size_t i = 0; i < B; i++)
    {
        ref.rotate_vector_inplace(ra[i], 3, glk);
        ref.add_inplace(ra[i], rb[i]);
        ref.negate_inplace(ra[i]);
        CHECK(same_ct(ra[i], ga[i]));
        CHECK(same_ct(rb[i], gb[i]));
    }
    {
        // unfused on the device: multiply (size 3), square of it (size 5), mod switch of a size-3 batch, transforms
        seal_b200::CiphertextBatch dx, dy;
        gpu.upload(a, dx);
        gpu.upload(b, dy);
        gpu.multiply_inplace(dx, dy);
        CHECK(dx.size() == 3);
        gpu.mod_switch_to_next_inplace(dx); // size 3: the reference switches every polynomial (evaluator.cpp:1263-1280)
        gpu.transform_from_ntt_inplace(dx);
        gpu.transform_to_ntt_inplace(dx);
        gpu.relinearize_inplace(dx, rlk);
        std::vector<Ciphertext> gx;
        gpu.download(dx, gx);
        for (size_t i = 0; i < B; i++)
        {
            Ciphertext r;
            ref.multiply(a[i], b[i], r);
            ref.mod_switch_to_next_inplace(r);
            ref.relinearize_inplace(r, rlk);
            CHECK(same_ct(r, gx[i]));
        }
        // single-ciphertext members on sizes other than 2 (ADVICE: the shim used to reject them)
        Ciphertext r3, g3;
        ref.multiply(a[0], b[0], r3);
        g3 = r3;
        ref.rescale_to_next_inplace(r3);
        gpu.rescale_to_next_inplace(g3);
        CHECK(r3.size() == 3 && same_ct(r3, g3));
        // identical exception for mismatching batches
        auto o = outcome([&] { gpu.add_inplace(dx, dy); });
        CHECK(o == "invalid_argument");
    }
    {
        // batch overload on std::vector with destination aliasing an operand (ADVICE: metadata was read after the overwrite)
        std::vector<Ciphertext> u = a, v = b;
        v[2].scale() = a[2].scale();
        gpu.multiply_relinearize(u, v, rlk, v);
        for (size_t i = 0; i < B; i++)
        {
            Ciphertext r;
            ref.multiply(a[i], b[i], r);
            ref.relinearize_inplace(r, rlk);
            CHECK(same_ct(r, v[i]));
        }
    }
    {
        // the key cache is keyed by content, never by address: destroy and regenerate Galois keys between two rotations
        // (SEAL's pool hands the freed block straight back, so the new key lands where the old one was)
        Ciphertext r, g;
        auto gk1 = std::make_unique<GaloisKeys>();
        keygen.create_galois_keys(std::vector<int>{ 1 }, *gk1);
        ref.rotate_vector(a[0], 1, *gk1, r);
        gpu.rotate_vector(a[0], 1, *gk1, g);
        CHECK(same_ct(r, g));
        const void *old_addr = gk1->data()[GaloisKeys::get_index(context.key_context_data()->galois_tool()->get_elt_from_step(1))][0].data().data();
        gk1.reset();
        KeyGenerator keygen2(context); // another secret key: a different tenant
        auto gk2 = std::make_unique<GaloisKeys>();
        keygen2.create_galois_keys(std::vector<int>{ 1 }, *gk2);
        const void *new_addr = gk2->data()[GaloisKeys::get_index(context.key_context_data()->galois_tool()->get_elt_from_step(1))][0].data().data();
        std::printf("galois key regenerated at %s address\n", old_addr == new_addr ? "the SAME" : "a different");
        ref.rotate_vector(a[0], 1, *gk2, r);
        gpu.rotate_vector(a[0], 1, *gk2, g);
        CHECK(same_ct(r, g));
        // eviction: a budget of one key keeps the cache at one entry and results stay right
        gpu.set_key_cache_limit(1);
        for (int step : { 1, 2, -1, 1 })
        {
            ref.rotate_vector(a[1], step, glk, r);
            gpu.rotate_vector(a[1], step, glk, g);
            CHECK(same_ct(r, g));
            CHECK(gpu.key_cache_entries() == 1);
        }
        gpu.clear_key_cache();
        CHECK(gpu.key_cache_entries() == 0);
        gpu.set_key_cache_limit(std::size_t(24) << 30);
    }
    {
        // relinearize of a size-4 ciphertext.  KeyGenerator only makes one relinearization key, so the second key slot is
        // filled with a copy (any valid key-switching key will do for a word-for-word comparison): both evaluators must
        // agree on the reference's loop (evaluator.cpp:1176-1187)
        RelinKeys two = rlk;
        two.data().resize(2);
        two.data()[1] = two.data()[0];
        Ciphertext c3, lo = a[0], r4, g4;
        ref.multiply(a[0], b[0], c3);
        lo.scale() = 4.0, c3.scale() = 4.0;
        ref.multiply(c3, lo, r4);
        g4 = r4;
        CHECK(r4.size() == 4);
        ref.relinearize_inplace(r4, two);
        gpu.relinearize_inplace(g4, two);
        CHECK(r4.size() == 2 && same_ct(r4, g4));
        auto x = outcome([&] { Ciphertext t4; ref.multiply(c3, lo, t4); ref.relinearize_inplace(t4, rlk); });
        auto y = outcome([&] { Ciphertext t4; ref.multiply(c3, lo, t4); gpu.relinearize_inplace(t4, rlk); });
        CHECK(x == y && x == "invalid_argument"); // not enough relinearization keys
        seal_b200::CiphertextBatch d4;
        std::vector<Ciphertext> v4(3), out4;
        for (auto &c : v4)
            ref.multiply(c3, lo, c);
        gpu.upload(v4, d4);
        gpu.relinearize_inplace(d4, two);
        gpu.download(d4, out4);
        for (auto &c : out4)
            CHECK(same_ct(r4, c));
    }
}

// seal_b200::CKKSEncoder and seal_b200::Encryptor (symmetric) against the reference's classes: identical plaintexts, decoded
// values and -- with a seeded random generator factory on the context, so that both sides draw the same bootstrap seed --
// identical fresh ciphertexts; cf. native/tests/seal/ckks.cpp (CKKSEncoderEncodeVectorDecodeTest), encryptor.cpp
// (BFVEncryptDecrypt / CKKSEncryptDecrypt, the symmetric halves)
static void test_encoder_and_encryptor()
{
    prng_seed_type seed{};
    seed[0] = 0xABCDEF;
    {
        EncryptionParameters parms(scheme_type::ckks);
        parms.set_poly_modulus_degree(8192);
        parms.set_coeff_modulus(CoeffModulus::Create(8192, { 60, 40, 40, 60 }));
        parms.set_random_generator(std::make_shared<Blake2xbPRNGFactory>(seed));
        SEALContext context(parms, true, sec_level_type::none);
        KeyGenerator keygen(context);
        seal::CKKSEncoder renc(context);
        seal::Encryptor rcrypt(context, keygen.secret_key());
        seal::Decryptor rdec(context, keygen.secret_key());
        seal_b200::Evaluator gev(context);
        seal_b200::CKKSEncoder genc(context, gev);
        seal_b200::Encryptor gcrypt(context, keygen.secret_key(), gev);
        CHECK(genc.slot_count() == renc.slot_count());
        std::mt19937_64 rng(3);
        std::uniform_real_distribution<double> dist(-10.0, 10.0);
        std::vector<std::complex<double>> cv(renc.slot_count());
        for (auto &v : cv)
            v = { dist(rng), dist(rng) };
        std::vector<double> rv(100);
        for (auto &v : rv)
            v = dist(rng);
        const double scale = std::pow(2.0, 40);
        Plaintext pr, pg;
        renc.encode(cv, scale, pr);
        genc.encode(cv, scale, pg);
        CHECK(same_plain(pr, pg));
        CHECK(pg.is_ntt_form());
        renc.encode(rv, scale, pr);
        genc.encode(rv, scale, pg);
        CHECK(same_plain(pr, pg));
        auto low = context.last_parms_id();
        renc.encode(cv, low, std::pow(2.0, 20), pr);
        genc.encode(cv, low, std::pow(2.0, 20), pg);
        CHECK(same_plain(pr, pg));
        std::vector<std::complex<double>> dr, dg;
        renc.decode(pr, dr);
        genc.decode(pg, dg);
        CHECK(dr.size() == dg.size() && std::memcmp(dr.data(), dg.data(), dr.size() * 16) == 0);
        std::vector<double> ddr, ddg;
        renc.decode(pr, ddr);
        genc.decode(pg, ddg);
        CHECK(ddr.size() == ddg.size() && std::memcmp(ddr.data(), ddg.data(), ddr.size() * 8) == 0);
        // batch encode = the single-vector results
        std::vector<std::vector<std::complex<double>>> many{ cv, std::vector<std::complex<double>>(cv.begin(), cv.begin() + 7), cv };
        std::vector<Plaintext> pb;
        genc.encode(many, context.first_parms_id(), scale, pb);
        for (size_t i = 0; i < many.size(); i++)
        {
            renc.encode(many[i], scale, pr);
            CHECK(same_plain(pr, pb[i]));
        }
        // the reference's exception types
        CHECK(outcome([&] { renc.encode(cv, std::pow(2.0, 300), pr); }) == outcome([&] { genc.encode(cv, std::pow(2.0, 300), pg); }));
        std::vector<std::complex<double>> big(4, { 1e200, 0 });
        CHECK(outcome([&] { renc.encode(big, scale, pr); }) == outcome([&] { genc.encode(big, scale, pg); }));
        std::vector<std::complex<double>> toolong(renc.slot_count() + 1);
        CHECK(outcome([&] { renc.encode(toolong, scale, pr); }) == outcome([&] { genc.encode(toolong, scale, pg); }));
        // symmetric encryption: the same bootstrap seed on both sides -> the same ciphertext
        renc.encode(cv, scale, pr);
        Ciphertext cr, cg;
        rcrypt.encrypt_symmetric(pr, cr);
        gcrypt.encrypt_symmetric(pr, cg);
        CHECK(same_ct(cr, cg));
        rcrypt.encrypt_zero_symmetric(cr);
        gcrypt.encrypt_zero_symmetric(cg);
        CHECK(same_ct(cr, cg));
        rcrypt.encrypt_zero_symmetric(low, cr);
        gcrypt.encrypt_zero_symmetric(low, cg);
        CHECK(same_ct(cr, cg));
        renc.encode(cv, low, std::pow(2.0, 20), pr);
        rcrypt.encrypt_symmetric(pr, cr);
        gcrypt.encrypt_symmetric(pr, cg);
        CHECK(same_ct(cr, cg));
        // public-key encryption: first level, a lower level (sampled one level up, divided down)
        {
            PublicKey pk;
            keygen.create_public_key(pk);
            seal::Encryptor rpub(context, pk);
            seal_b200::Encryptor gpub(context, pk, gev);
            renc.encode(cv, scale, pr);
            rpub.encrypt(pr, cr);
            gpub.encrypt(pr, cg);
            CHECK(same_ct(cr, cg));
            rpub.encrypt_zero(low, cr);
            gpub.encrypt_zero(low, cg);
            CHECK(same_ct(cr, cg));
            renc.encode(cv, low, std::pow(2.0, 20), pr);
            rpub.encrypt(pr, cr);
            gpub.encrypt(pr, cg);
            CHECK(same_ct(cr, cg));
            CHECK(outcome([&] { rpub.encrypt_symmetric(pr, cr); }) == outcome([&] { gpub.encrypt_symmetric(pr, cg); })); // secret key is not set
            CHECK(outcome([&] { rcrypt.encrypt(pr, cr); }) == outcome([&] { gcrypt.encrypt(pr, cg); }));                 // public key is not set
        }
        // round trip through the device classes only: encode -> encrypt -> (reference) decrypt -> decode
        genc.encode(cv, scale, pg);
        gcrypt.encrypt_symmetric(pg, cg);
        Plaintext back;
        rdec.decrypt(cg, back);
        genc.decode(back, dg);
        double err = 0;
        for (size_t i = 0; i < cv.size(); i++)
            err = std::max(err, std::abs(dg[i] - cv[i]));
        CHECK(err < 1e-6);
        // batch encryption: every member equals the single call (seeded factory: the same seed each time)
        std::vector<Plaintext> plains{ pg, pg, pg };
        std::vector<Ciphertext> cts;
        gcrypt.encrypt_symmetric(plains, cts);
        rcrypt.encrypt_symmetric(pg, cr);
        for (auto &c : cts)
            CHECK(same_ct(cr, c));
        CHECK(outcome([&] { Plaintext bad; rcrypt.encrypt_symmetric(bad, cr); }) == outcome([&] { Plaintext bad; gcrypt.encrypt_symmetric(bad, cg); }));
    }
    for (auto scheme : { scheme_type::bfv, scheme_type::bgv })
    {
        EncryptionParameters parms(scheme);
        parms.set_poly_modulus_degree(4096);
        parms.set_coeff_modulus(CoeffModulus::Create(4096, { 36, 36, 37 }));
        parms.set_plain_modulus(PlainModulus::Batching(4096, 20));
        parms.set_random_generator(std::make_shared<Blake2xbPRNGFactory>(seed));
        SEALContext context(parms, true, sec_level_type::none);
        KeyGenerator keygen(context);
        seal::BatchEncoder benc(context);
        seal::Encryptor rcrypt(context, keygen.secret_key());
        seal::Decryptor rdec(context, keygen.secret_key());
        seal_b200::Evaluator gev(context);
        seal_b200::Encryptor gcrypt(context, keygen.secret_key(), gev);
        std::vector<uint64_t> slots(benc.slot_count());
        for (size_t i = 0; i < slots.size(); i++)
            slots[i] = (i * 7919 + 13) % parms.plain_modulus().value();
        Plaintext p;
        benc.encode(slots, p);
        Ciphertext cr, cg;
        rcrypt.encrypt_symmetric(p, cr);
        gcrypt.encrypt_symmetric(p, cg);
        CHECK(same_ct(cr, cg));
        rcrypt.encrypt_zero_symmetric(cr);
        gcrypt.encrypt_zero_symmetric(cg);
        CHECK(same_ct(cr, cg));
        Plaintext back;
        rdec.decrypt(cg, back);
        CHECK(back.is_zero());
        Plaintext small("1x^3 + 2");
        rcrypt.encrypt_symmetric(small, cr);
        gcrypt.encrypt_symmetric(small, cg);
        CHECK(same_ct(cr, cg));
        PublicKey pk;
        keygen.create_public_key(pk);
        seal::Encryptor rpub(context, pk);
        seal_b200::Encryptor gpub(context, pk, keygen.secret_key(), gev);
        rpub.encrypt(p, cr);
        gpub.encrypt(p, cg);
        CHECK(same_ct(cr, cg));
        rdec.decrypt(cg, back);
        CHECK(back == p);
        rpub.encrypt_zero(context.last_parms_id(), cr);
        gpub.encrypt_zero(context.last_parms_id(), cg);
        CHECK(same_ct(cr, cg));
    }
    // default factory: fresh seeds, two encryptions differ and decrypt correctly
    {
        EncryptionParameters parms(scheme_type::bfv);
        parms.set_poly_modulus_degree(4096);
        parms.set_coeff_modulus(CoeffModulus::BFVDefault(4096));
        parms.set_plain_modulus(PlainModulus::Batching(4096, 20));
        SEALContext context(parms);
        KeyGenerator keygen(context);
        seal::Decryptor rdec(context, keygen.secret_key());
        seal_b200::Evaluator gev(context);
        seal_b200::Encryptor gcrypt(context, keygen.secret_key(), gev);
        Plaintext p("5x^2 + 1"), back;
        Ciphertext a, b;
        gcrypt.encrypt_symmetric(p, a);
        gcrypt.encrypt_symmetric(p, b);
        CHECK(!same_ct(a, b));
        rdec.decrypt(a, back);
        CHECK(back == p);
        CHECK(rdec.invariant_noise_budget(a) > 20);
    }
}

// ---- precedence matrix: invalid operands through seal::Evaluator, seal_b200::Evaluator on the same ciphertexts and on batches
// uploaded from them, with the exception type AND message compared; doubly-invalid cases show the order of the checks.  A batch
// keeps its words and metadata when a member throws.
template <class F>
static std::string thrown(F f)
{
    try
    {
        f();
        return "ok";
    }
    catch (const std::exception &e)
    {
        return outcome([] { throw; }) + ": " + e.what();
    }
}

struct Precedence
{
    seal::Evaluator &ref;
    seal_b200::Evaluator &gpu;
    // two copies of ct on the device
    seal_b200::CiphertextBatch up(const Ciphertext &ct) const
    {
        seal_b200::CiphertextBatch d;
        gpu.upload(std::vector<Ciphertext>(2, ct), d);
        return d;
    }
    seal_b200::PlaintextBatch up(const Plaintext &pt) const
    {
        seal_b200::PlaintextBatch d;
        gpu.upload(std::vector<Plaintext>(2, pt), d);
        return d;
    }
    // r(x) on the reference, s(x) on the drop-in, b(batch of x) on the drop-in: the same error, and the batch unchanged
    template <class R, class S, class B>
    void operator()(const char *name, const Ciphertext &x, R r, S s, B b) const
    {
        Ciphertext rx = x, sx = x;
        const std::string want = thrown([&] { r(rx); }), one = thrown([&] { s(sx); });
        seal_b200::CiphertextBatch d = up(x);
        const std::string batch = thrown([&] { b(d); });
        std::vector<Ciphertext> back;
        gpu.download(d, back);
        const bool kept = back.size() == 2 && same_ct(back[0], x) && same_ct(back[1], x);
        g_checks++;
        if (want == "ok" || one != want || batch != want || !kept)
        {
            g_fail++;
            std::printf("FAIL precedence %s: reference [%s], Ciphertext [%s], batch [%s]%s\n", name, want.c_str(), one.c_str(), batch.c_str(),
                        kept ? "" : ", batch changed");
        }
    }
    // the same member on both evaluators and the batch: f(evaluator, operand) for the first two, g(batch) for the third
    template <class F, class G>
    void same(const char *name, const Ciphertext &x, F f, G g) const
    {
        (*this)(name, x, [&](Ciphertext &t) { f(ref, t); }, [&](Ciphertext &t) { f(gpu, t); }, g);
    }
    // a plaintext member: reference, drop-in and PlaintextBatch give the same error
    template <class F>
    void plain(const char *name, const Plaintext &p, F f) const
    {
        Plaintext rp = p, sp = p;
        seal_b200::PlaintextBatch d = up(p);
        const std::string want = thrown([&] { f(ref, rp); }), one = thrown([&] { f(gpu, sp); }), batch = thrown([&] { f(gpu, d); });
        g_checks++;
        if (want == "ok" || one != want || batch != want)
        {
            g_fail++;
            std::printf("FAIL precedence %s: reference [%s], Plaintext [%s], batch [%s]\n", name, want.c_str(), one.c_str(), batch.c_str());
        }
    }
};

static void test_precedence_ckks()
{
    EncryptionParameters parms(scheme_type::ckks);
    const size_t n = 16384;
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::Create(n, { 60, 50, 50, 40, 60 })); // 200 bits at the first data level
    SEALContext context(parms, true, sec_level_type::none);
    KeyGenerator keygen(context);
    PublicKey pk;
    keygen.create_public_key(pk);
    RelinKeys rlk;
    keygen.create_relin_keys(rlk);
    GaloisKeys glk;
    keygen.create_galois_keys(std::vector<int>{ 1 }, glk);
    Encryptor encryptor(context, pk);
    CKKSEncoder encoder(context);
    seal::Evaluator ref(context);
    seal_b200::Evaluator gpu(context);
    const Precedence check{ ref, gpu };
    auto fresh = [&](double scale) {
        Plaintext p;
        encoder.encode(std::vector<double>(n / 2, 1.0), scale, p);
        Ciphertext c;
        encryptor.encrypt(p, c);
        return c;
    };
    const double s40 = std::pow(2.0, 40);
    Ciphertext x = fresh(s40), y = fresh(s40), y_low, y_coeff, x_coeff, x_last, x_big = x, m3, m4;
    ref.mod_switch_to_next(y, y_low);
    ref.transform_from_ntt(y, y_coeff);
    ref.transform_from_ntt(x, x_coeff);
    ref.mod_switch_to(x, context.last_parms_id(), x_last);
    x_big.scale() = std::pow(2.0, 120);
    ref.multiply(x, y, m3);
    ref.multiply(m3, y, m4);
    // size 9 by three unrelinearized products: at scale 2^10 the product of two is only too large, at 2^20 also out of bounds
    auto size9 = [&](double scale) {
        Ciphertext c = fresh(scale);
        for (int i = 0; i < 3; i++)
        {
            const Ciphertext d = c;
            ref.multiply_inplace(c, d);
        }
        return c;
    };
    const Ciphertext s9 = size9(std::pow(2.0, 10)), t9 = size9(std::pow(2.0, 20));
    Plaintext p, p_low, p_big;
    encoder.encode(std::vector<double>(n / 2, 2.0), s40, p);
    ref.mod_switch_to_next(p, p_low);
    p_big = p, p_big.scale() = std::pow(2.0, 120);

    auto multiply = [&](const char *name, const Ciphertext &a, const Ciphertext &b) {
        check.same(name, a, [&](auto &ev, Ciphertext &t) { ev.multiply_inplace(t, b); },
                   [&](seal_b200::CiphertextBatch &d) { auto e = check.up(b); gpu.multiply_inplace(d, e); });
    };
    multiply("CKKS multiply parameter mismatch", x, y_low);
    multiply("CKKS multiply form", x, y_coeff);
    multiply("CKKS multiply size", s9, s9);
    multiply("CKKS multiply scale", x_big, x_big);
    multiply("CKKS multiply size and scale", t9, t9);
    multiply("CKKS multiply mismatch and form", x_coeff, y_low);
    auto add = [&](const char *name, const Ciphertext &a, const Ciphertext &b) {
        check.same(name, a, [&](auto &ev, Ciphertext &t) { ev.sub_inplace(t, b); },
                   [&](seal_b200::CiphertextBatch &d) { auto e = check.up(b); gpu.sub_inplace(d, e); });
    };
    Ciphertext y_scaled = y;
    y_scaled.scale() *= 2;
    add("CKKS sub parameter mismatch", x, y_low);
    add("CKKS sub form", x, y_coeff);
    add("CKKS sub scale", x, y_scaled);
    add("CKKS sub form and scale", x_coeff, y_scaled);
    auto multiply_plain = [&](const char *name, const Ciphertext &a, const Plaintext &q) {
        check.same(name, a, [&](auto &ev, Ciphertext &t) { ev.multiply_plain_inplace(t, q); },
                   [&](seal_b200::CiphertextBatch &d) { auto e = check.up(q); gpu.multiply_plain_inplace(d, e); });
    };
    multiply_plain("CKKS multiply_plain parameter mismatch", x, p_low);
    multiply_plain("CKKS multiply_plain scale", x_big, p_big);
    multiply_plain("CKKS multiply_plain mismatch and scale", x_big, [&] { Plaintext q = p_low; q.scale() = p_big.scale(); return q; }());
    auto add_plain = [&](const char *name, const Ciphertext &a, const Plaintext &q) {
        check.same(name, a, [&](auto &ev, Ciphertext &t) { ev.add_plain_inplace(t, q); },
                   [&](seal_b200::CiphertextBatch &d) { auto e = check.up(q); gpu.add_plain_inplace(d, e); });
    };
    add_plain("CKKS add_plain form", x_coeff, p);
    add_plain("CKKS add_plain parameter mismatch", x, p_low);
    add_plain("CKKS add_plain scale", x, p_big);
    add_plain("CKKS add_plain form and mismatch", x_coeff, p_low);
    RelinKeys rlk_bad = rlk;
    rlk_bad.parms_id() = parms_id_zero;
    auto relinearize = [&](const char *name, const Ciphertext &a, const RelinKeys &k) {
        check.same(name, a, [&](auto &ev, Ciphertext &t) { ev.relinearize_inplace(t, k); }, [&](seal_b200::CiphertextBatch &d) { gpu.relinearize_inplace(d, k); });
    };
    Ciphertext m3_coeff;
    ref.transform_from_ntt(m3, m3_coeff);
    relinearize("CKKS relinearize key level", m3, rlk_bad);
    relinearize("CKKS relinearize too few keys", m4, rlk);
    relinearize("CKKS relinearize form", m3_coeff, rlk);
    relinearize("CKKS relinearize key level and too few keys", m4, rlk_bad);
    GaloisKeys glk_bad = glk;
    glk_bad.parms_id() = parms_id_zero;
    const std::uint32_t e1 = context.key_context_data()->galois_tool()->get_elt_from_step(1);
    const std::uint32_t e2 = context.key_context_data()->galois_tool()->get_elt_from_step(2);
    auto galois = [&](const char *name, const Ciphertext &a, std::uint32_t elt, const GaloisKeys &k) {
        check.same(name, a, [&](auto &ev, Ciphertext &t) { ev.apply_galois_inplace(t, elt, k); },
                   [&](seal_b200::CiphertextBatch &d) { gpu.apply_galois_inplace(d, elt, k); });
    };
    galois("CKKS apply_galois key level", x, e1, glk_bad);
    galois("CKKS apply_galois missing key", x, e2, glk);
    galois("CKKS apply_galois even element", x, 4, glk);
    galois("CKKS apply_galois element too large", x, 2 * n + 1, glk);
    galois("CKKS apply_galois size", m3, e1, glk);
    galois("CKKS apply_galois form", x_coeff, e1, glk);
    galois("CKKS apply_galois size and form", m3_coeff, e1, glk);
    check.same("CKKS rotate_rows scheme", x, [&](auto &ev, Ciphertext &t) { ev.rotate_rows_inplace(t, 1, glk); },
               [&](seal_b200::CiphertextBatch &d) { gpu.rotate_rows_inplace(d, 1, glk); });
    check.same("CKKS rotate_vector missing key", x, [&](auto &ev, Ciphertext &t) { ev.rotate_vector_inplace(t, 2, glk); },
               [&](seal_b200::CiphertextBatch &d) { gpu.rotate_vector_inplace(d, 2, glk); });
    check.same("CKKS rotate_vector key level and missing key", x, [&](auto &ev, Ciphertext &t) { ev.rotate_vector_inplace(t, 2, glk_bad); },
               [&](seal_b200::CiphertextBatch &d) { gpu.rotate_vector_inplace(d, 2, glk_bad); });
    check.same("CKKS complex_conjugate missing key", x, [&](auto &ev, Ciphertext &t) { ev.complex_conjugate_inplace(t, glk); },
               [&](seal_b200::CiphertextBatch &d) { gpu.complex_conjugate_inplace(d, glk); });
    check.same("CKKS rotate_columns scheme", x, [&](auto &ev, Ciphertext &t) { ev.rotate_columns_inplace(t, glk); },
               [&](seal_b200::CiphertextBatch &d) { gpu.rotate_columns_inplace(d, glk); });
    auto rescale = [&](const char *name, const Ciphertext &a) {
        check.same(name, a, [&](auto &ev, Ciphertext &t) { ev.rescale_to_next_inplace(t); }, [&](seal_b200::CiphertextBatch &d) { gpu.rescale_to_next_inplace(d); });
    };
    Ciphertext x_huge = x, x_huge_coeff = x_coeff;
    x_huge.scale() = x_huge_coeff.scale() = std::pow(2.0, 250);
    rescale("CKKS rescale_to_next end of chain", x_last);
    rescale("CKKS rescale_to_next form", x_coeff);
    rescale("CKKS rescale_to_next scale", x_huge);
    rescale("CKKS rescale_to_next form and scale", x_huge_coeff);
    check.same("CKKS mod_switch_to_next form", x_coeff, [&](auto &ev, Ciphertext &t) { ev.mod_switch_to_next_inplace(t); },
               [&](seal_b200::CiphertextBatch &d) { gpu.mod_switch_to_next_inplace(d); });
    check.same("CKKS mod_switch_to_next scale", x_huge, [&](auto &ev, Ciphertext &t) { ev.mod_switch_to_next_inplace(t); },
               [&](seal_b200::CiphertextBatch &d) { gpu.mod_switch_to_next_inplace(d); });
    const parms_id_type top = x.parms_id();
    check.same("CKKS rescale_to a higher level", y_low, [&](auto &ev, Ciphertext &t) { ev.rescale_to_inplace(t, top); },
               [&](seal_b200::CiphertextBatch &d) { gpu.rescale_to_inplace(d, top); });
    check.same("CKKS mod_switch_to a higher level", y_low, [&](auto &ev, Ciphertext &t) { ev.mod_switch_to_inplace(t, top); },
               [&](seal_b200::CiphertextBatch &d) { gpu.mod_switch_to_inplace(d, top); });
    Plaintext p_tight = p, p_last;
    p_tight.scale() = std::pow(2.0, 170); // within the first level's 200 bits, not the next level's 160
    ref.mod_switch_to(p, context.last_parms_id(), p_last);
    check.plain("CKKS plaintext mod_switch_to_next scale", p_tight, [](auto &ev, auto &q) { ev.mod_switch_to_next_inplace(q); });
    check.plain("CKKS plaintext mod_switch_to_next end of chain", p_last, [](auto &ev, auto &q) { ev.mod_switch_to_next_inplace(q); });
    check.plain("CKKS plaintext mod_switch_to a higher level", p_low, [&](auto &ev, auto &q) { ev.mod_switch_to_inplace(q, top); });
}

// BFV and BGV: the per-scheme form rules, rotations, plaintext level changes and multiply_relinearize_inplace against its chain
static void test_precedence_integer(scheme_type scheme)
{
    const bool bfv = scheme == scheme_type::bfv;
    EncryptionParameters parms(scheme);
    const size_t n = 4096;
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::Create(n, { 30, 30, 40 }));
    parms.set_plain_modulus(PlainModulus::Batching(n, 20));
    SEALContext context(parms, true, sec_level_type::none);
    KeyGenerator keygen(context);
    PublicKey pk;
    keygen.create_public_key(pk);
    RelinKeys rlk;
    keygen.create_relin_keys(rlk);
    GaloisKeys glk;
    keygen.create_galois_keys(std::vector<int>{ 1 }, glk);
    Encryptor encryptor(context, pk);
    BatchEncoder encoder(context);
    seal::Evaluator ref(context);
    seal_b200::Evaluator gpu(context);
    const Precedence check{ ref, gpu };
    Plaintext p, p_ntt, p_ntt_low, p_last;
    encoder.encode(std::vector<std::uint64_t>(n, 3), p);
    ref.transform_to_ntt(p, context.first_parms_id(), p_ntt);
    ref.transform_to_ntt(p, context.last_parms_id(), p_ntt_low);
    p_last = p_ntt_low;
    Ciphertext x, y, x_wrong, y_low, x_last, x_last_wrong, m3, m3_wrong;
    encryptor.encrypt(p, x);
    encryptor.encrypt(p, y);
    if (bfv)
        ref.transform_to_ntt(x, x_wrong);
    else
        ref.transform_from_ntt(x, x_wrong);
    ref.mod_switch_to_next(y, y_low);
    ref.mod_switch_to_next(x, x_last);
    if (bfv)
        ref.transform_to_ntt(x_last, x_last_wrong);
    else
        ref.transform_from_ntt(x_last, x_last_wrong);
    ref.multiply(x, y, m3);
    if (bfv)
        ref.transform_to_ntt(m3, m3_wrong);
    else
        ref.transform_from_ntt(m3, m3_wrong);
    const std::string tag = bfv ? "BFV " : "BGV ";
    auto name = [&](const char *what) { static std::string s; s = tag + what; return s.c_str(); };

    auto multiply = [&](const char *what, const Ciphertext &a, const Ciphertext &b) {
        check.same(name(what), a, [&](auto &ev, Ciphertext &t) { ev.multiply_inplace(t, b); },
                   [&](seal_b200::CiphertextBatch &d) { auto e = check.up(b); gpu.multiply_inplace(d, e); });
    };
    multiply("multiply parameter mismatch", x, y_low);
    multiply("multiply form", x_wrong, y);
    multiply("multiply mismatch and form", x_wrong, y_low);
    auto add_plain = [&](const char *what, const Ciphertext &a, const Plaintext &q) {
        check.same(name(what), a, [&](auto &ev, Ciphertext &t) { ev.add_plain_inplace(t, q); },
                   [&](seal_b200::CiphertextBatch &d) { auto e = check.up(q); gpu.add_plain_inplace(d, e); });
    };
    add_plain("add_plain encrypted form", x_wrong, p);
    add_plain("add_plain plain form", x, p_ntt);
    add_plain("add_plain both forms", x_wrong, p_ntt);
    auto multiply_plain = [&](const char *what, const Ciphertext &a, const Plaintext &q) {
        check.same(name(what), a, [&](auto &ev, Ciphertext &t) { ev.multiply_plain_inplace(t, q); },
                   [&](seal_b200::CiphertextBatch &d) { auto e = check.up(q); gpu.multiply_plain_inplace(d, e); });
    };
    multiply_plain("multiply_plain parameter mismatch", x, p_ntt_low);
    check.same(name("sub form"), x, [&](auto &ev, Ciphertext &t) { ev.sub_inplace(t, x_wrong); },
               [&](seal_b200::CiphertextBatch &d) { auto e = check.up(x_wrong); gpu.sub_inplace(d, e); });
    RelinKeys rlk_bad = rlk, rlk_none;
    rlk_bad.parms_id() = parms_id_zero;
    rlk_none.parms_id() = context.key_parms_id();
    check.same(name("relinearize form"), m3_wrong, [&](auto &ev, Ciphertext &t) { ev.relinearize_inplace(t, rlk); },
               [&](seal_b200::CiphertextBatch &d) { gpu.relinearize_inplace(d, rlk); });
    // multiply_relinearize_inplace stands for multiply_inplace, then relinearize_inplace
    auto multiply_relinearize = [&](const char *what, const Ciphertext &a, const Ciphertext &b, const RelinKeys &k) {
        check(name(what), a, [&](Ciphertext &t) { ref.multiply_inplace(t, b); ref.relinearize_inplace(t, k); },
              [&](Ciphertext &t) { gpu.multiply_inplace(t, b); gpu.relinearize_inplace(t, k); },
              [&](seal_b200::CiphertextBatch &d) { auto e = check.up(b); gpu.multiply_relinearize_inplace(d, e, k); });
    };
    multiply_relinearize("multiply_relinearize key level", x, y, rlk_bad);
    multiply_relinearize("multiply_relinearize no key", x, y, rlk_none);
    multiply_relinearize("multiply_relinearize form", x_wrong, y, rlk);
    multiply_relinearize("multiply_relinearize key level and form", x_wrong, y, rlk_bad);
    check.same(name("rotate_vector scheme"), x, [&](auto &ev, Ciphertext &t) { ev.rotate_vector_inplace(t, 1, glk); },
               [&](seal_b200::CiphertextBatch &d) { gpu.rotate_vector_inplace(d, 1, glk); });
    check.same(name("rotate_rows missing key"), x, [&](auto &ev, Ciphertext &t) { ev.rotate_rows_inplace(t, 2, glk); },
               [&](seal_b200::CiphertextBatch &d) { gpu.rotate_rows_inplace(d, 2, glk); });
    check.same(name("rotate_columns missing key"), x, [&](auto &ev, Ciphertext &t) { ev.rotate_columns_inplace(t, glk); },
               [&](seal_b200::CiphertextBatch &d) { gpu.rotate_columns_inplace(d, glk); });
    check.same(name("complex_conjugate scheme"), x, [&](auto &ev, Ciphertext &t) { ev.complex_conjugate_inplace(t, glk); },
               [&](seal_b200::CiphertextBatch &d) { gpu.complex_conjugate_inplace(d, glk); });
    check.same(name("rescale_to_next scheme"), x, [&](auto &ev, Ciphertext &t) { ev.rescale_to_next_inplace(t); },
               [&](seal_b200::CiphertextBatch &d) { gpu.rescale_to_next_inplace(d); });
    check.same(name("rescale_to_next end of chain and scheme"), x_last, [&](auto &ev, Ciphertext &t) { ev.rescale_to_next_inplace(t); },
               [&](seal_b200::CiphertextBatch &d) { gpu.rescale_to_next_inplace(d); });
    check.same(name("mod_switch_to_next form"), x_wrong, [&](auto &ev, Ciphertext &t) { ev.mod_switch_to_next_inplace(t); },
               [&](seal_b200::CiphertextBatch &d) { gpu.mod_switch_to_next_inplace(d); });
    check.same(name("mod_switch_to_next end of chain and form"), x_last_wrong, [&](auto &ev, Ciphertext &t) { ev.mod_switch_to_next_inplace(t); },
               [&](seal_b200::CiphertextBatch &d) { gpu.mod_switch_to_next_inplace(d); });
    check.plain(name("plaintext mod_switch_to_next form"), p, [](auto &ev, auto &q) { ev.mod_switch_to_next_inplace(q); });
    check.plain(name("plaintext mod_switch_to_next end of chain"), p_last, [](auto &ev, auto &q) { ev.mod_switch_to_next_inplace(q); });
    if (!bfv)
        return;
    // parameters without batching: rotations fail on that before they look at the keys
    EncryptionParameters nb(scheme_type::bfv);
    nb.set_poly_modulus_degree(n);
    nb.set_coeff_modulus(CoeffModulus::Create(n, { 30, 30, 40 }));
    nb.set_plain_modulus(1024);
    SEALContext nbc(nb, true, sec_level_type::none);
    KeyGenerator nbk(nbc);
    PublicKey nbpk;
    nbk.create_public_key(nbpk);
    Encryptor nbe(nbc, nbpk);
    seal::Evaluator nbref(nbc);
    seal_b200::Evaluator nbgpu(nbc);
    const Precedence nbcheck{ nbref, nbgpu };
    Plaintext one("1");
    Ciphertext z;
    nbe.encrypt(one, z);
    GaloisKeys none;
    nbcheck.same("BFV rotate_rows without batching", z, [&](auto &ev, Ciphertext &t) { ev.rotate_rows_inplace(t, 1, none); },
                 [&](seal_b200::CiphertextBatch &d) { nbgpu.rotate_rows_inplace(d, 1, none); });
    nbcheck.same("BFV rotate_columns without batching", z, [&](auto &ev, Ciphertext &t) { ev.rotate_columns_inplace(t, none); },
                 [&](seal_b200::CiphertextBatch &d) { nbgpu.rotate_columns_inplace(d, none); });
}

int main()
{
    try
    {
        test_ckks();
        test_bfv();
        test_bgv();
        test_batches_and_keys();
        test_encoder_and_encryptor();
        test_precedence_ckks();
        test_precedence_integer(scheme_type::bfv);
        test_precedence_integer(scheme_type::bgv);
    }
    catch (const std::exception &e)
    {
        std::printf("FAIL: unexpected exception: %s\n", e.what());
        return 2;
    }
    std::printf("%s: %d checks, %d failed\n", g_fail ? "FAIL" : "PASS", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
