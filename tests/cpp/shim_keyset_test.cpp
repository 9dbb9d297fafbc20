// tests/cpp/shim_keyset_test.cpp -- the device key sets (DeviceRelinKeys / DeviceGaloisKeys) and the CiphertextBatch streams of
// seal_b200::Evaluator and seal_b200::KeyGenerator (include/seal_b200/evaluator.hpp, keygenerator.hpp) against the seal:: classes:
//   * every batch member that switches keys, with device keys, against seal::Evaluator with host keys: words, metadata, exception
//     types and messages (missing key, the NAF fallback, keys of a foreign parms_id);
//   * key sets uploaded from seal:: objects and loaded from none, zlib and seeded streams, a chosen subset of Galois keys;
//   * KeyGenerator's device overloads under seeded Blake2xb and Shake256 factories against its seal:: overloads, by key switching;
//   * batch load of Ciphertext::save (none, zlib) and encrypt_symmetric (seeded) streams against seal::Ciphertext::load, batch save
//     bytes against seal::Ciphertext::save, and the mixed-metadata and corrupt-stream errors.
// Built by oracle/keyset.mk into oracle/_ref/bin/shim_keyset_test; run by tests/test_gpu_keyset_load.py.
//   shim_keyset_test                   the checks
//   shim_keyset_test --bench [n B]     wall time of loading B seeded ciphertext streams into a batch against seal::Ciphertext::load
//                                      plus Evaluator::upload (defaults 32768 64)
#include "seal/seal.h"
#include "seal_b200/evaluator.hpp"
#include "seal_b200/keygenerator.hpp"
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
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

// same exception type, and the same message unless type_only
static void same_throw(const std::function<void()> &ours, const std::function<void()> &theirs, const char *what, bool type_only = false)
{
    std::string m1, m2;
    const std::string t1 = caught(ours, &m1), t2 = caught(theirs, &m2);
    g_checks++;
    if (t1 != t2 || (!type_only && m1 != m2) || t1 == "none")
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
           a.dyn_array().size() == b.dyn_array().size() && std::memcmp(a.data(), b.data(), a.dyn_array().size() * sizeof(uint64_t)) == 0;
}

static void same_batch(const seal_b200::Evaluator &ev, const seal_b200::CiphertextBatch &b, const std::vector<Ciphertext> &want, const std::string &what)
{
    std::vector<Ciphertext> got;
    ev.download(b, got);
    g_checks++;
    bool ok = got.size() == want.size();
    for (size_t i = 0; ok && i < got.size(); i++)
        ok = same_ct(got[i], want[i]);
    if (!ok)
    {
        g_fail++;
        std::printf("FAIL %s: batch differs from the reference\n", what.c_str());
    }
}

template <class T>
static std::vector<seal_byte> bytes_of(const T &obj, compr_mode_type mode)
{
    std::vector<seal_byte> b(static_cast<size_t>(obj.save_size(mode)));
    b.resize(static_cast<size_t>(obj.save(b.data(), b.size(), mode)));
    return b;
}

static EncryptionParameters params(scheme_type scheme, size_t n, const std::vector<int> &bits, std::shared_ptr<UniformRandomGeneratorFactory> f = nullptr)
{
    EncryptionParameters parms(scheme);
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::Create(n, bits));
    if (scheme != scheme_type::ckks)
        parms.set_plain_modulus(PlainModulus::Batching(n, 20));
    if (f)
        parms.set_random_generator(f);
    return parms;
}

static std::vector<Ciphertext> encrypt_some(const SEALContext &context, Encryptor &enc, size_t B, std::mt19937_64 &rng)
{
    const auto &parms = context.first_context_data()->parms();
    std::vector<Ciphertext> cts(B);
    for (auto &c : cts)
    {
        Plaintext p;
        if (parms.scheme() == scheme_type::ckks)
        {
            CKKSEncoder e(context);
            std::vector<double> v(parms.poly_modulus_degree() / 2);
            for (auto &x : v)
                x = static_cast<double>(rng() % 1000) / 1000.0;
            e.encode(v, std::pow(2.0, 30), p);
        }
        else
        {
            p.resize(parms.poly_modulus_degree());
            for (size_t i = 0; i < parms.poly_modulus_degree(); i++)
                p[i] = rng() % parms.plain_modulus().value();
        }
        enc.encrypt(p, c);
    }
    return cts;
}

// every key-switching batch member with device keys against seal::Evaluator with host keys, for one scheme
static void evaluator_checks(scheme_type scheme, const char *name)
{
    const size_t n = 4096, B = 3;
    SEALContext context(params(scheme, n, { 40, 30, 30, 40 }), true, sec_level_type::none);
    KeyGenerator keygen(context);
    PublicKey pk;
    keygen.create_public_key(pk);
    RelinKeys rk;
    keygen.create_relin_keys(rk);
    GaloisKeys gk; // steps 1, -1, 2, 4, -4 and the column / conjugation element: rotations by 3 and 5 take the NAF fallback, 7 fails
    keygen.create_galois_keys(std::vector<int>{ 1, -1, 2, 4, -4, 0 }, gk);
    Encryptor enc(context, pk);
    seal::Evaluator rev(context);
    seal_b200::Evaluator ev(context);
    const bool ckks = scheme == scheme_type::ckks;
    std::mt19937_64 rng(11);
    std::string what = std::string(name) + ": ";

    // four ways to the same device keys: upload, and none / zlib / subset loads of the reference's streams
    seal_b200::DeviceRelinKeys drk, drk_z;
    seal_b200::DeviceGaloisKeys dgk, dgk_n, dgk_sub;
    ev.upload(rk, drk);
    ev.upload(gk, dgk);
    auto rk_z = bytes_of(rk, compr_mode_type::zlib);
    auto gk_n = bytes_of(gk, compr_mode_type::none);
    ev.load(rk_z.data(), rk_z.size(), drk_z);
    ev.load(gk_n.data(), gk_n.size(), dgk_n);
    const auto *tool = context.key_context_data()->galois_tool();
    const uint32_t e1 = tool->get_elt_from_step(1), e4 = tool->get_elt_from_step(4), em1 = tool->get_elt_from_step(-1);
    auto gk_z = bytes_of(gk, compr_mode_type::zlib);
    ev.load(gk_z.data(), gk_z.size(), std::vector<uint32_t>{ e4, em1, e1, e4 }, dgk_sub);
    CHECK(drk.size() == rk.size() && drk_z.size() == rk.size() && drk.has_key(2) && !drk.has_key(3));
    CHECK(dgk.size() == gk.size() && dgk_n.size() == gk.size() && dgk_sub.size() == 3);
    CHECK(dgk_sub.has_key(e1) && dgk_sub.has_key(e4) && !dgk_sub.has_key(tool->get_elt_from_step(2)));
    CHECK(drk.parms_id() == context.key_parms_id() && dgk_sub.parms_id() == context.key_parms_id());
    CHECK(drk.device_bytes() > 0 && dgk.device_bytes() == gk.size() * drk.device_bytes());
    CHECK(caught([&] { ev.load(gk_z.data(), gk_z.size(), std::vector<uint32_t>{ tool->get_elt_from_step(8) }, dgk_sub); }) ==
          typeid(std::invalid_argument).name());
    CHECK(dgk_sub.size() == 3); // unchanged by the failed load

    const auto cts = encrypt_some(context, enc, B, rng);
    seal_b200::CiphertextBatch b;
    // relinearize_inplace and multiply_relinearize_inplace
    for (auto *keys : { &drk, &drk_z })
    {
        std::vector<Ciphertext> want = cts;
        for (auto &c : want)
            rev.multiply_inplace(c, c), rev.relinearize_inplace(c, rk);
        ev.upload(cts, b);
        ev.multiply_inplace(b, b);
        ev.relinearize_inplace(b, *keys);
        same_batch(ev, b, want, what + "relinearize");
        seal_b200::CiphertextBatch o;
        ev.upload(cts, b), ev.upload(cts, o);
        ev.multiply_relinearize_inplace(b, o, *keys);
        same_batch(ev, b, want, what + "multiply_relinearize");
    }
    // rotations, with every device key set that holds the keys
    auto rot = [&](const seal_b200::DeviceGaloisKeys &keys, int steps, const char *tag) {
        std::vector<Ciphertext> want = cts;
        for (auto &c : want)
            ckks ? rev.rotate_vector_inplace(c, steps, gk) : rev.rotate_rows_inplace(c, steps, gk);
        ev.upload(cts, b);
        ckks ? ev.rotate_vector_inplace(b, steps, keys) : ev.rotate_rows_inplace(b, steps, keys);
        same_batch(ev, b, want, what + tag + " steps " + std::to_string(steps));
    };
    for (int steps : { 1, -1, 3, 5, -4 })
        rot(dgk, steps, "rotate"), rot(dgk_n, steps, "rotate (none stream)");
    rot(dgk_sub, 3, "rotate (subset)");
    {
        std::vector<Ciphertext> want = cts;
        for (auto &c : want)
            ckks ? rev.complex_conjugate_inplace(c, gk) : rev.rotate_columns_inplace(c, gk);
        ev.upload(cts, b);
        ckks ? ev.complex_conjugate_inplace(b, dgk) : ev.rotate_columns_inplace(b, dgk);
        same_batch(ev, b, want, what + "conjugate / rotate_columns");
        want = cts;
        for (auto &c : want)
            rev.apply_galois_inplace(c, e4, gk);
        ev.upload(cts, b);
        ev.apply_galois_inplace(b, e4, dgk_sub);
        same_batch(ev, b, want, what + "apply_galois");
    }
    // multiply_many and exponentiate (BFV / BGV)
    if (!ckks)
    {
        std::vector<std::vector<Ciphertext>> ops(3);
        for (auto &o : ops)
            o = encrypt_some(context, enc, B, rng);
        std::vector<Ciphertext> want(B);
        for (size_t i = 0; i < B; i++)
            rev.multiply_many({ ops[0][i], ops[1][i], ops[2][i] }, rk, want[i]);
        std::vector<seal_b200::CiphertextBatch> bs(3);
        for (size_t j = 0; j < 3; j++)
            ev.upload(ops[j], bs[j]);
        ev.multiply_many(bs, drk, b);
        same_batch(ev, b, want, what + "multiply_many");
        want = cts;
        for (auto &c : want)
            rev.exponentiate_inplace(c, 5, rk);
        ev.upload(cts, b);
        ev.exponentiate_inplace(b, 5, drk);
        same_batch(ev, b, want, what + "exponentiate_inplace");
        seal_b200::CiphertextBatch d;
        ev.upload(cts, b);
        ev.exponentiate(b, 5, drk_z, d);
        same_batch(ev, d, want, what + "exponentiate");
    }
    // the exceptions of the seal:: overloads
    Ciphertext one = cts[0];
    ev.upload(cts, b);
    same_throw([&] { ckks ? ev.rotate_vector_inplace(b, 7, dgk) : ev.rotate_rows_inplace(b, 7, dgk); },
               [&] { ckks ? rev.rotate_vector_inplace(one, 7, gk) : rev.rotate_rows_inplace(one, 7, gk); }, "missing key (NAF)");
    same_throw([&] { ev.apply_galois_inplace(b, tool->get_elt_from_step(2), dgk_sub); },
               [&] { rev.apply_galois_inplace(one, tool->get_elt_from_step(2), GaloisKeys()); }, "missing key", true);
    SEALContext other(params(scheme, n, { 40, 30, 40 }), true, sec_level_type::none);
    KeyGenerator okg(other);
    RelinKeys ork;
    GaloisKeys ogk;
    okg.create_relin_keys(ork);
    okg.create_galois_keys(std::vector<int>{ 1 }, ogk);
    seal_b200::Evaluator oev(other);
    seal_b200::DeviceRelinKeys fdrk;
    seal_b200::DeviceGaloisKeys fdgk;
    oev.upload(ork, fdrk);
    oev.upload(ogk, fdgk);
    same_throw([&] { ev.apply_galois_inplace(b, e1, fdgk); }, [&] { rev.apply_galois_inplace(one, e1, ogk); }, "foreign galois keys");
    same_throw([&] { ckks ? ev.rotate_vector_inplace(b, 1, fdgk) : ev.rotate_rows_inplace(b, 1, fdgk); },
               [&] { ckks ? rev.rotate_vector_inplace(one, 1, ogk) : rev.rotate_rows_inplace(one, 1, ogk); }, "foreign galois keys (rotate)");
    Ciphertext sq = cts[0];
    rev.multiply_inplace(sq, sq);
    ev.multiply_inplace(b, b);
    same_throw([&] { ev.relinearize_inplace(b, fdrk); }, [&] { rev.relinearize_inplace(sq, ork); }, "foreign relin keys");
    same_throw([&] { ev.upload(ork, fdrk); }, [&] { rev.relinearize_inplace(sq, ork); }, "upload of foreign keys", true);
    // keys of another device context with the same parameters
    seal_b200::Evaluator ev2(context);
    seal_b200::DeviceRelinKeys other_ctx;
    ev2.upload(rk, other_ctx);
    CHECK(caught([&] { ev.relinearize_inplace(b, other_ctx); }) == typeid(std::invalid_argument).name());
    // KeyGenerator's device overloads, same parameters: they do not touch the Evaluator's key cache
    CHECK(ev.key_cache_entries() == 0);
}

// KeyGenerator's device overloads under a seeded factory: the same draws as its seal:: overloads, so the same keys
static void keygen_checks(std::shared_ptr<UniformRandomGeneratorFactory> factory, const char *name)
{
    const size_t n = 4096, B = 2;
    SEALContext context(params(scheme_type::bgv, n, { 40, 30, 30, 40 }, factory), true, sec_level_type::none);
    KeyGenerator sk_gen(context);
    seal_b200::Evaluator ev(context);
    seal_b200::KeyGenerator kg(context, sk_gen.secret_key(), ev);
    RelinKeys rk;
    GaloisKeys gk;
    seal_b200::DeviceRelinKeys drk;
    seal_b200::DeviceGaloisKeys dgk, dgk_all;
    kg.create_relin_keys(rk);
    kg.create_relin_keys(drk);
    kg.create_galois_keys(std::vector<int>{ 1, -2 }, gk);
    kg.create_galois_keys(std::vector<int>{ 1, -2 }, dgk);
    kg.create_galois_keys(dgk_all);
    auto all = context.key_context_data()->galois_tool()->get_elts_all(); // lists the element of order 2 twice
    std::sort(all.begin(), all.end());
    all.erase(std::unique(all.begin(), all.end()), all.end());
    CHECK(drk.size() == 1 && dgk.size() == 2 && dgk_all.size() == all.size());
    PublicKey pk;
    sk_gen.create_public_key(pk);
    Encryptor enc(context, pk);
    seal::Evaluator rev(context);
    std::mt19937_64 rng(5);
    const auto cts = encrypt_some(context, enc, B, rng);
    std::vector<Ciphertext> want = cts;
    for (auto &c : want)
        rev.multiply_inplace(c, c), rev.relinearize_inplace(c, rk), rev.rotate_rows_inplace(c, -2, gk), rev.rotate_rows_inplace(c, 1, gk);
    seal_b200::CiphertextBatch b;
    ev.upload(cts, b);
    ev.multiply_inplace(b, b);
    ev.relinearize_inplace(b, drk);
    ev.rotate_rows_inplace(b, -2, dgk);
    ev.rotate_rows_inplace(b, 1, dgk_all);
    same_batch(ev, b, want, std::string(name) + ": KeyGenerator device keys");
    CHECK(caught([&] { kg.create_galois_keys(std::vector<uint32_t>{ 3, 4 }, dgk); }) == typeid(std::invalid_argument).name());
    CHECK(dgk.size() == 2);
}

// batch load and save against seal::Ciphertext::load / save
static void stream_checks(scheme_type scheme, const char *name)
{
    const size_t n = 4096, B = 4;
    SEALContext context(params(scheme, n, { 40, 30, 30, 40 }), true, sec_level_type::none);
    KeyGenerator keygen(context);
    PublicKey pk;
    keygen.create_public_key(pk);
    Encryptor enc(context, pk), senc(context, keygen.secret_key());
    seal::Evaluator rev(context);
    seal_b200::Evaluator ev(context);
    std::mt19937_64 rng(3);
    std::string what = std::string(name) + ": ";
    auto cts = encrypt_some(context, enc, B, rng);
    for (auto &c : cts)
        rev.multiply_inplace(c, c); // size 3, with a CKKS scale and a BGV correction factor that differ from 1
    for (compr_mode_type mode : { compr_mode_type::none, compr_mode_type::zlib })
    {
        std::vector<std::vector<seal_byte>> streams;
        std::vector<const seal_byte *> ptrs;
        std::vector<size_t> sizes;
        for (auto &c : cts)
            streams.push_back(bytes_of(c, mode));
        for (auto &s : streams)
            ptrs.push_back(s.data()), sizes.push_back(s.size());
        seal_b200::CiphertextBatch b;
        ev.load(ptrs.data(), sizes.data(), B, b);
        std::vector<Ciphertext> want(B);
        for (size_t i = 0; i < B; i++)
            want[i].load(context, streams[i].data(), streams[i].size());
        same_batch(ev, b, want, what + "load " + std::to_string(static_cast<int>(mode)));
        ev.unsafe_load(ptrs.data(), sizes.data(), B, b);
        same_batch(ev, b, want, what + "unsafe_load");
        std::vector<std::vector<seal_byte>> saved;
        ev.save(b, saved, mode);
        CHECK(saved == streams);
        CHECK(ev.save_size(b, mode) == cts[0].save_size(mode));
    }
    // seeded streams of encrypt_symmetric
    std::vector<std::vector<seal_byte>> seeded;
    std::vector<const seal_byte *> ptrs;
    std::vector<size_t> sizes;
    for (size_t i = 0; i < B; i++)
    {
        Plaintext p(n);
        for (size_t j = 0; j < n; j++)
            p[j] = scheme == scheme_type::ckks ? 0 : rng() % context.first_context_data()->parms().plain_modulus().value();
        if (scheme == scheme_type::ckks)
        {
            CKKSEncoder e(context);
            e.encode(0.25, std::pow(2.0, 30), p);
        }
        seeded.push_back(bytes_of(senc.encrypt_symmetric(p), compr_mode_type::none));
    }
    for (auto &s : seeded)
        ptrs.push_back(s.data()), sizes.push_back(s.size());
    seal_b200::CiphertextBatch b;
    ev.load(ptrs.data(), sizes.data(), B, b);
    std::vector<Ciphertext> want(B);
    for (size_t i = 0; i < B; i++)
        want[i].load(context, seeded[i].data(), seeded[i].size());
    same_batch(ev, b, want, what + "seeded load");
    // mixed metadata: nothing is written
    Ciphertext low = want[1];
    rev.mod_switch_to_next_inplace(low);
    auto low_s = bytes_of(low, compr_mode_type::none);
    std::vector<const seal_byte *> mixed = { seeded[0].data(), low_s.data() };
    std::vector<size_t> mixed_sizes = { seeded[0].size(), low_s.size() };
    CHECK(caught([&] { ev.load(mixed.data(), mixed_sizes.data(), 2, b); }) == typeid(std::invalid_argument).name());
    same_batch(ev, b, want, what + "batch unchanged after a mixed-metadata load");
    // corrupt streams: what seal::Ciphertext::load throws
    auto bad = seeded[0];
    bad[0] = seal_byte{ 0 }; // header magic
    const seal_byte *bp = bad.data();
    size_t bs = bad.size();
    Ciphertext sink;
    same_throw([&] { ev.load(&bp, &bs, 1, b); }, [&] { sink.load(context, bad.data(), bad.size()); }, "corrupt header", true);
    auto big = bytes_of(cts[0], compr_mode_type::none);
    std::memset(big.data() + big.size() - 8, 0xFF, 8); // a word >= q
    bp = big.data(), bs = big.size();
    same_throw([&] { ev.load(&bp, &bs, 1, b); }, [&] { sink.load(context, big.data(), big.size()); }, "word out of range", true);
    same_batch(ev, b, want, what + "batch unchanged after a corrupt load");
}

static int bench(size_t n, size_t B)
{
    std::vector<int> bits(16, 50);
    SEALContext context(params(scheme_type::ckks, n, bits), true, sec_level_type::none);
    KeyGenerator keygen(context);
    Encryptor senc(context, keygen.secret_key());
    seal_b200::Evaluator ev(context);
    std::vector<std::vector<seal_byte>> streams;
    std::vector<const seal_byte *> ptrs;
    std::vector<size_t> sizes;
    for (size_t i = 0; i < B; i++)
        streams.push_back(bytes_of(senc.encrypt_zero_symmetric(), compr_mode_type::none));
    for (auto &s : streams)
        ptrs.push_back(s.data()), sizes.push_back(s.size());
    seal_b200::CiphertextBatch b;
    using clk = std::chrono::steady_clock;
    double best_dev = 1e30, best_ref = 1e30;
    for (int rep = 0; rep < 4; rep++)
    {
        auto t0 = clk::now();
        ev.load(ptrs.data(), sizes.data(), B, b);
        ev.synchronize();
        auto t1 = clk::now();
        std::vector<Ciphertext> cts(B);
        for (size_t i = 0; i < B; i++)
            cts[i].load(context, streams[i].data(), streams[i].size());
        ev.upload(cts, b);
        ev.synchronize();
        auto t2 = clk::now();
        if (rep) // the first round warms up the allocations
        {
            best_dev = std::min(best_dev, std::chrono::duration<double, std::milli>(t1 - t0).count());
            best_ref = std::min(best_ref, std::chrono::duration<double, std::milli>(t2 - t1).count());
        }
    }
    std::printf("BENCH batch load of %zu seeded ciphertexts, n = %zu, 16 primes: device %.1f ms, seal::Ciphertext::load + upload %.1f ms\n", B, n,
                best_dev, best_ref);
    return 0;
}

int main(int argc, char **argv)
{
    if (argc > 1 && std::strcmp(argv[1], "--bench") == 0)
        return bench(argc > 2 ? std::strtoul(argv[2], nullptr, 10) : 32768, argc > 3 ? std::strtoul(argv[3], nullptr, 10) : 64);
    evaluator_checks(scheme_type::bfv, "BFV");
    evaluator_checks(scheme_type::bgv, "BGV");
    evaluator_checks(scheme_type::ckks, "CKKS");
    prng_seed_type seed{};
    seed[0] = 0x5EED;
    keygen_checks(std::make_shared<Blake2xbPRNGFactory>(seed), "Blake2xb");
    keygen_checks(std::make_shared<Shake256PRNGFactory>(seed), "Shake256");
    stream_checks(scheme_type::bfv, "BFV");
    stream_checks(scheme_type::bgv, "BGV");
    stream_checks(scheme_type::ckks, "CKKS");
    std::printf("%d checks, %d failed\n", g_checks, g_fail);
    std::printf(g_fail ? "FAIL\n" : "PASS\n");
    return g_fail ? 1 : 0;
}
