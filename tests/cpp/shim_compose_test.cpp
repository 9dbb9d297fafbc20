// tests/cpp/shim_compose_test.cpp -- the composition members of seal_b200::Evaluator on CiphertextBatch (add_inplace / sub_inplace
// across sizes and correction factors, add_many, multiply_many, exponentiate, mod_switch_to / rescale_to; include/seal_b200/evaluator.hpp)
// against seal::Evaluator on the same seal::Ciphertexts: words and metadata of every member, exception types and messages, and the
// number of key-switching passes and products of multiply_many / exponentiate.
// Built by oracle/compose.mk into oracle/_ref/bin/shim_compose_test; run by tests/test_gpu_compositions.py.
//   shim_compose_test            the checks
//   shim_compose_test --bench [n primes m batch]
//                                wall time of multiply_many and exponentiate(16) on batches against the same products made one
//                                multiply_relinearize_inplace call per pair in the reference's order (defaults 65536 32 16 64)
#include "seal/seal.h"
#include "seal_b200/evaluator.hpp"
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
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
           a.dyn_array().size() == b.dyn_array().size() && std::memcmp(a.data(), b.data(), a.dyn_array().size() * sizeof(uint64_t)) == 0;
}

static void same_batch(const seal_b200::Evaluator &ev, const seal_b200::CiphertextBatch &b, const std::vector<Ciphertext> &want, const std::string &what)
{
    std::vector<Ciphertext> got;
    ev.download(b, got);
    CHECK(got.size() == want.size());
    for (size_t i = 0; i < got.size() && i < want.size(); i++)
        if (!same_ct(got[i], want[i]))
        {
            g_checks++, g_fail++;
            std::printf("FAIL %s: ciphertext %zu differs\n", what.c_str(), i);
            return;
        }
    g_checks++;
}

// member i of every operand
static std::vector<Ciphertext> column(const std::vector<std::vector<Ciphertext>> &ops, size_t i)
{
    std::vector<Ciphertext> c;
    for (auto &o : ops)
        c.push_back(o[i]);
    return c;
}

// launches per kernel name since the last reset
static std::map<std::string, unsigned long long> launches(sb200_context *ctx)
{
    std::map<std::string, unsigned long long> m;
    char name[128];
    double ms = 0, bytes = 0;
    unsigned long long n = 0;
    for (size_t i = 0; sb200_profile_read(ctx, i, name, sizeof(name), &ms, &n, &bytes) == SB200_OK; i++)
        m[name] += n;
    return m;
}

// SEAL's multiply_many loop (evaluator.cpp:1649-1724) replayed literally on leaf ids, O(m): the distinct products (hash-consed on
// (left, right)) and the number of dependency levels among them
static void replay(const std::vector<size_t> &leaf_ids, size_t &distinct, size_t &waves)
{
    std::map<std::pair<size_t, size_t>, size_t> made;
    std::map<size_t, size_t> depth; // id -> depth
    size_t next = 1000000;
    for (size_t id : leaf_ids)
        depth[id] = 0;
    auto mul = [&](size_t a, size_t b) {
        auto it = made.find({ a, b });
        if (it != made.end())
            return it->second;
        const size_t id = next++;
        depth[id] = std::max(depth[a], depth[b]) + 1;
        return made[{ a, b }] = id;
    };
    std::vector<size_t> products;
    for (size_t i = 0; i + 1 < leaf_ids.size(); i += 2)
        products.push_back(mul(leaf_ids[i], leaf_ids[i + 1]));
    if (leaf_ids.size() & 1)
        products.push_back(leaf_ids.back());
    for (size_t i = 0; i + 1 < products.size(); i += 2)
        products.push_back(mul(products[i], products[i + 1]));
    distinct = made.size();
    waves = 0;
    for (auto &kv : made)
        waves = std::max(waves, depth[kv.second]);
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
    explicit Setup(const EncryptionParameters &parms)
        : context(parms, true, sec_level_type::none), keygen(context), pk(make_pk(keygen)), rk(make_rk(keygen)), enc(context, pk), rev(context),
          ev(context)
    {}
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

static std::vector<Ciphertext> encrypt_some(Setup &s, size_t B, std::mt19937_64 &rng, double scale = 0)
{
    std::vector<Ciphertext> cts(B);
    const auto &parms = s.context.first_context_data()->parms();
    for (auto &c : cts)
    {
        Plaintext p;
        if (parms.scheme() == scheme_type::ckks)
        {
            CKKSEncoder e(s.context);
            std::vector<double> v(parms.poly_modulus_degree() / 2);
            for (auto &x : v)
                x = static_cast<double>(rng() % 1000) / 1000.0;
            e.encode(v, scale, p);
        }
        else
        {
            p.resize(parms.poly_modulus_degree());
            for (size_t i = 0; i < parms.poly_modulus_degree(); i++)
                p[i] = rng() % parms.plain_modulus().value();
        }
        s.enc.encrypt(p, c);
    }
    return cts;
}

// a chain of add / sub steps and add_many over operands of mixed sizes (and, for BGV, mixed correction factors)
static void linear_checks(Setup &s, const char *name, double scale)
{
    std::mt19937_64 rng(7);
    const size_t B = 3;
    const bool ckks = s.context.first_context_data()->parms().scheme() == scheme_type::ckks;
    const bool bgv = s.context.first_context_data()->parms().scheme() == scheme_type::bgv;
    auto fresh = [&] { return encrypt_some(s, B, rng, scale); };
    // operands at the second level: size 2, size 3 (an unrelinearized square), size 4 (a cube); BGV factors differ after
    // mod_switch_to_next and a square of it
    auto at_level2 = [&](size_t size) {
        std::vector<Ciphertext> c = fresh();
        for (auto &x : c)
        {
            if (size >= 3)
            {
                Ciphertext y = x;
                s.rev.multiply_inplace(x, y);
                if (size == 4)
                    s.rev.multiply_inplace(x, y);
            }
            if (ckks)
                s.rev.rescale_to_next_inplace(x), x.scale() = scale;
            else
                s.rev.mod_switch_to_next_inplace(x);
        }
        return c;
    };
    std::vector<std::vector<Ciphertext>> ops = { at_level2(2), at_level2(3), at_level2(4), at_level2(2), at_level2(3) };
    if (bgv)
    {
        // a fresh encryption of zero at the same level keeps correction factor 1
        std::vector<Ciphertext> z(B);
        for (auto &c : z)
            s.enc.encrypt_zero(ops[0][0].parms_id(), c);
        ops.push_back(z);
        CHECK(ops[0][0].correction_factor() != 1);
    }
    std::vector<seal_b200::CiphertextBatch> d(ops.size());
    for (size_t j = 0; j < ops.size(); j++)
        s.ev.upload(ops[j], d[j]);

    // add / sub in both size orders (the longer operand's tail copied or negated), with balancing where factors differ
    for (size_t a = 0; a < ops.size(); a++)
        for (size_t b = 0; b < ops.size(); b++)
            for (int sub = 0; sub < 2; sub++)
            {
                if (a == b)
                    continue;
                seal_b200::CiphertextBatch x;
                s.ev.copy(d[a], x);
                std::vector<Ciphertext> want = ops[a];
                for (size_t i = 0; i < B; i++)
                    sub ? s.rev.sub_inplace(want[i], ops[b][i]) : s.rev.add_inplace(want[i], ops[b][i]);
                sub ? s.ev.sub_inplace(x, d[b]) : s.ev.add_inplace(x, d[b]);
                same_batch(s.ev, x, want, std::string(name) + (sub ? " sub " : " add ") + std::to_string(a) + "," + std::to_string(b));
            }
    // x + x and x - x through one object
    {
        seal_b200::CiphertextBatch x;
        s.ev.copy(d[1], x);
        std::vector<Ciphertext> want = ops[1];
        for (auto &w : want)
            s.rev.add_inplace(w, w);
        s.ev.add_inplace(x, x);
        same_batch(s.ev, x, want, std::string(name) + " add to itself");
    }
    // add_many of 1 .. all operands, in both orders
    for (int rev_order = 0; rev_order < 2; rev_order++)
        for (size_t m = 1; m <= ops.size(); m++)
        {
            std::vector<seal_b200::CiphertextBatch> sel(m);
            std::vector<std::vector<Ciphertext>> sel_ct;
            for (size_t j = 0; j < m; j++)
            {
                const size_t k = rev_order ? ops.size() - 1 - j : j;
                s.ev.copy(d[k], sel[j]);
                sel_ct.push_back(ops[k]);
            }
            seal_b200::CiphertextBatch out;
            s.ev.add_many(sel, out);
            std::vector<Ciphertext> want(B);
            for (size_t i = 0; i < B; i++)
                s.rev.add_many(column(sel_ct, i), want[i]);
            same_batch(s.ev, out, want, std::string(name) + " add_many m=" + std::to_string(m) + (rev_order ? " reversed" : ""));
        }
    // errors, before anything is written
    {
        Ciphertext r0 = ops[0][0], r1 = fresh()[0], rdst;
        seal_b200::CiphertextBatch top, x;
        s.ev.upload(std::vector<Ciphertext>{ r1 }, top);
        seal_b200::CiphertextBatch one;
        s.ev.upload(std::vector<Ciphertext>{ r0 }, one);
        same_throw([&] { s.ev.add_inplace(one, top); }, [&] { s.rev.add_inplace(r0, r1); }, "add parameter mismatch");
        same_throw([&] { s.ev.sub_inplace(one, top); }, [&] { s.rev.sub_inplace(r0, r1); }, "sub parameter mismatch");
        same_throw([&] { s.ev.add_many({}, x); }, [&] { s.rev.add_many({}, rdst); }, "add_many empty");
        std::vector<Ciphertext> rv = { r0, r0 };
        same_throw([&] { s.ev.add_many(d, d[0]); }, [&] { s.rev.add_many(rv, rv[1]); }, "add_many destination among operands");
        std::vector<seal_b200::CiphertextBatch> mixed(2);
        s.ev.copy(one, mixed[0]);
        s.ev.copy(top, mixed[1]);
        same_throw([&] { s.ev.add_many(mixed, x); }, [&] { s.rev.add_many({ r0, r1 }, rdst); }, "add_many parameter mismatch");
        if (ckks)
        {
            Ciphertext r2 = r0;
            r2.scale() *= 2;
            seal_b200::CiphertextBatch sc;
            s.ev.upload(std::vector<Ciphertext>{ r2 }, sc);
            same_throw([&] { s.ev.add_inplace(one, sc); }, [&] { s.rev.add_inplace(r0, r2); }, "add scale mismatch");
            Ciphertext r3 = r0;
            s.rev.transform_from_ntt_inplace(r3);
            seal_b200::CiphertextBatch nt;
            s.ev.upload(std::vector<Ciphertext>{ r3 }, nt);
            same_throw([&] { s.ev.add_inplace(one, nt); }, [&] { s.rev.add_inplace(r0, r3); }, "add NTT form mismatch");
        }
        std::vector<Ciphertext> got;
        s.ev.download(one, got);
        CHECK(same_ct(got[0], ops[0][0]));
    }
    // mod_switch_to / rescale_to the last level
    {
        const auto last = s.context.last_parms_id();
        std::vector<Ciphertext> c = fresh();
        seal_b200::CiphertextBatch x;
        s.ev.upload(c, x);
        std::vector<Ciphertext> want = c;
        for (auto &w : want)
            s.rev.mod_switch_to_inplace(w, last);
        seal_b200::CiphertextBatch y;
        s.ev.copy(x, y);
        s.ev.mod_switch_to_inplace(y, last);
        same_batch(s.ev, y, want, std::string(name) + " mod_switch_to");
        same_throw([&] { s.ev.mod_switch_to_inplace(y, s.context.first_parms_id()); },
                   [&] { s.rev.mod_switch_to_inplace(want[0], s.context.first_parms_id()); }, "mod_switch_to a higher level");
        if (ckks)
        {
            std::vector<Ciphertext> sq = c;
            for (auto &w : sq)
                s.rev.square_inplace(w), s.rev.relinearize_inplace(w, s.rk);
            seal_b200::CiphertextBatch z;
            s.ev.upload(sq, z);
            const auto to = s.context.first_context_data()->next_context_data()->parms_id();
            for (auto &w : sq)
                s.rev.rescale_to_inplace(w, to);
            s.ev.rescale_to_inplace(z, to);
            same_batch(s.ev, z, sq, std::string(name) + " rescale_to");
        }
        else
        {
            Ciphertext r = c[0];
            same_throw([&] { s.ev.rescale_to_inplace(x, last); }, [&] { s.rev.rescale_to_inplace(r, last); }, "rescale_to of a non-CKKS scheme");
        }
    }
}

// multiply_many with m = 1 .. 9 (some operands equal in value) and exponentiate, words, metadata and pass counts
static void product_checks(Setup &s, const char *name)
{
    std::mt19937_64 rng(9);
    const size_t B = 2;
    sb200_context *ctx = s.ev.native_handle();
    sb200_profile_enable(ctx, 1);
    std::vector<std::vector<Ciphertext>> pool;
    for (int j = 0; j < 5; j++)
        pool.push_back(encrypt_some(s, B, rng));
    // a kernel that runs once per key-switching call of one chunk: calibrated on one multiply_relinearize_inplace
    std::string pass_kernel;
    {
        seal_b200::CiphertextBatch a, b;
        s.ev.upload(pool[0], a), s.ev.upload(pool[1], b);
        s.ev.synchronize();
        sb200_profile_reset(ctx);
        s.ev.multiply_relinearize_inplace(a, b, s.rk);
        s.ev.synchronize();
        for (auto &kv : launches(ctx))
            if (kv.second == 1 && pass_kernel.empty())
                pass_kernel = kv.first;
        CHECK(!pass_kernel.empty());
    }
    for (size_t m = 1; m <= 9; m++)
    {
        std::vector<std::vector<Ciphertext>> ops;
        std::vector<size_t> ids;
        for (size_t j = 0; j < m; j++)
        {
            ops.push_back(pool[(j * 3) % pool.size()]); // operands repeat in value
            ids.push_back(j);
        }
        std::vector<seal_b200::CiphertextBatch> d(m);
        for (size_t j = 0; j < m; j++)
            s.ev.upload(ops[j], d[j]);
        s.ev.synchronize();
        sb200_profile_reset(ctx);
        seal_b200::CiphertextBatch out;
        s.ev.multiply_many(d, s.rk, out);
        s.ev.synchronize();
        std::vector<Ciphertext> want(B);
        for (size_t i = 0; i < B; i++)
            s.rev.multiply_many(column(ops, i), s.rk, want[i]);
        same_batch(s.ev, out, want, std::string(name) + " multiply_many m=" + std::to_string(m));
        size_t distinct = 0, waves = 0;
        replay(ids, distinct, waves);
        CHECK(launches(ctx)[pass_kernel] == waves);
    }
    for (uint64_t e : { 1, 2, 3, 5, 6, 8, 13, 16 })
    {
        seal_b200::CiphertextBatch x;
        s.ev.upload(pool[2], x);
        s.ev.synchronize();
        sb200_profile_reset(ctx);
        s.ev.exponentiate_inplace(x, e, s.rk);
        s.ev.synchronize();
        auto counts = launches(ctx);
        std::vector<Ciphertext> want = pool[2];
        for (auto &w : want)
            s.rev.exponentiate_inplace(w, e, s.rk);
        same_batch(s.ev, x, want, std::string(name) + " exponentiate " + std::to_string(e));
        size_t distinct = 0, waves = 0;
        replay(std::vector<size_t>(e, 0), distinct, waves);
        if (e == 16)
            CHECK(distinct == 4 && waves == 4);
        if (e == 13)
            CHECK(distinct == 5 && waves == 4);
        CHECK(counts[pass_kernel] == waves);
        seal_b200::CiphertextBatch y;
        s.ev.upload(pool[2], y);
        seal_b200::CiphertextBatch z;
        s.ev.exponentiate(y, e, s.rk, z);
        same_batch(s.ev, z, want, std::string(name) + " exponentiate (out of place) " + std::to_string(e));
    }
    // errors
    {
        Ciphertext r = pool[0][0], rdst;
        seal_b200::CiphertextBatch x, dst;
        s.ev.upload(std::vector<Ciphertext>{ r }, x);
        same_throw([&] { s.ev.exponentiate_inplace(x, 0, s.rk); }, [&] { s.rev.exponentiate_inplace(r, 0, s.rk); }, "exponentiate 0");
        same_throw([&] { s.ev.multiply_many({}, s.rk, dst); }, [&] { s.rev.multiply_many({}, s.rk, rdst); }, "multiply_many empty");
        std::vector<seal_b200::CiphertextBatch> two(2);
        s.ev.copy(x, two[0]), s.ev.copy(x, two[1]);
        std::vector<Ciphertext> rtwo = { r, r };
        same_throw([&] { s.ev.multiply_many(two, s.rk, two[1]); }, [&] { s.rev.multiply_many(rtwo, s.rk, rtwo[1]); },
                   "multiply_many destination among operands");
        Ciphertext low = r;
        s.rev.mod_switch_to_next_inplace(low);
        seal_b200::CiphertextBatch xl;
        s.ev.upload(std::vector<Ciphertext>{ low }, xl);
        std::vector<seal_b200::CiphertextBatch> mixed(2);
        s.ev.copy(x, mixed[0]), s.ev.copy(xl, mixed[1]);
        same_throw([&] { s.ev.multiply_many(mixed, s.rk, dst); }, [&] { s.rev.multiply_many({ r, low }, s.rk, rdst); },
                   "multiply_many parameter mismatch");
    }
    sb200_profile_enable(ctx, 0);
}

static void ckks_unsupported()
{
    EncryptionParameters parms(scheme_type::ckks);
    parms.set_poly_modulus_degree(4096);
    parms.set_coeff_modulus(CoeffModulus::Create(4096, { 40, 30, 30, 40 }));
    Setup s(parms);
    std::mt19937_64 rng(3);
    std::vector<Ciphertext> c = encrypt_some(s, 1, rng, std::pow(2.0, 30));
    seal_b200::CiphertextBatch x, dst;
    s.ev.upload(c, x);
    Ciphertext r = c[0], rdst;
    std::vector<seal_b200::CiphertextBatch> two(2);
    s.ev.copy(x, two[0]), s.ev.copy(x, two[1]);
    same_throw([&] { s.ev.multiply_many(two, s.rk, dst); }, [&] { s.rev.multiply_many({ r, r }, s.rk, rdst); }, "CKKS multiply_many");
    same_throw([&] { s.ev.exponentiate_inplace(x, 3, s.rk); }, [&] { s.rev.exponentiate_inplace(r, 3, s.rk); }, "CKKS exponentiate");
    linear_checks(s, "CKKS", std::pow(2.0, 30));
}

static EncryptionParameters integer_parms(scheme_type scheme, size_t n, const std::vector<int> &bits)
{
    EncryptionParameters parms(scheme);
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::Create(n, bits));
    parms.set_plain_modulus(PlainModulus::Batching(n, 20));
    return parms;
}

static int bench(int argc, char **argv)
{
    const size_t n = argc > 2 ? std::strtoul(argv[2], nullptr, 10) : 65536, k = argc > 3 ? std::strtoul(argv[3], nullptr, 10) : 32;
    const size_t m = argc > 4 ? std::strtoul(argv[4], nullptr, 10) : 16, B = argc > 5 ? std::strtoul(argv[5], nullptr, 10) : 64;
    Setup s(integer_parms(scheme_type::bgv, n, std::vector<int>(k, 50)));
    std::mt19937_64 rng(5);
    // the timings do not depend on the words: one encrypted ciphertext fills every member
    std::vector<Ciphertext> one = encrypt_some(s, 1, rng);
    std::vector<Ciphertext> members(B, one[0]);
    std::vector<seal_b200::CiphertextBatch> ops(m);
    for (auto &o : ops)
        s.ev.upload(members, o);
    auto wall = [&](const std::function<void()> &f) {
        f(); // warm-up: key upload, scratch growth
        s.ev.synchronize();
        const auto t0 = std::chrono::steady_clock::now();
        f();
        s.ev.synchronize();
        return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    };
    // the reference's order, one multiply_relinearize_inplace per pair
    auto pairwise = [&](std::vector<const seal_b200::CiphertextBatch *> leaves) {
        std::vector<seal_b200::CiphertextBatch> prods;
        prods.reserve(2 * leaves.size());
        std::vector<const seal_b200::CiphertextBatch *> q;
        for (size_t i = 0; i + 1 < leaves.size(); i += 2)
        {
            prods.emplace_back();
            s.ev.copy(*leaves[i], prods.back());
            s.ev.multiply_relinearize_inplace(prods.back(), *leaves[i + 1], s.rk);
            q.push_back(&prods.back());
        }
        if (leaves.size() & 1)
            q.push_back(leaves.back());
        for (size_t i = 0; i + 1 < q.size(); i += 2)
        {
            prods.emplace_back();
            s.ev.copy(*q[i], prods.back());
            s.ev.multiply_relinearize_inplace(prods.back(), *q[i + 1], s.rk);
            q.push_back(&prods.back());
        }
    };
    std::vector<const seal_b200::CiphertextBatch *> leaves;
    for (auto &o : ops)
        leaves.push_back(&o);
    seal_b200::CiphertextBatch out;
    const double t_many = wall([&] { s.ev.multiply_many(ops, s.rk, out); });
    const double t_pairs = wall([&] { pairwise(leaves); });
    const double t_exp = wall([&] { s.ev.exponentiate(ops[0], 16, s.rk, out); });
    const double t_exp_pairs = wall([&] { pairwise(std::vector<const seal_b200::CiphertextBatch *>(16, &ops[0])); });
    std::printf("{\"n\": %zu, \"primes\": %zu, \"operands\": %zu, \"batch\": %zu, \"multiply_many_ms\": %.2f, \"pairwise_ms\": %.2f, "
                "\"exponentiate16_ms\": %.2f, \"exponentiate16_pairwise_ms\": %.2f}\n",
                n, k, m, B, t_many, t_pairs, t_exp, t_exp_pairs);
    return 0;
}

int main(int argc, char **argv)
{
    if (argc > 1 && std::strcmp(argv[1], "--bench") == 0)
        return bench(argc, argv);
    {
        Setup s(integer_parms(scheme_type::bfv, 4096, { 40, 40, 40, 40 }));
        linear_checks(s, "BFV", 0);
        product_checks(s, "BFV");
    }
    {
        Setup s(integer_parms(scheme_type::bgv, 4096, { 40, 40, 40, 40 }));
        linear_checks(s, "BGV", 0);
        product_checks(s, "BGV");
    }
    ckks_unsupported();
    std::printf("%d checks, %d failures\n", g_checks, g_fail);
    if (g_fail)
        return 1;
    std::printf("shim_compose_test ok\n");
    return 0;
}
