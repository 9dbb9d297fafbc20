// tests/cpp/shim_noise_test.cpp -- seal_b200::Decryptor::invariant_noise_budget (include/seal_b200/decryptor.hpp) against
// seal::Decryptor: the budget along a multiplication chain (BFV, BGV), every exception type and message (CKKS, the wrong NTT form,
// an empty ciphertext), and the CiphertextBatch overloads of invariant_noise_budget and decrypt against the reference applied to the
// downloaded members.  Built by oracle/noise.mk into oracle/_ref/bin/shim_noise_test; run by tests/test_gpu_noise.py.
#include "seal/seal.h"
#include "seal_b200/decryptor.hpp"
#include <cmath>
#include <cstdio>
#include <cstring>
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

// the exception both throw: same type, same message
template <class F, class G>
static void same_throw(F ours, G theirs, const char *what)
{
    std::string t1 = "none", m1, t2 = "none", m2;
    try
    {
        ours();
    }
    catch (const std::exception &e)
    {
        t1 = typeid(e).name(), m1 = e.what();
    }
    try
    {
        theirs();
    }
    catch (const std::exception &e)
    {
        t2 = typeid(e).name(), m2 = e.what();
    }
    g_checks++;
    if (t1 != t2 || m1 != m2 || t1 == "none")
    {
        g_fail++;
        std::printf("FAIL %s: ours %s '%s', reference %s '%s'\n", what, t1.c_str(), m1.c_str(), t2.c_str(), m2.c_str());
    }
}

static bool same_plain(const Plaintext &a, const Plaintext &b)
{
    return a.coeff_count() == b.coeff_count() && a.parms_id() == b.parms_id() &&
           std::memcmp(a.data(), b.data(), a.coeff_count() * sizeof(uint64_t)) == 0;
}

static void test_chain(scheme_type scheme)
{
    const size_t n = 4096;
    EncryptionParameters parms(scheme);
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(scheme == scheme_type::bfv ? CoeffModulus::BFVDefault(n) : CoeffModulus::Create(n, { 60, 50, 50, 50, 60 }));
    parms.set_plain_modulus(PlainModulus::Batching(n, 20));
    SEALContext context(parms, true, sec_level_type::none);
    KeyGenerator keygen(context);
    RelinKeys rk;
    keygen.create_relin_keys(rk);
    seal::Encryptor enc(context, keygen.secret_key());
    seal::Evaluator rev(context);
    seal::Decryptor rdec(context, keygen.secret_key());
    seal_b200::Evaluator gev(context);
    seal_b200::Decryptor gdec(context, keygen.secret_key(), gev);
    BatchEncoder be(context);
    std::vector<Ciphertext> cts(3);
    for (size_t i = 0; i < cts.size(); i++)
    {
        Plaintext p;
        be.encode(std::vector<uint64_t>(n, i + 2), p);
        enc.encrypt_symmetric(p, cts[i]);
    }
    for (int step = 0; step < 8; step++)
    {
        bool all_zero = true;
        for (auto &ct : cts)
        {
            const int want = rdec.invariant_noise_budget(ct);
            CHECK(gdec.invariant_noise_budget(ct) == want);
            all_zero = all_zero && want == 0;
        }
        // the batch overloads against the reference on the downloaded members
        seal_b200::CiphertextBatch batch;
        gev.upload(cts, batch);
        std::vector<int> budgets;
        gdec.invariant_noise_budget(batch, budgets);
        std::vector<Plaintext> plains;
        gdec.decrypt(batch, plains);
        std::vector<Ciphertext> back(cts.size());
        gev.download(batch, back);
        CHECK(budgets.size() == cts.size() && plains.size() == cts.size());
        for (size_t i = 0; i < cts.size() && i < budgets.size() && i < plains.size(); i++)
        {
            CHECK(budgets[i] == rdec.invariant_noise_budget(back[i]));
            Plaintext want;
            rdec.decrypt(back[i], want);
            CHECK(same_plain(plains[i], want));
        }
        if (all_zero)
            break;
        for (auto &ct : cts)
        {
            rev.multiply_inplace(ct, ct);
            rev.relinearize_inplace(ct, rk);
            if (scheme == scheme_type::bgv && ct.coeff_modulus_size() > 1)
                rev.mod_switch_to_next_inplace(ct);
        }
    }
    for (auto &ct : cts)
        CHECK(gdec.invariant_noise_budget(ct) == 0);
    // a size-3 ciphertext (before relinearization) and the wrong form
    Ciphertext c3 = cts[0];
    rev.multiply_inplace(c3, cts[1]);
    CHECK(gdec.invariant_noise_budget(c3) == rdec.invariant_noise_budget(c3));
    Ciphertext wrong = cts[0];
    wrong.is_ntt_form() = !wrong.is_ntt_form();
    same_throw([&] { gdec.invariant_noise_budget(wrong); }, [&] { (void)rdec.invariant_noise_budget(wrong); }, "wrong NTT form");
    Ciphertext empty(context);
    same_throw([&] { gdec.invariant_noise_budget(empty); }, [&] { (void)rdec.invariant_noise_budget(empty); }, "empty ciphertext");
    // a batch of another context
    seal_b200::Evaluator other(context);
    seal_b200::CiphertextBatch foreign;
    other.upload(cts, foreign);
    std::vector<int> budgets;
    bool threw = false;
    try
    {
        gdec.invariant_noise_budget(foreign, budgets);
    }
    catch (const std::invalid_argument &)
    {
        threw = true;
    }
    CHECK(threw);
    std::vector<Plaintext> plains;
    threw = false;
    try
    {
        gdec.decrypt(foreign, plains);
    }
    catch (const std::invalid_argument &)
    {
        threw = true;
    }
    CHECK(threw);
}

static void test_ckks()
{
    const size_t n = 4096;
    EncryptionParameters parms(scheme_type::ckks);
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(CoeffModulus::Create(n, { 50, 40, 50 }));
    SEALContext context(parms, true, sec_level_type::none);
    KeyGenerator keygen(context);
    seal::Encryptor enc(context, keygen.secret_key());
    seal::Decryptor rdec(context, keygen.secret_key());
    seal_b200::Evaluator gev(context);
    seal_b200::Decryptor gdec(context, keygen.secret_key(), gev);
    CKKSEncoder ce(context);
    Plaintext p;
    ce.encode(std::vector<double>(n / 2, 1.5), std::pow(2.0, 30), p);
    Ciphertext ct;
    enc.encrypt_symmetric(p, ct);
    same_throw([&] { gdec.invariant_noise_budget(ct); }, [&] { (void)rdec.invariant_noise_budget(ct); }, "CKKS");
    seal_b200::CiphertextBatch batch;
    gev.upload(std::vector<Ciphertext>{ ct, ct }, batch);
    std::vector<Plaintext> plains;
    gdec.decrypt(batch, plains);
    Plaintext want;
    rdec.decrypt(ct, want);
    CHECK(plains.size() == 2 && same_plain(plains[1], want) && plains[1].scale() == want.scale());
}

int main()
{
    test_chain(scheme_type::bfv);
    test_chain(scheme_type::bgv);
    test_ckks();
    std::printf("%d checks, %d failed\n", g_checks, g_fail);
    if (g_fail)
        return 1;
    std::printf("shim_noise_test ok\n");
    return 0;
}
