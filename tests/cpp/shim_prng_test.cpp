// tests/cpp/shim_prng_test.cpp -- seal_b200::Encryptor (include/seal_b200/encryptor.hpp) against seal::Encryptor when the
// parameters carry a Shake256PRNGFactory: words and metadata of every fresh ciphertext must be the reference's.  Built by
// oracle/prng.mk into oracle/_ref/bin/shim_prng_test (it links the reference library); run by tests/test_gpu_prng.py.
#include "seal/seal.h"
#include "seal_b200/encryptor.hpp"
#include <cmath>
#include <cstdio>
#include <cstring>
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

// words and metadata
static bool same_ct(const Ciphertext &a, const Ciphertext &b)
{
    if (a.parms_id() != b.parms_id() || a.size() != b.size() || a.is_ntt_form() != b.is_ntt_form() ||
        a.coeff_modulus_size() != b.coeff_modulus_size() || a.poly_modulus_degree() != b.poly_modulus_degree())
        return false;
    double sa = a.scale(), sb = b.scale();
    if (std::memcmp(&sa, &sb, sizeof(double)) != 0 || a.correction_factor() != b.correction_factor())
        return false;
    return std::memcmp(a.data(), b.data(), a.size() * a.coeff_modulus_size() * a.poly_modulus_degree() * sizeof(uint64_t)) == 0;
}

// seal_b200::Encryptor with Shake256PRNGFactory(seed) on the parameters: the bootstrap / public-key PRNG is SHAKE256 on both sides
// (util/rlwe.cpp:224, :322), c_1 is expanded with the default factory's PRNG; secret- and public-key encryption, all three schemes
static void test_encryptor_shake256()
{
    prng_seed_type seed{};
    seed[0] = 0x5EED;
    seed[3] = 17;
    for (auto scheme : { scheme_type::ckks, scheme_type::bfv, scheme_type::bgv })
    {
        EncryptionParameters parms(scheme);
        const size_t n = scheme == scheme_type::ckks ? 8192 : 4096;
        parms.set_poly_modulus_degree(n);
        parms.set_coeff_modulus(scheme == scheme_type::ckks ? CoeffModulus::Create(n, { 60, 40, 40, 60 }) : CoeffModulus::Create(n, { 36, 36, 37 }));
        if (scheme != scheme_type::ckks)
            parms.set_plain_modulus(PlainModulus::Batching(n, 20));
        parms.set_random_generator(std::make_shared<Shake256PRNGFactory>(seed));
        SEALContext context(parms, true, sec_level_type::none);
        KeyGenerator keygen(context);
        PublicKey pk;
        keygen.create_public_key(pk);
        seal::Encryptor rcrypt(context, pk, keygen.secret_key());
        seal_b200::Evaluator gev(context);
        seal_b200::Encryptor gcrypt(context, pk, keygen.secret_key(), gev);
        Plaintext p;
        if (scheme == scheme_type::ckks)
        {
            seal::CKKSEncoder enc(context);
            enc.encode(std::vector<double>{ 1.5, -2.25, 3.0 }, std::pow(2.0, 40), p);
        }
        else
        {
            seal::BatchEncoder enc(context);
            std::vector<uint64_t> slots(enc.slot_count());
            for (size_t i = 0; i < slots.size(); i++)
                slots[i] = (i * 31 + 7) % parms.plain_modulus().value();
            enc.encode(slots, p);
        }
        Ciphertext cr, cg;
        rcrypt.encrypt_symmetric(p, cr);
        gcrypt.encrypt_symmetric(p, cg);
        CHECK(same_ct(cr, cg));
        rcrypt.encrypt_zero_symmetric(cr);
        gcrypt.encrypt_zero_symmetric(cg);
        CHECK(same_ct(cr, cg));
        rcrypt.encrypt_zero_symmetric(context.last_parms_id(), cr);
        gcrypt.encrypt_zero_symmetric(context.last_parms_id(), cg);
        CHECK(same_ct(cr, cg));
        rcrypt.encrypt(p, cr);
        gcrypt.encrypt(p, cg);
        CHECK(same_ct(cr, cg));
        rcrypt.encrypt_zero(context.last_parms_id(), cr);
        gcrypt.encrypt_zero(context.last_parms_id(), cg);
        CHECK(same_ct(cr, cg));
        rcrypt.encrypt_zero(cr);
        gcrypt.encrypt_zero(cg);
        CHECK(same_ct(cr, cg));
        CHECK(cg.is_ntt_form() == (scheme != scheme_type::bfv) && cg.scale() == cr.scale() && cg.correction_factor() == cr.correction_factor());
    }
}

int main()
{
    try
    {
        test_encryptor_shake256();
    }
    catch (const std::exception &e)
    {
        std::printf("FAIL: unexpected exception: %s\n", e.what());
        return 2;
    }
    std::printf("%s: %d checks, %d failed\n", g_fail ? "FAIL" : "PASS", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
