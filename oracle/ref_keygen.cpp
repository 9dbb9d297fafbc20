// oracle/ref_keygen.cpp -- TEST INFRASTRUCTURE ONLY.
// A flat C wrapper around the UNMODIFIED reference's KeyGenerator for the tests and the measurement tool of the device's key
// generation (tests/test_keygen_oracle.py, tests/test_gpu_keygen.py, tools/keygen_bench.py): a context whose parameters carry a
// Blake2xbPRNGFactory or a Shake256PRNGFactory with the seed {seed, 0, ..., 0}, its KeyGenerator, and the words of the keys
// create_public_key / create_relin_keys / create_galois_keys put into their destination objects.  Like ref_prng.cpp it contains no
// arithmetic of its own.  Built by oracle/keygen.mk into oracle/_ref/libsealref_keygen.so.
#include "seal/seal.h"
#include <cstring>
#include <memory>
#include <string>
#include <vector>

using namespace seal;

static thread_local std::string g_err;

struct refkg_ctx
{
    std::unique_ptr<SEALContext> context;
    std::unique_ptr<KeyGenerator> keygen;
    size_t n = 0, k = 0;
};

#define REF_TRY try {
#define REF_CATCH(ret)              \
    }                               \
    catch (const std::exception &e) \
    {                               \
        g_err = e.what();           \
        return ret;                 \
    }

extern "C" const char *refkg_last_error(void)
{
    return g_err.c_str();
}

// scheme 1 BFV, 2 CKKS, 3 BGV; prng 1 Blake2xbPRNGFactory, 2 Shake256PRNGFactory, seeded {seed, 0, ..., 0}: every create() of the
// factory returns a PRNG of that seed, so the secret key and every bootstrap PRNG of the keys start from it
extern "C" refkg_ctx *refkg_create(int scheme, size_t n, const uint64_t *moduli, size_t k, uint64_t plain_modulus, uint64_t seed, int prng)
{
    REF_TRY
    auto c = std::make_unique<refkg_ctx>();
    EncryptionParameters parms(static_cast<scheme_type>(scheme));
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(std::vector<Modulus>(moduli, moduli + k));
    if (parms.scheme() != scheme_type::ckks)
        parms.set_plain_modulus(plain_modulus);
    prng_seed_type s{};
    s[0] = seed;
    if (prng == static_cast<int>(prng_type::blake2xb))
        parms.set_random_generator(std::make_shared<Blake2xbPRNGFactory>(s));
    else if (prng == static_cast<int>(prng_type::shake256))
        parms.set_random_generator(std::make_shared<Shake256PRNGFactory>(s));
    else
        throw std::invalid_argument("prng_type");
    c->context = std::make_unique<SEALContext>(parms, true, sec_level_type::none);
    if (!c->context->parameters_set())
        throw std::invalid_argument(c->context->parameter_error_message());
    c->keygen = std::make_unique<KeyGenerator>(*c->context);
    c->n = n, c->k = k;
    return c.release();
    REF_CATCH(nullptr)
}

extern "C" void refkg_destroy(refkg_ctx *c)
{
    delete c;
}

extern "C" int refkg_secret_key(refkg_ctx *c, uint64_t *out) // [k][n], NTT form
{
    REF_TRY
    std::memcpy(out, c->keygen->secret_key().data().data(), c->k * c->n * sizeof(uint64_t));
    return 0;
    REF_CATCH(-1)
}

// KeyGenerator::create_public_key(PublicKey &): [2][k][n]; out may be NULL (the key is made and dropped)
extern "C" int refkg_public_key(refkg_ctx *c, uint64_t *out)
{
    REF_TRY
    PublicKey pk;
    c->keygen->create_public_key(pk);
    if (out)
        std::memcpy(out, pk.data().data(), 2 * c->k * c->n * sizeof(uint64_t));
    return 0;
    REF_CATCH(-1)
}

// KeyGenerator::create_relin_keys(RelinKeys &) (galois_elt 0) / create_galois_keys({galois_elt}, GaloisKeys &): the entry's
// [k-1][2][k][n] words into out (may be NULL); returns the digit count
extern "C" long refkg_kswitch_key(refkg_ctx *c, uint32_t galois_elt, uint64_t *out)
{
    REF_TRY
    const std::vector<PublicKey> *v = nullptr;
    RelinKeys rk;
    GaloisKeys gk;
    if (galois_elt == 0)
    {
        c->keygen->create_relin_keys(rk);
        v = &rk.data()[0];
    }
    else
    {
        c->keygen->create_galois_keys(std::vector<uint32_t>{ galois_elt }, gk);
        v = &gk.data()[GaloisKeys::get_index(galois_elt)];
    }
    const size_t words = 2 * c->k * c->n;
    if (out)
        for (size_t j = 0; j < v->size(); j++)
            std::memcpy(out + j * words, (*v)[j].data().data(), words * sizeof(uint64_t));
    return static_cast<long>(v->size());
    REF_CATCH(-1)
}

// GaloisTool::get_elts_all() of the key level: the elements create_galois_keys(GaloisKeys &) makes keys for; returns the count
extern "C" long refkg_galois_elts_all(refkg_ctx *c, uint32_t *out, size_t capacity)
{
    REF_TRY
    const auto elts = c->context->key_context_data()->galois_tool()->get_elts_all();
    if (elts.size() > capacity)
        throw std::invalid_argument("capacity");
    std::copy(elts.begin(), elts.end(), out);
    return static_cast<long>(elts.size());
    REF_CATCH(-1)
}
