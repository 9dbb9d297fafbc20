// oracle/ref_noise.cpp -- TEST INFRASTRUCTURE ONLY.
// A flat C wrapper around the UNMODIFIED reference for the tests of the device's invariant noise budget (tests/noise_ref.py):
// a context and a Decryptor under a given secret key, and Decryptor::invariant_noise_budget of arbitrary ciphertext words in a
// given form.  Like ref_capi.cpp it contains no arithmetic of its own: every number it returns is computed by the reference.
// Built by oracle/noise.mk into oracle/_ref/libsealref_noise.so.
#include "seal/seal.h"
#include <cstring>
#include <memory>
#include <string>
#include <vector>

using namespace seal;

static thread_local std::string g_err;

struct sealnoise_ctx
{
    std::unique_ptr<SEALContext> context;
    std::unique_ptr<Decryptor> decryptor;
    size_t n = 0;
};

#define REF_TRY try {
#define REF_CATCH(ret)              \
    }                               \
    catch (const std::exception &e) \
    {                               \
        g_err = e.what();           \
        return ret;                 \
    }

extern "C" const char *sealnoise_last_error(void)
{
    return g_err.c_str();
}

// scheme 1 BFV, 2 CKKS, 3 BGV (SEALContext(parms, true, sec_level_type::none)); secret_key = SecretKey::data(): [k][n] words in NTT
// form at the key level
extern "C" sealnoise_ctx *sealnoise_create(int scheme, size_t n, const uint64_t *moduli, size_t k, uint64_t plain_modulus,
                                           const uint64_t *secret_key)
{
    REF_TRY
    auto c = std::make_unique<sealnoise_ctx>();
    EncryptionParameters parms(static_cast<scheme_type>(scheme));
    parms.set_poly_modulus_degree(n);
    parms.set_coeff_modulus(std::vector<Modulus>(moduli, moduli + k));
    if (parms.scheme() != scheme_type::ckks)
        parms.set_plain_modulus(plain_modulus);
    c->context = std::make_unique<SEALContext>(parms, true, sec_level_type::none);
    if (!c->context->parameters_set())
        throw std::invalid_argument(c->context->parameter_error_message());
    SecretKey sk;
    sk.data().resize(k * n);
    std::memcpy(sk.data().data(), secret_key, k * n * sizeof(uint64_t));
    sk.data().parms_id() = c->context->key_parms_id();
    c->decryptor = std::make_unique<Decryptor>(*c->context, sk);
    c->n = n;
    return c.release();
    REF_CATCH(nullptr)
}

extern "C" void sealnoise_destroy(sealnoise_ctx *c)
{
    delete c;
}

// Decryptor::invariant_noise_budget of a ciphertext [size][L][n] at the level with L primes (L = k: the key level); -1 with the
// reference's message (sealnoise_last_error) when the reference throws
extern "C" int sealnoise_budget(sealnoise_ctx *c, size_t L, size_t size, int is_ntt_form, const uint64_t *ct, int *budget)
{
    REF_TRY
    auto cd = c->context->key_context_data();
    while (cd && cd->parms().coeff_modulus().size() != L)
        cd = cd->next_context_data();
    if (!cd)
        throw std::invalid_argument("no level with that many primes");
    Ciphertext x;
    x.resize(*c->context, cd->parms_id(), size);
    std::memcpy(x.data(), ct, size * L * c->n * sizeof(uint64_t));
    x.is_ntt_form() = is_ntt_form != 0;
    *budget = c->decryptor->invariant_noise_budget(x);
    return 0;
    REF_CATCH(-1)
}
