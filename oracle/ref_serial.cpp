// oracle/ref_serial.cpp -- TEST INFRASTRUCTURE ONLY.
// A flat C wrapper around the UNMODIFIED reference's seed-compressed objects for the tests and the measurement tool of the device's
// seeded streams (tests/test_gpu_serializable.py, tools/keygen_bench.py --stream): a context whose parameters carry a
// Blake2xbPRNGFactory or a Shake256PRNGFactory with the seed {seed, 0, ..., 0}, its KeyGenerator and a symmetric Encryptor, and the
// bytes Serializable<...>::save(compr_mode_type::none) writes for create_public_key(), create_relin_keys(), create_galois_keys(elts),
// encrypt_symmetric(plain) and encrypt_zero_symmetric(parms_id); plus the reference's own load of such streams.  It contains no
// arithmetic and no serialization code of its own.  Built by oracle/serial.mk into oracle/_ref/libsealref_serial.so.
#include "seal/seal.h"
#include <cstring>
#include <memory>
#include <string>
#include <vector>

using namespace seal;

static thread_local std::string g_err;

struct refser_ctx
{
    std::unique_ptr<SEALContext> context;
    std::unique_ptr<KeyGenerator> keygen;
    std::unique_ptr<Encryptor> encryptor;
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

extern "C" const char *refser_last_error(void)
{
    return g_err.c_str();
}

// scheme 1 BFV, 2 CKKS, 3 BGV; prng 1 Blake2xbPRNGFactory, 2 Shake256PRNGFactory, seeded {seed, 0, ..., 0}
extern "C" refser_ctx *refser_create(int scheme, size_t n, const uint64_t *moduli, size_t k, uint64_t plain_modulus, uint64_t seed, int prng)
{
    REF_TRY
    auto c = std::make_unique<refser_ctx>();
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
    c->encryptor = std::make_unique<Encryptor>(*c->context, c->keygen->secret_key());
    c->n = n, c->k = k;
    return c.release();
    REF_CATCH(nullptr)
}

extern "C" void refser_destroy(refser_ctx *c)
{
    delete c;
}

extern "C" int refser_secret_key(refser_ctx *c, uint64_t *out) // [k][n], NTT form
{
    REF_TRY
    std::memcpy(out, c->keygen->secret_key().data().data(), c->k * c->n * sizeof(uint64_t));
    return 0;
    REF_CATCH(-1)
}

// the object's save(compr_mode_type::none) into out (capacity bytes); returns the byte count, or -1
template <class T>
static long save(const T &obj, uint8_t *out, size_t capacity)
{
    const auto size = static_cast<size_t>(obj.save_size(compr_mode_type::none));
    if (!out)
        return static_cast<long>(size);
    if (size > capacity)
        throw std::invalid_argument("capacity");
    return static_cast<long>(obj.save(reinterpret_cast<seal_byte *>(out), capacity, compr_mode_type::none));
}

// parms_id of the level with L primes
static parms_id_type level(const refser_ctx *c, size_t L)
{
    for (auto cd = c->context->key_context_data(); cd; cd = cd->next_context_data())
        if (cd->parms().coeff_modulus().size() == L)
            return cd->parms_id();
    throw std::invalid_argument("no level with that many primes");
}

// out NULL: returns the size only (the key is still made: the factory's draws advance as in a real call)
extern "C" long refser_public_key(refser_ctx *c, uint8_t *out, size_t capacity)
{
    REF_TRY
    return save(c->keygen->create_public_key(), out, capacity);
    REF_CATCH(-1)
}

extern "C" long refser_relin_keys(refser_ctx *c, uint8_t *out, size_t capacity)
{
    REF_TRY
    return save(c->keygen->create_relin_keys(), out, capacity);
    REF_CATCH(-1)
}

// create_galois_keys(elts); all != 0: create_galois_keys() (the default set)
extern "C" long refser_galois_keys(refser_ctx *c, const uint32_t *elts, size_t count, int all, uint8_t *out, size_t capacity)
{
    REF_TRY
    if (all)
        return save(c->keygen->create_galois_keys(), out, capacity);
    return save(c->keygen->create_galois_keys(std::vector<uint32_t>(elts, elts + count)), out, capacity);
    REF_CATCH(-1)
}

// encrypt_symmetric(plain): CKKS plain = [L][n] NTT form at the level with L primes and the given scale; BFV / BGV plain = [n]
// coefficients (L ignored)
extern "C" long refser_encrypt_symmetric(refser_ctx *c, size_t L, const uint64_t *plain, double scale, uint8_t *out, size_t capacity)
{
    REF_TRY
    Plaintext p;
    if (c->context->key_context_data()->parms().scheme() == scheme_type::ckks)
    {
        p.parms_id() = parms_id_zero;
        p.resize(L * c->n);
        std::memcpy(p.data(), plain, L * c->n * sizeof(uint64_t));
        p.parms_id() = level(c, L);
        p.scale() = scale;
    }
    else
    {
        p.resize(c->n);
        std::memcpy(p.data(), plain, c->n * sizeof(uint64_t));
    }
    return save(c->encryptor->encrypt_symmetric(p), out, capacity);
    REF_CATCH(-1)
}

extern "C" long refser_encrypt_zero_symmetric(refser_ctx *c, size_t L, uint8_t *out, size_t capacity)
{
    REF_TRY
    return save(c->encryptor->encrypt_zero_symmetric(level(c, L)), out, capacity);
    REF_CATCH(-1)
}

// Ciphertext::load (validating) of a stream, seeded or not; out = its words [size][L][n]; returns the word count
extern "C" long refser_load_ciphertext(refser_ctx *c, const uint8_t *in, size_t len, uint64_t *out, size_t capacity_words)
{
    REF_TRY
    Ciphertext ct;
    ct.load(*c->context, reinterpret_cast<const seal_byte *>(in), len);
    const size_t words = ct.size() * ct.coeff_modulus_size() * ct.poly_modulus_degree();
    if (words > capacity_words)
        throw std::invalid_argument("capacity");
    std::memcpy(out, ct.data(), words * sizeof(uint64_t));
    return static_cast<long>(words);
    REF_CATCH(-1)
}

// PublicKey::load; out = [2][k][n]
extern "C" long refser_load_public_key(refser_ctx *c, const uint8_t *in, size_t len, uint64_t *out)
{
    REF_TRY
    PublicKey pk;
    pk.load(*c->context, reinterpret_cast<const seal_byte *>(in), len);
    std::memcpy(out, pk.data().data(), 2 * c->k * c->n * sizeof(uint64_t));
    return 0;
    REF_CATCH(-1)
}

// RelinKeys::load (galois_elt 0) / GaloisKeys::load; out = the entry's [k-1][2][k][n] words; returns the digit count
extern "C" long refser_load_kswitch(refser_ctx *c, const uint8_t *in, size_t len, uint32_t galois_elt, uint64_t *out)
{
    REF_TRY
    RelinKeys rk;
    GaloisKeys gk;
    const std::vector<PublicKey> *v;
    if (galois_elt == 0)
    {
        rk.load(*c->context, reinterpret_cast<const seal_byte *>(in), len);
        v = &rk.key(2);
    }
    else
    {
        gk.load(*c->context, reinterpret_cast<const seal_byte *>(in), len);
        v = &gk.key(galois_elt);
    }
    const size_t words = 2 * c->k * c->n;
    for (size_t j = 0; j < v->size(); j++)
        std::memcpy(out + j * words, (*v)[j].data().data(), words * sizeof(uint64_t));
    return static_cast<long>(v->size());
    REF_CATCH(-1)
}
