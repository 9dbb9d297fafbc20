// oracle/ref_prng.cpp -- TEST INFRASTRUCTURE ONLY.
// A flat C wrapper around the UNMODIFIED reference for the tests of the device's PRNG paths (tests/refprng.py): contexts whose
// parameters carry a Blake2xbPRNGFactory or a Shake256PRNGFactory, the PRNG streams themselves, encryption under those contexts,
// and the seed-compressed objects SEAL users save (Serializable<Ciphertext>, KeyGenerator::create_relin_keys() /
// create_galois_keys()) with the reference's own loaders.  Like ref_capi.cpp it contains no arithmetic of its own: every number
// it returns is computed by the reference.  Built by oracle/prng.mk into oracle/_ref/libsealref_prng.so.
#include "seal/seal.h"
#include <cstring>
#include <memory>
#include <string>
#include <vector>

using namespace seal;

static thread_local std::string g_err;

struct sealprng_ctx
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

static compr_mode_type mode_of(int mode)
{
    if (mode == 0)
        return compr_mode_type::none;
    if (mode == 1)
        return compr_mode_type::zlib;
    throw std::invalid_argument("unsupported compression mode");
}

static parms_id_type level_id(const sealprng_ctx *c, size_t L)
{
    if (L == c->k)
        return c->context->key_parms_id();
    auto cd = c->context->first_context_data();
    while (cd && cd->parms().coeff_modulus().size() != L)
        cd = cd->next_context_data();
    if (!cd)
        throw std::invalid_argument("no level with that many primes");
    return cd->parms_id();
}

extern "C" const char *sealprng_last_error(void)
{
    return g_err.c_str();
}

// scheme 1 BFV, 2 CKKS, 3 BGV; the parameters' random generator factory is of prng_type `prng` (1 Blake2xbPRNGFactory,
// 2 Shake256PRNGFactory) with the default seed {seed, 0, ..., 0}: keys and encryptions are deterministic
extern "C" sealprng_ctx *sealprng_create(int scheme, size_t n, const uint64_t *moduli, size_t k, uint64_t plain_modulus, uint64_t seed,
                                         int prng)
{
    REF_TRY
    auto c = std::make_unique<sealprng_ctx>();
    EncryptionParameters parms(static_cast<scheme_type>(scheme));
    parms.set_poly_modulus_degree(n);
    std::vector<Modulus> mods(moduli, moduli + k);
    parms.set_coeff_modulus(mods);
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

extern "C" void sealprng_destroy(sealprng_ctx *c)
{
    delete c;
}

// the first `bytes` bytes UniformRandomGenerator::generate returns for Blake2xbPRNG(seed) (1) / Shake256PRNG(seed) (2)
extern "C" int sealprng_stream(int type, const uint64_t *seed8, size_t bytes, uint8_t *out)
{
    REF_TRY
    prng_seed_type s;
    std::copy_n(seed8, prng_seed_uint64_count, s.begin());
    auto prng = UniformRandomGeneratorInfo(static_cast<prng_type>(type), s).make_prng();
    if (!prng)
        throw std::invalid_argument("prng_type");
    prng->generate(bytes, reinterpret_cast<seal_byte *>(out));
    return 0;
    REF_CATCH(-1)
}

extern "C" int sealprng_secret_key(sealprng_ctx *c, uint64_t *out) // [k][n], NTT form
{
    REF_TRY
    std::memcpy(out, c->keygen->secret_key().data().data(), c->k * c->n * sizeof(uint64_t));
    return 0;
    REF_CATCH(-1)
}

extern "C" int sealprng_public_key(sealprng_ctx *c, uint64_t *out) // KeyGenerator::create_public_key: [2][k][n]
{
    REF_TRY
    PublicKey pk;
    c->keygen->create_public_key(pk);
    std::memcpy(out, pk.data().data(), 2 * c->k * c->n * sizeof(uint64_t));
    return 0;
    REF_CATCH(-1)
}

// Encryptor::encrypt_zero_symmetric(parms_id of the level with L primes, ct): [2][L][n]
extern "C" int sealprng_encrypt_zero_symmetric(sealprng_ctx *c, size_t L, uint64_t *out2)
{
    REF_TRY
    Encryptor encryptor(*c->context, c->keygen->secret_key());
    Ciphertext ct;
    encryptor.encrypt_zero_symmetric(level_id(c, L), ct);
    std::memcpy(out2, ct.data(), 2 * L * c->n * sizeof(uint64_t));
    return 0;
    REF_CATCH(-1)
}

// Encryptor(public key)::encrypt_zero(parms_id of the level with L primes; L == k: the key level): [2][L][n]
extern "C" int sealprng_encrypt_zero_asymmetric(sealprng_ctx *c, size_t L, uint64_t *out2)
{
    REF_TRY
    PublicKey pk;
    c->keygen->create_public_key(pk);
    Encryptor encryptor(*c->context, pk);
    Ciphertext ct;
    encryptor.encrypt_zero(level_id(c, L), ct);
    std::memcpy(out2, ct.data(), 2 * L * c->n * sizeof(uint64_t));
    return 0;
    REF_CATCH(-1)
}

// Encryptor::encrypt_zero_symmetric().save(): the seed-compressed ciphertext at the first data level, compr_mode `mode`
extern "C" long sealprng_seeded_ct_stream(sealprng_ctx *c, int mode, uint8_t *out, size_t capacity)
{
    REF_TRY
    Encryptor encryptor(*c->context, c->keygen->secret_key());
    return static_cast<long>(encryptor.encrypt_zero_symmetric().save(reinterpret_cast<seal_byte *>(out), capacity, mode_of(mode)));
    REF_CATCH(-1)
}

// Ciphertext::load of any stream (seeded or not, any compression) -> [size][L][n] words; returns size * L (rows)
extern "C" long sealprng_ct_load(sealprng_ctx *c, const uint8_t *in, size_t len, uint64_t *out, size_t capacity_words)
{
    REF_TRY
    Ciphertext ct;
    ct.load(*c->context, reinterpret_cast<const seal_byte *>(in), len);
    const size_t words = ct.size() * ct.coeff_modulus_size() * c->n;
    if (words > capacity_words)
        throw std::invalid_argument("capacity");
    std::memcpy(out, ct.data(), words * sizeof(uint64_t));
    return static_cast<long>(ct.size() * ct.coeff_modulus_size());
    REF_CATCH(-1)
}

// KeyGenerator::create_relin_keys() (galois_elt 0) / create_galois_keys({galois_elt}): the seeded objects, compr_mode `mode`
extern "C" long sealprng_seeded_kswitch_keys_stream(sealprng_ctx *c, uint32_t galois_elt, int mode, uint8_t *out, size_t capacity)
{
    REF_TRY
    auto *dst = reinterpret_cast<seal_byte *>(out);
    if (galois_elt == 0)
        return static_cast<long>(c->keygen->create_relin_keys().save(dst, capacity, mode_of(mode)));
    return static_cast<long>(c->keygen->create_galois_keys(std::vector<uint32_t>{ galois_elt }).save(dst, capacity, mode_of(mode)));
    REF_CATCH(-1)
}

// KSwitchKeys::load of such a stream; data()[index] as [digit][2][k][n] into out; returns the digit count
extern "C" long sealprng_kswitch_keys_load(sealprng_ctx *c, const uint8_t *in, size_t len, size_t index, uint64_t *out, size_t capacity_words)
{
    REF_TRY
    KSwitchKeys keys;
    keys.load(*c->context, reinterpret_cast<const seal_byte *>(in), len);
    if (index >= keys.data().size())
        throw std::out_of_range("index");
    const auto &v = keys.data()[index];
    const size_t words = 2 * c->k * c->n;
    if (v.size() * words > capacity_words)
        throw std::invalid_argument("capacity");
    for (size_t j = 0; j < v.size(); j++)
        std::memcpy(out + j * words, v[j].data().data(), words * sizeof(uint64_t));
    return static_cast<long>(v.size());
    REF_CATCH(-1)
}
