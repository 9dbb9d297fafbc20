// oracle/ref_keyset.cpp -- TEST INFRASTRUCTURE ONLY.
// A flat C wrapper around the UNMODIFIED reference for the tests and the measurement tool of the device's key-set loader
// (tests/test_gpu_keyset_load.py, tools/keyset_bench.py): a context whose parameters carry a Blake2xbPRNGFactory or a
// Shake256PRNGFactory with the seed {seed, 0, ..., 0}, its KeyGenerator and a symmetric Encryptor; the bytes RelinKeys / GaloisKeys /
// Ciphertext::save write in compr_mode none or zlib, or Serializable<...>::save(none) writes for the seeded objects; and the
// reference's own load of such streams back to words.  It contains no arithmetic and no serialization code of its own.  Built by
// oracle/keyset.mk into oracle/_ref/libsealref_keyset.so.
#include "seal/seal.h"
#include <cstring>
#include <memory>
#include <string>
#include <vector>

using namespace seal;

static thread_local std::string g_err;

struct refks_ctx
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

extern "C" const char *refks_last_error(void)
{
    return g_err.c_str();
}

// scheme 1 BFV, 2 CKKS, 3 BGV; prng 1 Blake2xbPRNGFactory, 2 Shake256PRNGFactory, seeded {seed, 0, ..., 0}
extern "C" refks_ctx *refks_create(int scheme, size_t n, const uint64_t *moduli, size_t k, uint64_t plain_modulus, uint64_t seed, int prng)
{
    REF_TRY
    auto c = std::make_unique<refks_ctx>();
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

extern "C" void refks_destroy(refks_ctx *c)
{
    delete c;
}

extern "C" int refks_secret_key(refks_ctx *c, uint64_t *out) // [k][n], NTT form
{
    REF_TRY
    std::memcpy(out, c->keygen->secret_key().data().data(), c->k * c->n * sizeof(uint64_t));
    return 0;
    REF_CATCH(-1)
}

// mode 0 = save(compr_mode none), 1 = save(compr_mode zlib), 2 = the seeded Serializable object saved with compr_mode none.
// out NULL: returns the size only (the object is still made: the factory's draws advance as in a real call); else the byte count
template <class T>
static long save(const T &obj, int mode, uint8_t *out, size_t capacity)
{
    const compr_mode_type m = mode == 1 ? compr_mode_type::zlib : compr_mode_type::none;
    std::vector<seal_byte> buf(static_cast<size_t>(obj.save_size(m)));
    const auto size = static_cast<size_t>(obj.save(buf.data(), buf.size(), m));
    if (!out)
        return static_cast<long>(size);
    if (size > capacity)
        throw std::invalid_argument("capacity");
    std::memcpy(out, buf.data(), size);
    return static_cast<long>(size);
}

extern "C" long refks_relin_keys(refks_ctx *c, int mode, uint8_t *out, size_t capacity)
{
    REF_TRY
    if (mode == 2)
        return save(c->keygen->create_relin_keys(), 0, out, capacity);
    RelinKeys rk;
    c->keygen->create_relin_keys(rk);
    return save(rk, mode, out, capacity);
    REF_CATCH(-1)
}

// create_galois_keys(elts); all != 0: create_galois_keys() (the default set)
extern "C" long refks_galois_keys(refks_ctx *c, const uint32_t *elts, size_t count, int all, int mode, uint8_t *out, size_t capacity)
{
    REF_TRY
    const std::vector<uint32_t> e(elts, elts + count);
    if (mode == 2)
        return save(all ? c->keygen->create_galois_keys() : c->keygen->create_galois_keys(e), 0, out, capacity);
    GaloisKeys gk;
    if (all)
        c->keygen->create_galois_keys(gk);
    else
        c->keygen->create_galois_keys(e, gk);
    return save(gk, mode, out, capacity);
    REF_CATCH(-1)
}

// the galois elements of create_galois_keys() (GaloisTool::get_elts_all), count returned
extern "C" long refks_galois_elts_all(refks_ctx *c, uint32_t *out, size_t capacity)
{
    REF_TRY
    const auto e = c->context->key_context_data()->galois_tool()->get_elts_all();
    if (e.size() > capacity)
        throw std::invalid_argument("capacity");
    std::memcpy(out, e.data(), e.size() * sizeof(uint32_t));
    return static_cast<long>(e.size());
    REF_CATCH(-1)
}

// encrypt_zero_symmetric at the level with L primes, saved with `mode` as above
extern "C" long refks_encrypt_zero(refks_ctx *c, size_t L, int mode, uint8_t *out, size_t capacity)
{
    REF_TRY
    parms_id_type pid = parms_id_zero;
    for (auto cd = c->context->key_context_data(); cd; cd = cd->next_context_data())
        if (cd->parms().coeff_modulus().size() == L)
            pid = cd->parms_id();
    if (mode == 2)
        return save(c->encryptor->encrypt_zero_symmetric(pid), 0, out, capacity);
    Ciphertext ct;
    c->encryptor->encrypt_zero_symmetric(pid, ct);
    return save(ct, mode, out, capacity);
    REF_CATCH(-1)
}

// Ciphertext::load of a stream; out = its words [size][L][n]; returns the word count
extern "C" long refks_load_ciphertext(refks_ctx *c, const uint8_t *in, size_t len, uint64_t *out, size_t capacity_words)
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

// RelinKeys::load (galois_elt 0) / GaloisKeys::load; out = the entry's [k-1][2][k][n] words; returns the digit count
extern "C" long refks_load_kswitch(refks_ctx *c, const uint8_t *in, size_t len, uint32_t galois_elt, uint64_t *out)
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
