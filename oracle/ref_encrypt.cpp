// oracle/ref_encrypt.cpp -- TEST INFRASTRUCTURE ONLY.
// A flat C wrapper around the UNMODIFIED reference for the tests of encryption of device-resident plaintexts
// (tests/test_gpu_encrypt_batch.py): seal::Encryptor::encrypt / encrypt_symmetric of one plaintext under a context whose
// parameters carry a Blake2xbPRNGFactory or a Shake256PRNGFactory seeded with a given 8-word seed, with a given secret or public
// key.  parms_id does not depend on the factory, so one key serves every such context.  Like ref_prng.cpp it contains no
// arithmetic of its own: every word it returns is computed by the reference.  Built by oracle/encrypt.mk into
// oracle/_ref/libsealref_encrypt.so.
#include "seal/seal.h"
#include <cstring>
#include <memory>
#include <sstream>
#include <string>
#include <vector>

using namespace seal;

static thread_local std::string g_err;

extern "C" const char *sealenc_last_error(void)
{
    return g_err.c_str();
}

// scheme 1 BFV, 2 CKKS, 3 BGV; key = the secret key [k][n] (is_asymmetric 0) or the public key [2][k][n] (1), NTT form at the key
// level; seed8 / prng: the factory of the parameters (1 Blake2xbPRNGFactory, 2 Shake256PRNGFactory).  plain: CKKS [L][n] NTT form
// at the level with L primes and the given scale; BFV / BGV coeff_count words < t (L ignored: the first level).
// save_seed = 0: out = the ciphertext [2][L'][n].  save_seed = 1 (symmetric only): the Serializable<Ciphertext>'s c_0 ([L'][n]
// into out) and its seed (8 words into out_seed).  Returns L' (the primes of the result) or -1.
extern "C" long sealenc_encrypt(int scheme, size_t n, const uint64_t *moduli, size_t k, uint64_t plain_modulus, const uint64_t *key,
                                int is_asymmetric, const uint64_t *seed8, int prng, int save_seed, const uint64_t *plain,
                                size_t plain_words, size_t L, double scale, uint64_t *out, uint64_t *out_seed)
{
    try
    {
        EncryptionParameters parms(static_cast<scheme_type>(scheme));
        parms.set_poly_modulus_degree(n);
        parms.set_coeff_modulus(std::vector<Modulus>(moduli, moduli + k));
        if (parms.scheme() != scheme_type::ckks)
            parms.set_plain_modulus(plain_modulus);
        prng_seed_type s;
        std::copy_n(seed8, prng_seed_uint64_count, s.begin());
        if (prng == static_cast<int>(prng_type::blake2xb))
            parms.set_random_generator(std::make_shared<Blake2xbPRNGFactory>(s));
        else if (prng == static_cast<int>(prng_type::shake256))
            parms.set_random_generator(std::make_shared<Shake256PRNGFactory>(s));
        else
            throw std::invalid_argument("prng_type");
        SEALContext context(parms, true, sec_level_type::none);
        if (!context.parameters_set())
            throw std::invalid_argument(context.parameter_error_message());

        Plaintext p;
        p.resize(plain_words);
        std::memcpy(p.data(), plain, plain_words * sizeof(uint64_t));
        if (parms.scheme() == scheme_type::ckks)
        {
            auto cd = context.first_context_data();
            while (cd && cd->parms().coeff_modulus().size() != L)
                cd = cd->next_context_data();
            if (!cd)
                throw std::invalid_argument("no level with that many primes");
            p.parms_id() = cd->parms_id();
            p.scale() = scale;
        }

        std::unique_ptr<Encryptor> enc;
        if (is_asymmetric)
        {
            PublicKey pk;
            pk.data().resize(context, context.key_parms_id(), 2);
            std::memcpy(pk.data().data(), key, 2 * k * n * sizeof(uint64_t));
            pk.data().is_ntt_form() = true;
            enc = std::make_unique<Encryptor>(context, pk);
        }
        else
        {
            SecretKey sk;
            sk.data().resize(k * n);
            std::memcpy(sk.data().data(), key, k * n * sizeof(uint64_t));
            sk.data().parms_id() = context.key_parms_id();
            enc = std::make_unique<Encryptor>(context, sk);
        }
        Ciphertext ct;
        if (save_seed)
        {
            if (is_asymmetric)
                throw std::invalid_argument("save_seed is symmetric only");
            // the seeded object's stream: c_0 through the reference's own Ciphertext::load, the seed from the stream's trailing
            // UniformRandomGeneratorInfo (uncompressed: its last 64 bytes)
            std::stringstream ss;
            enc->encrypt_symmetric(p).save(ss, compr_mode_type::none);
            const std::string bytes = ss.str();
            ct.load(context, reinterpret_cast<const seal_byte *>(bytes.data()), bytes.size());
            std::memcpy(out_seed, bytes.data() + bytes.size() - 64, 64);
            std::memcpy(out, ct.data(), ct.coeff_modulus_size() * n * sizeof(uint64_t));
            return static_cast<long>(ct.coeff_modulus_size());
        }
        if (is_asymmetric)
            enc->encrypt(p, ct);
        else
            enc->encrypt_symmetric(p, ct);
        std::memcpy(out, ct.data(), 2 * ct.coeff_modulus_size() * n * sizeof(uint64_t));
        return static_cast<long>(ct.coeff_modulus_size());
    }
    catch (const std::exception &e)
    {
        g_err = e.what();
        return -1;
    }
}
