// include/seal_b200/keygenerator.hpp -- same-signature stand-in for seal::KeyGenerator constructed from an existing secret key
// (native/src/seal/keygenerator.h:45-290: create_public_key, create_relin_keys, create_galois_keys with a destination object) over
// the C-ABI of include/seal_b200.h.
//
//     seal::KeyGenerator sk_gen(context);                                 // the secret key is sampled by the reference (or loaded)
//     seal_b200::KeyGenerator keygen(context, sk_gen.secret_key());       // or (context, secret_key, evaluator) to share its device
//     keygen.create_relin_keys(rk);  keygen.create_galois_keys(gk);
//
// Every key is a set of key-level encryptions of zero in NTT form made on the device (sb200_public_key_generate,
// sb200_kswitch_key_generate).  The bootstrap seed of each encryption is drawn from the context's own random generator factory
// exactly where and in the order the reference draws it (one for the public key, one per digit of every key-switching key, Galois
// elements in the order given with duplicates skipped), so a context with a seeded factory (Blake2xbPRNGFactory or
// Shake256PRNGFactory) reproduces the reference's keys bit for bit and the default factory draws from the OS entropy source as the
// reference does.  The overloads without a destination return seal_b200::Serializable<...> (serializable.hpp): the seed-compressed
// stream KeyGenerator's Serializable<...> would save, written on the device (sb200_public_key_generate_seeded,
// sb200_kswitch_keys_generate_seeded) with c_1 never leaving it, from seeds drawn as the destination overloads draw them.
// Secret-key sampling stays with seal::KeyGenerator, deliberately.
#pragma once

#include "../seal_b200.h"
#include "evaluator.hpp"
#include "serializable.hpp"
#include "seal/seal.h"
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <vector>

namespace seal_b200
{
    class KeyGenerator
    {
    public:
        // keygenerator.cpp:35-52; the device context is owned by this object
        KeyGenerator(const seal::SEALContext &context, const seal::SecretKey &secret_key, int device = 0)
            : KeyGenerator(context, secret_key, nullptr, device)
        {
        }
        // shares the device context of an existing evaluator, which must outlive this object
        KeyGenerator(const seal::SEALContext &context, const seal::SecretKey &secret_key, const Evaluator &evaluator)
            : KeyGenerator(context, secret_key, &evaluator, 0)
        {
        }
        ~KeyGenerator()
        {
            if (key_)
                sb200_secret_key_destroy(key_);
        }
        KeyGenerator(const KeyGenerator &) = delete;
        KeyGenerator &operator=(const KeyGenerator &) = delete;

        const seal::SecretKey &secret_key() const { return secret_key_; }

        // keygenerator.h:68-71 -> generate_pk (keygenerator.cpp:96-120)
        void create_public_key(seal::PublicKey &destination) const
        {
            auto &cd = *context_.key_context_data();
            int prng = 0;
            std::vector<std::uint64_t> seed = bootstrap_seeds(1, prng);
            seal::PublicKey pk;
            prepare(cd, pk);
            const int rc = sb200_public_key_generate(ctx_, key_, prng, ciphertext_prng(), seed.data(), pk.data().data(), nullptr);
            seal::util::seal_memzero(seed.data(), seed.size() * sizeof(std::uint64_t)); // the seeds determine the noise
            status(rc);
            pk.parms_id() = cd.parms_id();
            destination = std::move(pk);
        }
        // keygenerator.h:97-100 -> create_relin_keys(1, false) (keygenerator.cpp:122-161)
        void create_relin_keys(seal::RelinKeys &destination)
        {
            seal::RelinKeys rk;
            rk.data().resize(1);
            generate_one(0, rk.data()[0]);
            rk.parms_id() = context_.key_parms_id();
            destination = std::move(rk);
        }
        // keygenerator.h:145-148 -> create_galois_keys(galois_elts, false) (keygenerator.cpp:163-226)
        void create_galois_keys(const std::vector<std::uint32_t> &galois_elts, seal::GaloisKeys &destination)
        {
            const std::size_t n = context_.key_context_data()->parms().poly_modulus_degree();
            seal::GaloisKeys gk;
            gk.data().resize(n); // the largest number of keys is the number of coefficients
            for (const std::uint32_t elt : galois_elts)
            {
                if (!(elt & 1) || elt >= 2 * n)
                    throw std::invalid_argument("Galois element is not valid");
                if (gk.has_key(elt))
                    continue;
                generate_one(elt, gk.data()[seal::GaloisKeys::get_index(elt)]);
            }
            gk.parms_id() = context_.key_parms_id();
            destination = std::move(gk);
        }
        // keygenerator.h:202-209
        void create_galois_keys(const std::vector<int> &steps, seal::GaloisKeys &destination)
        {
            if (!context_.key_context_data()->qualifiers().using_batching)
                throw std::logic_error("encryption parameters do not support batching");
            create_galois_keys(context_.key_context_data()->galois_tool()->get_elts_from_steps(steps), destination);
        }
        // keygenerator.h:261-264
        void create_galois_keys(seal::GaloisKeys &destination)
        {
            create_galois_keys(context_.key_context_data()->galois_tool()->get_elts_all(), destination);
        }

        // ---- device key sets: the same keys, from the same seed draws, made on the device and kept there (sb200_kswitch_key_generate
        // with no host copy).  The keys belong to this generator's device context: to use them with an Evaluator, construct the
        // generator with that Evaluator. ----
        void create_relin_keys(DeviceRelinKeys &destination)
        {
            std::vector<sb200_kswitch_key *> keys(1, nullptr);
            generate_device(0, keys[0]);
            destination.assign(ctx_, context_.key_parms_id(), std::move(keys));
        }
        void create_galois_keys(const std::vector<std::uint32_t> &galois_elts, DeviceGaloisKeys &destination)
        {
            const std::size_t n = context_.key_context_data()->parms().poly_modulus_degree();
            std::vector<sb200_kswitch_key *> keys(n, nullptr);
            try
            {
                for (const std::uint32_t elt : galois_elts)
                {
                    if (!(elt & 1) || elt >= 2 * n)
                        throw std::invalid_argument("Galois element is not valid");
                    sb200_kswitch_key *&slot = keys[seal::GaloisKeys::get_index(elt)];
                    if (!slot)
                        generate_device(elt, slot);
                }
            }
            catch (...)
            {
                for (sb200_kswitch_key *k : keys)
                    if (k)
                        sb200_kswitch_key_destroy(k);
                throw;
            }
            destination.assign(ctx_, context_.key_parms_id(), std::move(keys));
        }
        void create_galois_keys(const std::vector<int> &steps, DeviceGaloisKeys &destination)
        {
            if (!context_.key_context_data()->qualifiers().using_batching)
                throw std::logic_error("encryption parameters do not support batching");
            create_galois_keys(context_.key_context_data()->galois_tool()->get_elts_from_steps(steps), destination);
        }
        void create_galois_keys(DeviceGaloisKeys &destination)
        {
            create_galois_keys(context_.key_context_data()->galois_tool()->get_elts_all(), destination);
        }

        // ---- Serializable overloads (keygenerator.h:73-76, 102-105, 160-163, 216-223, 270-273): seeded streams ----
        Serializable<seal::PublicKey> create_public_key() const
        {
            const std::size_t k = context_.key_context_data()->parms().coeff_modulus().size();
            int prng = 0;
            std::vector<std::uint64_t> seed = bootstrap_seeds(1, prng);
            std::vector<std::uint8_t> bytes(sb200_ciphertext_save_seeded_size(ctx_, k));
            const int rc = sb200_public_key_generate_seeded(ctx_, key_, prng, ciphertext_prng(), seed.data(), bytes.data(), bytes.size(), nullptr);
            seal::util::seal_memzero(seed.data(), seed.size() * sizeof(std::uint64_t));
            status(rc);
            return Serializable<seal::PublicKey>(std::move(bytes));
        }
        Serializable<seal::RelinKeys> create_relin_keys()
        {
            if (!context_.using_keyswitching())
                throw std::logic_error("keyswitching is not supported by the context");
            return Serializable<seal::RelinKeys>(seeded_keys({ 0 }));
        }
        Serializable<seal::GaloisKeys> create_galois_keys(const std::vector<std::uint32_t> &galois_elts)
        {
            if (!context_.using_keyswitching())
                throw std::logic_error("keyswitching is not supported by the context");
            const std::size_t n = context_.key_context_data()->parms().poly_modulus_degree();
            for (const std::uint32_t elt : galois_elts)
                if (!(elt & 1) || elt >= 2 * n)
                    throw std::invalid_argument("Galois element is not valid");
            return Serializable<seal::GaloisKeys>(seeded_keys(galois_elts));
        }
        Serializable<seal::GaloisKeys> create_galois_keys(const std::vector<int> &steps)
        {
            if (!context_.key_context_data()->qualifiers().using_batching)
                throw std::logic_error("encryption parameters do not support batching");
            return create_galois_keys(context_.key_context_data()->galois_tool()->get_elts_from_steps(steps));
        }
        Serializable<seal::GaloisKeys> create_galois_keys()
        {
            return create_galois_keys(context_.key_context_data()->galois_tool()->get_elts_all());
        }

    private:
        // the stream of the keys for `elts` ({0}: relinearization), one bootstrap seed per digit of every distinct element, drawn in
        // that order (generate_one_kswitch_key for each element, duplicates skipped)
        std::vector<std::uint8_t> seeded_keys(const std::vector<std::uint32_t> &elts)
        {
            std::vector<std::uint32_t> distinct;
            for (const std::uint32_t e : elts)
                if (std::find(distinct.begin(), distinct.end(), e) == distinct.end())
                    distinct.push_back(e);
            const std::size_t digits = context_.first_context_data()->parms().coeff_modulus().size();
            const std::uint32_t none = 0;
            const std::uint32_t *e = elts.empty() ? &none : elts.data(); // an empty list: a GaloisKeys object without keys
            std::vector<std::uint8_t> bytes(sb200_kswitch_keys_save_seeded_size(ctx_, e, elts.size()));
            int prng = 0;
            std::vector<std::uint64_t> seeds = bootstrap_seeds(distinct.size() * digits, prng);
            if (distinct.empty())
                prng = 1; // nothing is drawn or generated: an empty GaloisKeys object
            const int rc = sb200_kswitch_keys_generate_seeded(ctx_, key_, e, elts.size(), prng, ciphertext_prng(), seeds.data(),
                                                              bytes.data(), bytes.size());
            seal::util::seal_memzero(seeds.data(), seeds.size() * sizeof(std::uint64_t));
            status(rc);
            return bytes;
        }
        KeyGenerator(const seal::SEALContext &context, const seal::SecretKey &secret_key, const Evaluator *evaluator, int device)
            : context_(context)
        {
            if (!context_.parameters_set())
                throw std::invalid_argument("encryption parameters are not set correctly");
            if (!seal::is_valid_for(secret_key, context_))
                throw std::invalid_argument("secret key is not valid for encryption parameters");
            if (!evaluator)
                own_ = std::make_unique<Evaluator>(context_, device), evaluator = own_.get();
            ctx_ = evaluator->native_handle();
            secret_key_ = secret_key;
            status(sb200_secret_key_create(ctx_, secret_key_.data().data(), &key_));
        }

        // generate_one_kswitch_key (keygenerator.cpp:327-360): k - 1 digits at the key level, one bootstrap seed each
        void generate_one(std::uint32_t galois_elt, std::vector<seal::PublicKey> &destination)
        {
            if (!context_.using_keyswitching())
                throw std::logic_error("keyswitching is not supported by the context");
            auto &cd = *context_.key_context_data();
            const std::size_t digits = context_.first_context_data()->parms().coeff_modulus().size();
            const std::size_t words = 2 * cd.parms().coeff_modulus().size() * cd.parms().poly_modulus_degree();
            int prng = 0;
            std::vector<std::uint64_t> seeds = bootstrap_seeds(digits, prng);
            std::vector<std::uint64_t> h(digits * words);
            const int rc = sb200_kswitch_key_generate(ctx_, key_, galois_elt, prng, ciphertext_prng(), seeds.data(), h.data(), nullptr);
            seal::util::seal_memzero(seeds.data(), seeds.size() * sizeof(std::uint64_t));
            status(rc);
            destination.resize(digits);
            for (std::size_t j = 0; j < digits; j++)
            {
                prepare(cd, destination[j]);
                std::memcpy(destination[j].data().data(), h.data() + j * words, words * sizeof(std::uint64_t));
            }
        }
        // generate_one_kswitch_key with the key left on the device: the same seed draws as generate_one
        void generate_device(std::uint32_t galois_elt, sb200_kswitch_key *&out)
        {
            if (!context_.using_keyswitching())
                throw std::logic_error("keyswitching is not supported by the context");
            const std::size_t digits = context_.first_context_data()->parms().coeff_modulus().size();
            int prng = 0;
            std::vector<std::uint64_t> seeds = bootstrap_seeds(digits, prng);
            const int rc = sb200_kswitch_key_generate(ctx_, key_, galois_elt, prng, ciphertext_prng(), seeds.data(), nullptr, &out);
            seal::util::seal_memzero(seeds.data(), seeds.size() * sizeof(std::uint64_t));
            status(rc);
        }
        // the destination of util::encrypt_zero_symmetric at the key level with is_ntt_form = true (util/rlwe.cpp:282-287)
        void prepare(const seal::SEALContext::ContextData &cd, seal::PublicKey &pk) const
        {
            pk.data().resize(context_, cd.parms_id(), 2);
            pk.data().is_ntt_form() = true;
            pk.data().scale() = 1.0;
            pk.data().correction_factor() = 1;
        }

        // the bootstrap seeds of `count` encryptions, drawn from the key level's random generator factory as util/rlwe.cpp:288-292
        // draws them, and the prng_type of their PRNGs (encryptor.hpp: Encryptor::bootstrap_seeds)
        std::vector<std::uint64_t> bootstrap_seeds(std::size_t count, int &type) const
        {
            auto factory = context_.key_context_data()->parms().random_generator();
            if (!factory)
                factory = seal::UniformRandomGeneratorFactory::DefaultFactory();
            std::vector<std::uint64_t> seeds(count * 8);
            for (std::size_t b = 0; b < count; b++)
            {
                auto prng = factory->create();
                type = prng_type_of(*prng);
                const seal::prng_seed_type seed = prng->seed();
                static_assert(sizeof(seed) == 64, "prng_seed_type is 512 bits");
                std::memcpy(seeds.data() + b * 8, seed.data(), 64);
            }
            return seeds;
        }
        // c_1 is expanded with the default factory's PRNG (util/rlwe.cpp:329)
        static int ciphertext_prng()
        {
            return prng_type_of(*seal::UniformRandomGeneratorFactory::DefaultFactory()->create());
        }
        static int prng_type_of(seal::UniformRandomGenerator &prng)
        {
            const seal::prng_type t = prng.info().type();
            if (t != seal::prng_type::blake2xb && t != seal::prng_type::shake256)
                throw std::logic_error("unsupported prng_type: the device path implements Blake2xbPRNG and Shake256PRNG");
            return static_cast<int>(t);
        }
        static void status(int rc)
        {
            if (rc == SB200_OK)
                return;
            const std::string msg = sb200_last_error();
            if (rc == SB200_E_INVALID_ARG || rc == SB200_E_POINTER)
                throw std::invalid_argument(msg);
            if (rc == SB200_E_LOGIC)
                throw std::logic_error(msg);
            throw std::runtime_error(msg);
        }

        seal::SEALContext context_;
        std::unique_ptr<Evaluator> own_;
        sb200_context *ctx_ = nullptr;
        sb200_secret_key *key_ = nullptr;
        seal::SecretKey secret_key_;
    };
} // namespace seal_b200
