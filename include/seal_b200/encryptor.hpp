// include/seal_b200/encryptor.hpp -- same-signature stand-in for seal::Encryptor (native/src/seal/encryptor.h:113-380: encrypt /
// encrypt_zero with a public key, encrypt_symmetric / encrypt_zero_symmetric with a secret key, destination overloads) over the
// C-ABI of include/seal_b200.h.
//
//     seal_b200::Encryptor encryptor(context, public_key, evaluator);   // or (context, secret_key, evaluator), or both keys
//     encryptor.encrypt(plain, ct);  encryptor.encrypt_symmetric(plain, ct);
//
// The PRNG stream (Blake2xb or SHAKE256), the uniform polynomial, the centred binomial noise and c_0 = -(c_1 s + e) run on the
// device (sb200_encrypt_zero_symmetric_prng); the bootstrap seed of every encryption is drawn from the context's own random
// generator factory (parms.random_generator()->create(), util/rlwe.cpp:288-292), whose PRNG type the device follows, so a context
// with a seeded factory (Blake2xbPRNGFactory or Shake256PRNGFactory) reproduces the reference's ciphertexts bit for bit and the
// default factory draws from the OS entropy source as the reference does.  c_1 is expanded with the PRNG type of
// UniformRandomGeneratorFactory::DefaultFactory() (util/rlwe.cpp:329), i.e. of the reference this header is compiled against.
// Public-key encryption (ternary u, two noise polynomials, the sample one level up divided down:
// sb200_encrypt_zero_asymmetric_prng) follows the same rule.  Only a custom factory (prng_type::unknown) is rejected.
// The plaintext is added by the evaluator's device path.  The Serializable<Ciphertext> overloads (seeded output) stay with
// seal::Encryptor: Serializable<> cannot be constructed outside the reference.
#pragma once

#include "../seal_b200.h"
#include "evaluator.hpp"
#include "seal/seal.h"
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <vector>

namespace seal_b200
{
    class Encryptor
    {
    public:
        // shares the device context of an existing evaluator, which must outlive this object
        Encryptor(const seal::SEALContext &context, const seal::SecretKey &secret_key, const Evaluator &evaluator)
            : context_(context), ctx_(evaluator.native_handle())
        {
            if (!context_.parameters_set())
                throw std::invalid_argument("encryption parameters are not set correctly"); // encryptor.cpp:23-27
            if (!seal::is_valid_for(secret_key, context_))
                throw std::invalid_argument("secret key is not valid for encryption parameters"); // encryptor.cpp:76-80
            status(sb200_secret_key_create(ctx_, secret_key.data().data(), &key_));
        }
        Encryptor(const seal::SEALContext &context, const seal::PublicKey &public_key, const Evaluator &evaluator)
            : context_(context), ctx_(evaluator.native_handle())
        {
            if (!context_.parameters_set())
                throw std::invalid_argument("encryption parameters are not set correctly");
            set_public_key(public_key);
        }
        Encryptor(const seal::SEALContext &context, const seal::PublicKey &public_key, const seal::SecretKey &secret_key, const Evaluator &evaluator)
            : Encryptor(context, secret_key, evaluator)
        {
            set_public_key(public_key);
        }
        ~Encryptor()
        {
            if (key_)
                sb200_secret_key_destroy(key_);
            if (pk_)
                sb200_public_key_destroy(pk_);
        }
        // encryptor.h:164-173
        void set_public_key(const seal::PublicKey &public_key)
        {
            if (!seal::is_valid_for(public_key, context_))
                throw std::invalid_argument("public key is not valid for encryption parameters"); // encryptor.cpp:63-66
            if (pk_)
                sb200_public_key_destroy(pk_), pk_ = nullptr;
            status(sb200_public_key_create(ctx_, public_key.data().data(), &pk_));
        }

        // encryptor.h:113-140, 196-244 (public key)
        void encrypt(const seal::Plaintext &plain, seal::Ciphertext &destination, seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            std::vector<seal::Ciphertext> one(1);
            encrypt_batch(&plain, 1, one.data(), pool, true);
            destination = std::move(one[0]);
        }
        void encrypt(const std::vector<seal::Plaintext> &plains, std::vector<seal::Ciphertext> &destination,
                     seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination.resize(plains.size());
            if (!plains.empty())
                encrypt_batch(plains.data(), plains.size(), destination.data(), pool, true);
        }
        void encrypt_zero(seal::parms_id_type parms_id, seal::Ciphertext &destination, seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            std::vector<seal::Ciphertext> one(1);
            zero_batch(parms_id, 1, one.data(), nullptr, pool, true);
            destination = std::move(one[0]);
        }
        void encrypt_zero(seal::Ciphertext &destination, seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            encrypt_zero(context_.first_parms_id(), destination, std::move(pool));
        }
        Encryptor(const Encryptor &) = delete;
        Encryptor &operator=(const Encryptor &) = delete;

        // encryptor.h:327-351, 376-380
        void encrypt_zero_symmetric(seal::parms_id_type parms_id, seal::Ciphertext &destination,
                                    seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            std::vector<seal::Ciphertext> one(1);
            zero_batch(parms_id, 1, one.data(), nullptr, pool, false);
            destination = std::move(one[0]);
        }
        void encrypt_zero_symmetric(seal::Ciphertext &destination, seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            encrypt_zero_symmetric(context_.first_parms_id(), destination, std::move(pool));
        }
        // encryptor.h:273-300 -> Encryptor::encrypt_internal (encryptor.cpp:176-340)
        void encrypt_symmetric(const seal::Plaintext &plain, seal::Ciphertext &destination,
                               seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            std::vector<seal::Ciphertext> one(1);
            encrypt_batch(&plain, 1, one.data(), pool, false);
            destination = std::move(one[0]);
        }
        // ---- batch: B plaintexts of one level -> B fresh ciphertexts, one launch sequence for all of them ----
        void encrypt_symmetric(const std::vector<seal::Plaintext> &plains, std::vector<seal::Ciphertext> &destination,
                               seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination.resize(plains.size());
            if (!plains.empty())
                encrypt_batch(plains.data(), plains.size(), destination.data(), pool, false);
        }

    private:
        struct DeviceSlab
        {
            sb200_context *ctx;
            std::uint64_t *d = nullptr;
            DeviceSlab(sb200_context *c, std::size_t words) : ctx(c)
            {
                status(sb200_device_malloc(ctx, words * sizeof(std::uint64_t), &d));
            }
            ~DeviceSlab()
            {
                if (d)
                    sb200_device_free(ctx, d);
            }
            DeviceSlab(const DeviceSlab &) = delete;
            DeviceSlab &operator=(const DeviceSlab &) = delete;
        };

        // the bootstrap seeds of `count` encryptions, drawn exactly where the reference draws them (util/rlwe.cpp:288-292), and the
        // prng_type of their PRNGs (1 = blake2xb, 2 = shake256)
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
        static int prng_type_of(seal::UniformRandomGenerator &prng)
        {
            const seal::prng_type t = prng.info().type();
            if (t != seal::prng_type::blake2xb && t != seal::prng_type::shake256)
                throw std::logic_error("unsupported prng_type: the device path implements Blake2xbPRNG and Shake256PRNG");
            return static_cast<int>(t);
        }

        // encrypt_zero_internal (encryptor.cpp:88-174, symmetric branch) for `count` ciphertexts into a device slab that is either
        // downloaded here (d_keep == nullptr) or handed to the caller for the plaintext addition
        void zero_batch(seal::parms_id_type parms_id, std::size_t count, seal::Ciphertext *out, DeviceSlab *d_keep, const seal::MemoryPoolHandle &pool,
                        bool is_asymmetric) const
        {
            if (!pool)
                throw std::invalid_argument("pool is uninitialized");
            if (is_asymmetric && !pk_)
                throw std::logic_error("public key is not set"); // encryptor.cpp:181-187
            if (!is_asymmetric && !key_)
                throw std::logic_error("secret key is not set");
            auto cd = context_.get_context_data(parms_id);
            if (!cd)
                throw std::invalid_argument("parms_id is not valid for encryption parameters");
            auto &parms = cd->parms();
            const std::size_t L = parms.coeff_modulus().size(), n = parms.poly_modulus_degree(), words = 2 * L * n;
            int prng = 0;
            std::vector<std::uint64_t> seeds = bootstrap_seeds(count, prng);
            const int ct_prng = prng_type_of(*seal::UniformRandomGeneratorFactory::DefaultFactory()->create());
            DeviceSlab local(ctx_, d_keep ? 1 : count * words);
            std::uint64_t *d = d_keep ? d_keep->d : local.d;
            if (is_asymmetric)
                status(sb200_encrypt_zero_asymmetric_prng(ctx_, pk_, L, count, prng, seeds.data(), d, nullptr));
            else
                status(sb200_encrypt_zero_symmetric_prng(ctx_, key_, L, count, prng, ct_prng, seeds.data(), 0, d, nullptr, nullptr));
            seal::util::seal_memzero(seeds.data(), seeds.size() * sizeof(std::uint64_t)); // the seeds determine the noise
            const bool ntt = parms.scheme() != seal::scheme_type::bfv;
            for (std::size_t b = 0; b < count; b++)
            {
                out[b].resize(context_, parms_id, 2); // rlwe.cpp:282-287
                out[b].is_ntt_form() = ntt;
                out[b].scale() = 1.0;
                out[b].correction_factor() = 1;
            }
            if (!d_keep)
                download(d, count, words, out);
        }
        void download(const std::uint64_t *d, std::size_t count, std::size_t words, seal::Ciphertext *out) const
        {
            status(sb200_stream_synchronize(ctx_, nullptr));
            for (std::size_t b = 0; b < count; b++)
                status(sb200_memcpy_d2h(ctx_, out[b].data(), d + b * words, words * sizeof(std::uint64_t), nullptr));
            status(sb200_stream_synchronize(ctx_, nullptr));
        }

        void encrypt_batch(const seal::Plaintext *plains, std::size_t count, seal::Ciphertext *out, const seal::MemoryPoolHandle &pool,
                           bool is_asymmetric) const
        {
            if (is_asymmetric && !pk_)
                throw std::logic_error("public key is not set"); // encryptor.cpp:181-194
            if (!is_asymmetric && !key_)
                throw std::logic_error("secret key is not set");
            const auto scheme = context_.key_context_data()->parms().scheme();
            for (std::size_t b = 0; b < count; b++)
            {
                if (!seal::is_valid_for(plains[b], context_))
                    throw std::invalid_argument("plain is not valid for encryption parameters"); // encryptor.cpp:196-200
                if (scheme == seal::scheme_type::ckks && !plains[b].is_ntt_form())
                    throw std::invalid_argument("plain must be in NTT form");
                if (scheme != seal::scheme_type::ckks && plains[b].is_ntt_form())
                    throw std::invalid_argument("plain cannot be in NTT form");
                if (scheme == seal::scheme_type::ckks && plains[b].parms_id() != plains[0].parms_id())
                    throw std::invalid_argument("batch members must share parms_id");
            }
            const seal::parms_id_type parms_id = scheme == seal::scheme_type::ckks ? plains[0].parms_id() : context_.first_parms_id();
            auto cd = context_.get_context_data(parms_id);
            if (!cd)
                throw std::invalid_argument("plain is not valid for encryption parameters");
            const std::size_t L = cd->parms().coeff_modulus().size(), n = cd->parms().poly_modulus_degree(), words = 2 * L * n;
            DeviceSlab ct(ctx_, count * words);
            zero_batch(parms_id, count, out, &ct, pool, is_asymmetric);
            if (scheme == seal::scheme_type::ckks)
            {
                // c_0 += plain (encryptor.cpp:231-236): the plaintexts go up as a [count][1][L][n] slab and are added row by row
                DeviceSlab p(ctx_, count * L * n);
                for (std::size_t b = 0; b < count; b++)
                    status(sb200_memcpy_h2d(ctx_, p.d + b * L * n, plains[b].data(), L * n * sizeof(std::uint64_t), nullptr));
                for (std::size_t b = 0; b < count; b++)
                    status(sb200_add(ctx_, L, 1, 1, ct.d + b * words, p.d + b * L * n, ct.d + b * words, nullptr));
                for (std::size_t b = 0; b < count; b++)
                    out[b].scale() = plains[b].scale();
            }
            else
            {
                // BFV: c_0 += round(q m / t) (multiply_add_plain_with_scaling_variant, encryptor.cpp:211-214);
                // BGV: c_0 += NTT(lift(m)) (encryptor.cpp:250-330)
                std::vector<std::uint64_t> coeffs(count * n, 0);
                for (std::size_t b = 0; b < count; b++)
                    std::copy_n(plains[b].data(), plains[b].coeff_count(), coeffs.begin() + b * n);
                DeviceSlab p(ctx_, count * n);
                status(sb200_memcpy_h2d(ctx_, p.d, coeffs.data(), coeffs.size() * sizeof(std::uint64_t), nullptr));
                status(sb200_add_plain_coeff(ctx_, L, 2, count, 0, ct.d, p.d, nullptr, ct.d, nullptr));
            }
            download(ct.d, count, words, out);
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
        sb200_context *ctx_ = nullptr;
        sb200_secret_key *key_ = nullptr;
        sb200_public_key *pk_ = nullptr;
    };
} // namespace seal_b200
