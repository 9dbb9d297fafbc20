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
// The plaintext is added on the device by the encryption entry points themselves (sb200_encrypt_symmetric / _asymmetric); device-
// resident PlaintextBatch -> CiphertextBatch overloads keep the whole path on the GPU.  The overloads without a destination return
// seal_b200::Serializable<seal::Ciphertext> (serializable.hpp) as the reference's do: seeded for the symmetric ones (c_0 and the seed of
// c_1, sb200_ciphertext_save_seeded), the full ciphertext for the public-key ones (sb200_ciphertext_save).
#pragma once

#include "../seal_b200.h"
#include "evaluator.hpp"
#include "serializable.hpp"
#include "seal/seal.h"
#include <algorithm>
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
            zero_batch(parms_id, 1, one.data(), pool, true);
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
            zero_batch(parms_id, 1, one.data(), pool, false);
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

        // ---- device-resident batches: PlaintextBatch -> CiphertextBatch, nothing crosses PCIe but the seeds ----
        // Encryptor::encrypt_internal (encryptor.cpp:176-340) for every member, with its checks and messages, all made before anything
        // is written; the plaintext is added on the device (sb200_encrypt_asymmetric / sb200_encrypt_symmetric).  The seeds come from the
        // context's factory, one per ciphertext in member order, as the single-ciphertext overloads draw them.  The result carries the
        // reference's metadata: parms_id the plaintext's (CKKS) or first_parms_id (BFV / BGV), size 2, NTT form for CKKS / BGV, the
        // plaintext's scale (CKKS) or 1, correction factor 1.  The batches must belong to this encryptor's evaluator.
        void encrypt(const PlaintextBatch &plain, CiphertextBatch &destination) const
        {
            encrypt_device(plain, destination, true);
        }
        void encrypt_symmetric(const PlaintextBatch &plain, CiphertextBatch &destination) const
        {
            encrypt_device(plain, destination, false);
        }
        // `count` encryptions of zero at parms_id into a device batch
        void encrypt_zero(seal::parms_id_type parms_id, std::size_t count, CiphertextBatch &destination) const
        {
            zero_device(parms_id, count, destination, true);
        }
        void encrypt_zero_symmetric(seal::parms_id_type parms_id, std::size_t count, CiphertextBatch &destination) const
        {
            zero_device(parms_id, count, destination, false);
        }

        // ---- Serializable overloads (encryptor.h:142-162, 246-266, 302-317, 353-375) ----
        Serializable<seal::Ciphertext> encrypt(const seal::Plaintext &plain, seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            return serial(&plain, context_.first_parms_id(), pool, true);
        }
        Serializable<seal::Ciphertext> encrypt_zero(seal::parms_id_type parms_id, seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            return serial(nullptr, parms_id, pool, true);
        }
        Serializable<seal::Ciphertext> encrypt_zero(seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            return serial(nullptr, context_.first_parms_id(), pool, true);
        }
        Serializable<seal::Ciphertext> encrypt_symmetric(const seal::Plaintext &plain,
                                                         seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            return serial(&plain, context_.first_parms_id(), pool, false);
        }
        Serializable<seal::Ciphertext> encrypt_zero_symmetric(seal::parms_id_type parms_id,
                                                              seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            return serial(nullptr, parms_id, pool, false);
        }
        Serializable<seal::Ciphertext> encrypt_zero_symmetric(seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            return serial(nullptr, context_.first_parms_id(), pool, false);
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
        void check_key(bool is_asymmetric) const
        {
            if (is_asymmetric && !pk_)
                throw std::logic_error("public key is not set"); // encryptor.cpp:181-194
            if (!is_asymmetric && !key_)
                throw std::logic_error("secret key is not set");
        }

        // `count` encryptions at the level with L primes into the device slab d_out [count][2][L][n]: of the device plaintexts d_plain
        // (layout of sb200_encrypt_symmetric), or of zero when d_plain is null.  Seeds from the context's factory, wiped afterwards.
        // public_seeds (symmetric only): nullptr, or [count][8] = the seeds of c_1, with the ciphertexts made for a seeded stream
        // (save_seed: the Serializable<Ciphertext> variant)
        void launch(std::size_t L, std::size_t count, const std::uint64_t *d_plain, bool is_asymmetric, std::uint64_t *d_out,
                    std::uint64_t *public_seeds = nullptr) const
        {
            int prng = 0;
            std::vector<std::uint64_t> seeds = bootstrap_seeds(count, prng);
            const int ct_prng = ciphertext_prng();
            const int save_seed = public_seeds ? 1 : 0;
            int rc;
            if (is_asymmetric)
                rc = d_plain ? sb200_encrypt_asymmetric(ctx_, pk_, L, count, d_plain, prng, seeds.data(), d_out, nullptr)
                             : sb200_encrypt_zero_asymmetric_prng(ctx_, pk_, L, count, prng, seeds.data(), d_out, nullptr);
            else
                rc = d_plain ? sb200_encrypt_symmetric(ctx_, key_, L, count, d_plain, prng, ct_prng, seeds.data(), save_seed, d_out, public_seeds,
                                                       nullptr)
                             : sb200_encrypt_zero_symmetric_prng(ctx_, key_, L, count, prng, ct_prng, seeds.data(), save_seed, d_out,
                                                                 public_seeds, nullptr);
            seal::util::seal_memzero(seeds.data(), seeds.size() * sizeof(std::uint64_t)); // the seeds determine the noise
            status(rc);
        }
        // storage and metadata of `count` fresh ciphertexts at parms_id (rlwe.cpp:282-287; encrypt_internal's scale)
        void shape(CiphertextBatch &b, std::size_t count, seal::parms_id_type parms_id, std::size_t L, std::size_t n, double scale) const
        {
            const std::size_t words = count * 2 * L * n;
            if (b.ctx_ != ctx_)
            {
                b.release();
                b.ctx_ = ctx_;
            }
            if (b.cap_ < words)
            {
                b.release();
                status(sb200_device_malloc(ctx_, words * sizeof(std::uint64_t), &b.d_));
                b.cap_ = words;
            }
            b.batch_ = count, b.size_ = 2, b.L_ = L, b.n_ = n;
            b.parms_id_ = parms_id, b.ntt_ = context_.key_context_data()->parms().scheme() != seal::scheme_type::bfv;
            b.scale_ = scale, b.cf_ = 1;
        }
        // encrypt_internal's checks (encryptor.cpp:179-242) -> the parms_id of the result
        seal::parms_id_type check_plain(bool ntt, seal::parms_id_type parms_id) const
        {
            const auto scheme = context_.key_context_data()->parms().scheme();
            if (scheme == seal::scheme_type::ckks)
            {
                if (!ntt)
                    throw std::invalid_argument("plain must be in NTT form");
                if (!context_.get_context_data(parms_id))
                    throw std::invalid_argument("plain is not valid for encryption parameters");
                return parms_id;
            }
            if (ntt)
                throw std::invalid_argument("plain cannot be in NTT form");
            return context_.first_parms_id();
        }

        void encrypt_device(const PlaintextBatch &plain, CiphertextBatch &destination, bool is_asymmetric) const
        {
            check_key(is_asymmetric);
            if (plain.ctx_ != ctx_ || !plain.d_ || !plain.batch_)
                throw std::invalid_argument("plain is not valid for encryption parameters");
            if (!plain.ntt_ && plain.n_ != context_.key_context_data()->parms().poly_modulus_degree())
                throw std::invalid_argument("plain is not valid for encryption parameters");
            const seal::parms_id_type parms_id = check_plain(plain.ntt_, plain.parms_id_);
            auto cd = context_.get_context_data(parms_id);
            const std::size_t L = cd->parms().coeff_modulus().size(), n = cd->parms().poly_modulus_degree();
            const double scale = plain.ntt_ ? plain.scale_ : 1.0;
            shape(destination, plain.batch_, parms_id, L, n, scale);
            launch(L, plain.batch_, plain.d_, is_asymmetric, destination.d_);
        }
        void zero_device(seal::parms_id_type parms_id, std::size_t count, CiphertextBatch &destination, bool is_asymmetric) const
        {
            check_key(is_asymmetric);
            auto cd = context_.get_context_data(parms_id);
            if (!cd)
                throw std::invalid_argument("parms_id is not valid for encryption parameters");
            if (!count)
                throw std::invalid_argument("batch cannot be empty");
            const std::size_t L = cd->parms().coeff_modulus().size(), n = cd->parms().poly_modulus_degree();
            shape(destination, count, parms_id, L, n, 1.0);
            launch(L, count, nullptr, is_asymmetric, destination.d_);
        }

        // encrypt_zero_internal (encryptor.cpp:88-174) for `count` ciphertexts, downloaded into out
        void zero_batch(seal::parms_id_type parms_id, std::size_t count, seal::Ciphertext *out, const seal::MemoryPoolHandle &pool,
                        bool is_asymmetric) const
        {
            if (!pool)
                throw std::invalid_argument("pool is uninitialized");
            check_key(is_asymmetric);
            auto cd = context_.get_context_data(parms_id);
            if (!cd)
                throw std::invalid_argument("parms_id is not valid for encryption parameters");
            const std::size_t L = cd->parms().coeff_modulus().size(), n = cd->parms().poly_modulus_degree(), words = 2 * L * n;
            DeviceSlab d(ctx_, count * words);
            launch(L, count, nullptr, is_asymmetric, d.d);
            download(d.d, count, parms_id, words, 1.0, out);
        }
        void download(const std::uint64_t *d, std::size_t count, seal::parms_id_type parms_id, std::size_t words, double scale,
                      seal::Ciphertext *out) const
        {
            const bool ntt = context_.key_context_data()->parms().scheme() != seal::scheme_type::bfv;
            for (std::size_t b = 0; b < count; b++)
            {
                out[b].resize(context_, parms_id, 2); // rlwe.cpp:282-287
                out[b].is_ntt_form() = ntt;
                out[b].scale() = scale;
                out[b].correction_factor() = 1;
            }
            status(sb200_stream_synchronize(ctx_, nullptr));
            for (std::size_t b = 0; b < count; b++)
                status(sb200_memcpy_d2h(ctx_, out[b].data(), d + b * words, words * sizeof(std::uint64_t), nullptr));
            status(sb200_stream_synchronize(ctx_, nullptr));
        }

        // one slab upload of the plaintexts, one encryption call, one download
        void encrypt_batch(const seal::Plaintext *plains, std::size_t count, seal::Ciphertext *out, const seal::MemoryPoolHandle &pool,
                           bool is_asymmetric) const
        {
            check_key(is_asymmetric);
            const auto scheme = context_.key_context_data()->parms().scheme();
            for (std::size_t b = 0; b < count; b++)
            {
                if (!seal::is_valid_for(plains[b], context_))
                    throw std::invalid_argument("plain is not valid for encryption parameters"); // encryptor.cpp:196-200
                check_plain(plains[b].is_ntt_form(), plains[b].parms_id());
                if (scheme == seal::scheme_type::ckks && plains[b].parms_id() != plains[0].parms_id())
                    throw std::invalid_argument("batch members must share parms_id");
            }
            if (!pool)
                throw std::invalid_argument("pool is uninitialized");
            const seal::parms_id_type parms_id = check_plain(plains[0].is_ntt_form(), plains[0].parms_id());
            auto cd = context_.get_context_data(parms_id);
            const std::size_t L = cd->parms().coeff_modulus().size(), n = cd->parms().poly_modulus_degree(), words = 2 * L * n;
            // CKKS: [count][L][n] NTT form; BFV / BGV: [count][n] coefficients, zero above coeff_count
            const std::size_t pw = scheme == seal::scheme_type::ckks ? L * n : n;
            std::vector<std::uint64_t> host(count * pw, 0);
            for (std::size_t b = 0; b < count; b++)
                std::copy_n(plains[b].data(), std::min(plains[b].coeff_count(), pw), host.begin() + b * pw);
            DeviceSlab p(ctx_, count * pw), ct(ctx_, count * words);
            status(sb200_memcpy_h2d(ctx_, p.d, host.data(), host.size() * sizeof(std::uint64_t), nullptr));
            launch(L, count, p.d, is_asymmetric, ct.d);
            download(ct.d, count, parms_id, words, 1.0, out);
            if (scheme == seal::scheme_type::ckks)
                for (std::size_t b = 0; b < count; b++)
                    out[b].scale() = plains[b].scale(); // encryptor.cpp:237
        }

        // one encryption (of `plain`, or of zero at parms_id) as a stream: encrypt_internal's checks and metadata (encryptor.cpp:176-340),
        // then Serializable<Ciphertext>::save(none) of the result, seeded for the symmetric forms
        Serializable<seal::Ciphertext> serial(const seal::Plaintext *plain, seal::parms_id_type parms_id, const seal::MemoryPoolHandle &pool,
                                              bool is_asymmetric) const
        {
            check_key(is_asymmetric);
            const auto scheme = context_.key_context_data()->parms().scheme();
            double scale = 1.0;
            if (plain)
            {
                if (!seal::is_valid_for(*plain, context_))
                    throw std::invalid_argument("plain is not valid for encryption parameters"); // encryptor.cpp:196-200
                parms_id = check_plain(plain->is_ntt_form(), plain->parms_id());
                if (scheme == seal::scheme_type::ckks)
                    scale = plain->scale(); // encryptor.cpp:237
            }
            else if (!context_.get_context_data(parms_id))
                throw std::invalid_argument("parms_id is not valid for encryption parameters");
            if (!pool)
                throw std::invalid_argument("pool is uninitialized");
            auto cd = context_.get_context_data(parms_id);
            const std::size_t L = cd->parms().coeff_modulus().size(), n = cd->parms().poly_modulus_degree();
            DeviceSlab ct(ctx_, 2 * L * n);
            std::vector<std::uint64_t> pub(8);
            std::uint64_t *seeds_out = is_asymmetric ? nullptr : pub.data();
            if (plain)
            {
                // CKKS: [L][n] NTT form; BFV / BGV: [n] coefficients, zero above coeff_count
                const std::size_t pw = scheme == seal::scheme_type::ckks ? L * n : n;
                std::vector<std::uint64_t> host(pw, 0);
                std::copy_n(plain->data(), std::min(plain->coeff_count(), pw), host.begin());
                DeviceSlab p(ctx_, pw);
                status(sb200_memcpy_h2d(ctx_, p.d, host.data(), host.size() * sizeof(std::uint64_t), nullptr));
                launch(L, 1, p.d, is_asymmetric, ct.d, seeds_out);
            }
            else
                launch(L, 1, nullptr, is_asymmetric, ct.d, seeds_out);
            sb200_ct_info meta{};
            meta.is_ntt_form = scheme != seal::scheme_type::bfv, meta.scale = scale, meta.correction_factor = 1;
            std::vector<std::uint8_t> bytes(is_asymmetric ? sb200_ciphertext_save_size(ctx_, L, 2) : sb200_ciphertext_save_seeded_size(ctx_, L));
            std::uint8_t *out = bytes.data();
            status(is_asymmetric ? sb200_ciphertext_save(ctx_, 1, L, 2, ct.d, &meta, &out, bytes.size(), nullptr)
                                 : sb200_ciphertext_save_seeded(ctx_, 1, L, ct.d, &meta, pub.data(), ciphertext_prng(), &out, bytes.size(), nullptr));
            return Serializable<seal::Ciphertext>(std::move(bytes));
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
