// include/seal_b200/decryptor.hpp -- same-signature stand-in for seal::Decryptor (native/src/seal/decryptor.h) over the C-ABI
// of include/seal_b200.h: decrypt (the dot product with the secret key, BFV's scale-and-round, BGV's exact base conversion on the
// device, sb200_decrypt) and invariant_noise_budget (the phase composed modulo Q and reduced to one int on the device,
// sb200_invariant_noise_budget); checks, exception types and the shape of the resulting Plaintext are the reference's
// (decryptor.cpp:53-197, :409-486).  Both also take a device-resident CiphertextBatch of the evaluator's context.
#pragma once

#include "../seal_b200.h"
#include "evaluator.hpp"
#include "seal/seal.h"
#include <algorithm>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

namespace seal_b200
{
    class Decryptor
    {
    public:
        // shares the device context of an existing evaluator, which must outlive this object
        Decryptor(const seal::SEALContext &context, const seal::SecretKey &secret_key, const Evaluator &evaluator)
            : context_(context), ctx_(evaluator.native_handle())
        {
            if (!context_.parameters_set())
                throw std::invalid_argument("encryption parameters are not set correctly");
            if (!seal::is_valid_for(secret_key, context_))
                throw std::invalid_argument("secret key is not valid for encryption parameters");
            status(sb200_secret_key_create(ctx_, secret_key.data().data(), &key_));
        }
        ~Decryptor()
        {
            if (key_)
                sb200_secret_key_destroy(key_);
        }
        Decryptor(const Decryptor &) = delete;
        Decryptor &operator=(const Decryptor &) = delete;

        void decrypt(const seal::Ciphertext &encrypted, seal::Plaintext &destination)
        {
            if (!seal::is_valid_for(encrypted, context_))
                throw std::invalid_argument("encrypted is not valid for encryption parameters");
            if (encrypted.size() < SEAL_CIPHERTEXT_SIZE_MIN)
                throw std::invalid_argument("encrypted is empty");
            const auto scheme = context_.first_context_data()->parms().scheme();
            const std::size_t L = encrypted.coeff_modulus_size(), n = encrypted.poly_modulus_degree();
            if (scheme == seal::scheme_type::bfv && encrypted.is_ntt_form())
                throw std::invalid_argument("encrypted cannot be in NTT form"); // :113-116
            if (scheme != seal::scheme_type::bfv && !encrypted.is_ntt_form())
                throw std::invalid_argument("encrypted must be in NTT form"); // :139-142, :161-164
            destination.parms_id() = seal::parms_id_zero;
            if (scheme == seal::scheme_type::ckks)
            {
                destination.resize(L * n);
                status(sb200_decrypt_host(ctx_, key_, L, encrypted.size(), 1, encrypted.data(), nullptr, destination.data()));
                destination.parms_id() = encrypted.parms_id();
                destination.scale() = encrypted.scale();
                return;
            }
            destination.resize(n);
            const std::uint64_t cf = encrypted.correction_factor();
            status(sb200_decrypt_host(ctx_, key_, L, encrypted.size(), 1, encrypted.data(), scheme == seal::scheme_type::bgv ? &cf : nullptr,
                                      destination.data()));
            // the plaintext keeps its significant coefficients only (:131-134, :193-196)
            std::size_t count = n;
            while (count > 1 && destination.data()[count - 1] == 0)
                count--;
            destination.resize(count);
        }

        // Decryptor::invariant_noise_budget (decryptor.cpp:409-486): BFV and BGV only
        int invariant_noise_budget(const seal::Ciphertext &encrypted)
        {
            if (!seal::is_valid_for(encrypted, context_))
                throw std::invalid_argument("encrypted is not valid for encryption parameters");
            if (encrypted.size() < SEAL_CIPHERTEXT_SIZE_MIN)
                throw std::invalid_argument("encrypted is empty");
            check_form(encrypted.is_ntt_form());
            int budget = 0;
            status(sb200_invariant_noise_budget_host(ctx_, key_, encrypted.coeff_modulus_size(), encrypted.size(), 1, encrypted.data(), &budget));
            return budget;
        }

        // the budget of every member of a device-resident batch, destination[i] for member i; only the ints leave the GPU
        void invariant_noise_budget(const CiphertextBatch &encrypted, std::vector<int> &destination)
        {
            owned(encrypted);
            check_form(encrypted.ntt_);
            const std::size_t B = encrypted.batch_;
            std::uint64_t *d_out = nullptr;
            status(sb200_device_malloc(ctx_, B * sizeof(int), &d_out));
            destination.assign(B, 0);
            int rc = sb200_invariant_noise_budget(ctx_, key_, encrypted.L_, encrypted.size_, B, encrypted.d_, reinterpret_cast<int *>(d_out), nullptr);
            if (rc == SB200_OK)
                rc = sb200_memcpy_d2h(ctx_, destination.data(), d_out, B * sizeof(int), nullptr);
            if (rc == SB200_OK)
                rc = sb200_stream_synchronize(ctx_, nullptr);
            const std::string msg = rc == SB200_OK ? std::string() : sb200_last_error();
            sb200_device_free(ctx_, d_out);
            status(rc, msg);
        }

        // decrypt of every member of a device-resident batch (each with the batch's correction factor), destination[i] for member i
        void decrypt(const CiphertextBatch &encrypted, std::vector<seal::Plaintext> &destination)
        {
            owned(encrypted);
            const auto scheme = context_.first_context_data()->parms().scheme();
            if (encrypted.size_ < SEAL_CIPHERTEXT_SIZE_MIN)
                throw std::invalid_argument("encrypted is empty");
            if (scheme == seal::scheme_type::bfv && encrypted.ntt_)
                throw std::invalid_argument("encrypted cannot be in NTT form");
            if (scheme != seal::scheme_type::bfv && !encrypted.ntt_)
                throw std::invalid_argument("encrypted must be in NTT form");
            const std::size_t B = encrypted.batch_, L = encrypted.L_, n = encrypted.n_;
            const bool ckks = scheme == seal::scheme_type::ckks;
            const std::size_t words = ckks ? L * n : n;
            std::vector<std::uint64_t> cf(B, encrypted.cf_);
            std::vector<std::uint64_t> plain(B * words);
            std::uint64_t *d_out = nullptr;
            status(sb200_device_malloc(ctx_, B * words * sizeof(std::uint64_t), &d_out));
            int rc = sb200_decrypt(ctx_, key_, L, encrypted.size_, B, encrypted.d_, scheme == seal::scheme_type::bgv ? cf.data() : nullptr, d_out, nullptr);
            if (rc == SB200_OK)
                rc = sb200_memcpy_d2h(ctx_, plain.data(), d_out, B * words * sizeof(std::uint64_t), nullptr);
            if (rc == SB200_OK) // the plaintexts do not stay behind on the device
                rc = sb200_memcpy_h2d(ctx_, d_out, std::vector<std::uint64_t>(B * words, 0).data(), B * words * sizeof(std::uint64_t), nullptr);
            if (rc == SB200_OK)
                rc = sb200_stream_synchronize(ctx_, nullptr);
            const std::string msg = rc == SB200_OK ? std::string() : sb200_last_error();
            sb200_device_free(ctx_, d_out);
            status(rc, msg);
            destination.resize(B);
            for (std::size_t i = 0; i < B; i++)
            {
                seal::Plaintext &p = destination[i];
                p.parms_id() = seal::parms_id_zero;
                p.resize(words);
                std::copy(plain.begin() + i * words, plain.begin() + (i + 1) * words, p.data());
                if (ckks)
                {
                    p.parms_id() = encrypted.parms_id_;
                    p.scale() = encrypted.scale_;
                    continue;
                }
                std::size_t count = n; // the significant coefficients only, as decrypt does (:131-134, :193-196)
                while (count > 1 && p.data()[count - 1] == 0)
                    count--;
                p.resize(count);
            }
            std::fill(plain.begin(), plain.end(), 0);
        }

        // decrypt of every member of a device-resident batch into a device-resident PlaintextBatch: nothing leaves the GPU.  CKKS:
        // [B][L][n] NTT form with the batch's parms_id and scale; BFV / BGV: [B][n] coefficient form, parms_id_zero (BGV with the
        // batch's correction factor).  Checks as for the vector overload above.
        void decrypt(const CiphertextBatch &encrypted, PlaintextBatch &destination)
        {
            owned(encrypted);
            const auto scheme = context_.first_context_data()->parms().scheme();
            if (encrypted.size_ < SEAL_CIPHERTEXT_SIZE_MIN)
                throw std::invalid_argument("encrypted is empty");
            if (scheme == seal::scheme_type::bfv && encrypted.ntt_)
                throw std::invalid_argument("encrypted cannot be in NTT form");
            if (scheme != seal::scheme_type::bfv && !encrypted.ntt_)
                throw std::invalid_argument("encrypted must be in NTT form");
            const std::size_t B = encrypted.batch_, L = encrypted.L_, n = encrypted.n_;
            const bool ckks = scheme == seal::scheme_type::ckks;
            std::vector<std::uint64_t> cf(B, encrypted.cf_);
            status(destination.reserve(ctx_, B * (ckks ? L * n : n)));
            status(sb200_decrypt(ctx_, key_, L, encrypted.size_, B, encrypted.d_, scheme == seal::scheme_type::bgv ? cf.data() : nullptr,
                                 destination.d_, nullptr));
            destination.batch_ = B, destination.L_ = ckks ? L : 1, destination.n_ = n;
            destination.parms_id_ = ckks ? encrypted.parms_id_ : seal::parms_id_zero;
            destination.ntt_ = ckks, destination.scale_ = ckks ? encrypted.scale_ : 1.0;
        }

    private:
        // the reference's scheme and form checks of invariant_noise_budget, in its order (:424-436)
        void check_form(bool is_ntt_form) const
        {
            const auto scheme = context_.key_context_data()->parms().scheme();
            if (scheme != seal::scheme_type::bfv && scheme != seal::scheme_type::bgv)
                throw std::logic_error("unsupported scheme");
            if (scheme == seal::scheme_type::bfv && is_ntt_form)
                throw std::invalid_argument("BFV encrypted cannot be in NTT form");
            if (scheme == seal::scheme_type::bgv && !is_ntt_form)
                throw std::invalid_argument("BGV encrypted must be in NTT form");
        }
        // a batch of another context (or an empty one) is rejected as Evaluator rejects it
        void owned(const CiphertextBatch &b) const
        {
            if (b.ctx_ != ctx_ || !b.d_ || !b.batch_ || !context_.get_context_data(b.parms_id_))
                throw std::invalid_argument("encrypted is not valid for encryption parameters");
        }
        static void status(int rc) { status(rc, rc == SB200_OK ? std::string() : sb200_last_error()); }
        static void status(int rc, const std::string &msg)
        {
            if (rc == SB200_OK)
                return;
            if (rc == SB200_E_INVALID_ARG || rc == SB200_E_POINTER)
                throw std::invalid_argument(msg);
            if (rc == SB200_E_LOGIC)
                throw std::logic_error(msg);
            throw std::runtime_error(msg);
        }
        seal::SEALContext context_;
        sb200_context *ctx_ = nullptr;
        sb200_secret_key *key_ = nullptr;
    };
} // namespace seal_b200
