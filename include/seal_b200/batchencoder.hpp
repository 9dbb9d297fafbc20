// include/seal_b200/batchencoder.hpp -- same-signature stand-in for seal::BatchEncoder (native/src/seal/batchencoder.h:
// encode / decode of the 2 x n/2 slot matrix for BFV / BGV) over the C-ABI of include/seal_b200.h.
//
//     seal_b200::BatchEncoder encoder(context);          // or BatchEncoder(evaluator): shares the evaluator's device context
//     encoder.encode(values, plain);  encoder.decode(plain, values);
//
// The slot permutation and the transform modulo the plain modulus run on the device (sb200_batch_encode / _decode); the
// checks and exception types are the reference's (batchencoder.cpp:13-38, 84-330).
#pragma once

#include "../seal_b200.h"
#include "evaluator.hpp"
#include "seal/seal.h"
#include <algorithm>
#include <cstdint>
#include <stdexcept>
#include <vector>

namespace seal_b200
{
    class BatchEncoder
    {
    public:
        explicit BatchEncoder(const seal::SEALContext &context, int device = 0) : context_(context)
        {
            check_context();
            auto &parms = context_.key_context_data()->parms();
            std::vector<std::uint64_t> q;
            for (auto &m : parms.coeff_modulus())
                q.push_back(m.value());
            status(sb200_context_create(static_cast<int>(parms.scheme()), parms.poly_modulus_degree(), q.data(), q.size(),
                                        parms.plain_modulus().value(), device, &ctx_));
            owned_ = true;
        }
        // shares the device context (tables for the plain modulus included) of an existing evaluator, which must outlive this object
        explicit BatchEncoder(const seal::SEALContext &context, const Evaluator &evaluator) : context_(context), ctx_(evaluator.native_handle())
        {
            check_context();
        }
        ~BatchEncoder()
        {
            if (owned_ && ctx_)
                sb200_context_destroy(ctx_);
        }
        BatchEncoder(const BatchEncoder &) = delete;
        BatchEncoder &operator=(const BatchEncoder &) = delete;

        std::size_t slot_count() const noexcept { return slots_; }

        // batchencoder.cpp:84-128
        void encode(const std::vector<std::uint64_t> &values_matrix, seal::Plaintext &destination) const
        {
            if (values_matrix.size() > slots_)
                throw std::invalid_argument("values_matrix size is too large");
            for (auto v : values_matrix)
                if (v >= modulus_)
                    throw std::invalid_argument("input value is larger than plain_modulus");
            std::vector<std::uint64_t> slots(slots_, 0);
            std::copy(values_matrix.begin(), values_matrix.end(), slots.begin());
            run_encode(slots, destination);
        }
        // batchencoder.cpp:130-165
        void encode(const std::vector<std::int64_t> &values_matrix, seal::Plaintext &destination) const
        {
            if (values_matrix.size() > slots_)
                throw std::invalid_argument("values_matrix size is too large");
            std::vector<std::uint64_t> slots(slots_, 0);
            for (std::size_t i = 0; i < values_matrix.size(); i++)
            {
                const std::int64_t v = values_matrix[i];
                const std::uint64_t magnitude = v < 0 ? 0 - static_cast<std::uint64_t>(v) : static_cast<std::uint64_t>(v);
                if (magnitude > (modulus_ >> 1))
                    throw std::invalid_argument("input value is larger than plain_modulus");
                slots[i] = v < 0 ? modulus_ + static_cast<std::uint64_t>(v) : static_cast<std::uint64_t>(v);
            }
            run_encode(slots, destination);
        }
        // ---- device-resident plaintexts: B matrices -> a PlaintextBatch [B][n] in coefficient form, encoded on the device
        // (sb200_batch_encode).  Each matrix is checked as the single-plaintext overloads above check it.  Build the encoder with the
        // Evaluator (BatchEncoder(context, evaluator)) for that Evaluator to accept the batch.
        void encode(const std::vector<std::vector<std::uint64_t>> &values_matrices, PlaintextBatch &destination) const
        {
            std::vector<std::uint64_t> slots(values_matrices.size() * slots_, 0);
            for (std::size_t b = 0; b < values_matrices.size(); b++)
            {
                auto &m = values_matrices[b];
                if (m.size() > slots_)
                    throw std::invalid_argument("values_matrix size is too large");
                for (auto v : m)
                    if (v >= modulus_)
                        throw std::invalid_argument("input value is larger than plain_modulus");
                std::copy(m.begin(), m.end(), slots.begin() + b * slots_);
            }
            run_encode(slots, values_matrices.size(), destination);
        }
        void encode(const std::vector<std::vector<std::int64_t>> &values_matrices, PlaintextBatch &destination) const
        {
            std::vector<std::uint64_t> slots(values_matrices.size() * slots_, 0);
            for (std::size_t b = 0; b < values_matrices.size(); b++)
            {
                auto &m = values_matrices[b];
                if (m.size() > slots_)
                    throw std::invalid_argument("values_matrix size is too large");
                for (std::size_t i = 0; i < m.size(); i++)
                {
                    const std::int64_t v = m[i];
                    const std::uint64_t magnitude = v < 0 ? 0 - static_cast<std::uint64_t>(v) : static_cast<std::uint64_t>(v);
                    if (magnitude > (modulus_ >> 1))
                        throw std::invalid_argument("input value is larger than plain_modulus");
                    slots[b * slots_ + i] = v < 0 ? modulus_ + static_cast<std::uint64_t>(v) : static_cast<std::uint64_t>(v);
                }
            }
            run_encode(slots, values_matrices.size(), destination);
        }
        // batchencoder.cpp:229-266
        void decode(const seal::Plaintext &plain, std::vector<std::uint64_t> &destination,
                    seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination = run_decode(plain, pool);
        }
        // batchencoder.cpp:268-305
        void decode(const seal::Plaintext &plain, std::vector<std::int64_t> &destination,
                    seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            const std::vector<std::uint64_t> raw = run_decode(plain, pool);
            destination.resize(slots_);
            for (std::size_t i = 0; i < slots_; i++)
                destination[i] = raw[i] > (modulus_ >> 1) ? static_cast<std::int64_t>(raw[i]) - static_cast<std::int64_t>(modulus_)
                                                          : static_cast<std::int64_t>(raw[i]);
        }

        // ---- device-resident plaintexts: a PlaintextBatch in coefficient form -> B matrices, decoded on the device
        // (sb200_batch_decode); only the slots cross PCIe.  The batch must come from this encoder's device context.
        void decode(const PlaintextBatch &plain, std::vector<std::vector<std::uint64_t>> &destination) const
        {
            const std::vector<std::uint64_t> raw = run_decode(plain);
            destination.resize(plain.batch_);
            for (std::size_t b = 0; b < plain.batch_; b++)
                destination[b].assign(raw.begin() + b * slots_, raw.begin() + (b + 1) * slots_);
        }
        void decode(const PlaintextBatch &plain, std::vector<std::vector<std::int64_t>> &destination) const
        {
            const std::vector<std::uint64_t> raw = run_decode(plain);
            destination.resize(plain.batch_);
            for (std::size_t b = 0; b < plain.batch_; b++)
            {
                destination[b].resize(slots_);
                for (std::size_t i = 0; i < slots_; i++)
                {
                    const std::uint64_t v = raw[b * slots_ + i];
                    destination[b][i] = v > (modulus_ >> 1) ? static_cast<std::int64_t>(v) - static_cast<std::int64_t>(modulus_)
                                                            : static_cast<std::int64_t>(v);
                }
            }
        }

    private:
        std::vector<std::uint64_t> run_decode(const PlaintextBatch &plain) const
        {
            if (plain.ctx_ != ctx_ || !plain.d_ || !plain.batch_ || plain.n_ != slots_)
                throw std::invalid_argument("plain is not valid for encryption parameters");
            if (plain.ntt_)
                throw std::invalid_argument("plain cannot be in NTT form");
            std::vector<std::uint64_t> out(plain.batch_ * slots_);
            std::uint64_t *d_values = nullptr;
            status(sb200_device_malloc(ctx_, out.size() * sizeof(std::uint64_t), &d_values));
            int rc = sb200_batch_decode(ctx_, plain.batch_, plain.d_, d_values, nullptr);
            if (rc == SB200_OK)
                rc = sb200_memcpy_d2h(ctx_, out.data(), d_values, out.size() * sizeof(std::uint64_t), nullptr);
            if (rc == SB200_OK)
                rc = sb200_stream_synchronize(ctx_, nullptr);
            sb200_device_free(ctx_, d_values); // on success it leaves the last error alone
            status(rc);
            return out;
        }
        void check_context()
        {
            if (!context_.parameters_set())
                throw std::invalid_argument("encryption parameters are not set correctly"); // batchencoder.cpp:16-20
            auto &cd = *context_.first_context_data();
            if (cd.parms().scheme() != seal::scheme_type::bfv && cd.parms().scheme() != seal::scheme_type::bgv)
                throw std::invalid_argument("unsupported scheme");
            if (!cd.qualifiers().using_batching)
                throw std::invalid_argument("encryption parameters are not valid for batching");
            slots_ = cd.parms().poly_modulus_degree();
            modulus_ = cd.parms().plain_modulus().value();
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
        void run_encode(const std::vector<std::uint64_t> &slots, seal::Plaintext &destination) const
        {
            destination.resize(slots_);
            destination.parms_id() = seal::parms_id_zero;
            status(sb200_batch_encode_host(ctx_, 1, slots.data(), destination.data()));
        }
        void run_encode(const std::vector<std::uint64_t> &slots, std::size_t B, PlaintextBatch &destination) const
        {
            if (!B)
                throw std::invalid_argument("batch cannot be empty");
            std::uint64_t *d_values = nullptr;
            status(sb200_device_malloc(ctx_, slots.size() * sizeof(std::uint64_t), &d_values));
            int rc = sb200_memcpy_h2d(ctx_, d_values, slots.data(), slots.size() * sizeof(std::uint64_t), nullptr);
            if (rc == SB200_OK)
                rc = destination.reserve(ctx_, slots.size());
            if (rc == SB200_OK)
                rc = sb200_batch_encode(ctx_, B, d_values, destination.d_, nullptr);
            sb200_device_free(ctx_, d_values);
            status(rc);
            destination.batch_ = B, destination.L_ = 1, destination.n_ = slots_;
            destination.parms_id_ = seal::parms_id_zero, destination.ntt_ = false, destination.scale_ = 1.0;
        }
        std::vector<std::uint64_t> run_decode(const seal::Plaintext &plain, const seal::MemoryPoolHandle &pool) const
        {
            if (!seal::is_valid_for(plain, context_))
                throw std::invalid_argument("plain is not valid for encryption parameters");
            if (plain.is_ntt_form())
                throw std::invalid_argument("plain cannot be in NTT form");
            if (!pool)
                throw std::invalid_argument("pool is uninitialized");
            std::vector<std::uint64_t> coeffs(slots_, 0), out(slots_);
            std::copy(plain.data(), plain.data() + std::min(plain.coeff_count(), slots_), coeffs.begin());
            status(sb200_batch_decode_host(ctx_, 1, coeffs.data(), out.data()));
            return out;
        }

        seal::SEALContext context_;
        sb200_context *ctx_ = nullptr;
        bool owned_ = false;
        std::size_t slots_ = 0;
        std::uint64_t modulus_ = 0;
    };
} // namespace seal_b200
