// include/seal_b200/ckks.hpp -- same-signature stand-in for seal::CKKSEncoder (native/src/seal/ckks.h: encode / decode of vectors
// of real or complex numbers into NTT-form plaintexts) over the C-ABI of include/seal_b200.h.
//
//     seal_b200::CKKSEncoder encoder(context, evaluator);   // shares the evaluator's device context
//     encoder.encode(values, scale, plain);  encoder.decode(plain, values);
//
// The embedding transform (double-precision complex FFT), the rounding and the residue decomposition run on the device
// (sb200_ckks_encode / sb200_ckks_decode) and reproduce the reference's plaintexts and decoded values bit for bit; the checks and
// exception types are the reference's (ckks.h:455-807).  The scalar overloads (ckks.h:272-377: one double, complex number or int64
// in every slot) have the reference's declarations and make the same plaintexts (sb200_ckks_encode_scalar_host).  The batch
// members are the extension the reference does not have, among them the scalar ones on PlaintextBatch (encode of one value,
// encode_scalars of one value per plaintext).
#pragma once

#include "../seal_b200.h"
#include "evaluator.hpp"
#include "seal/seal.h"
#include <complex>
#include <cstdint>
#include <stdexcept>
#include <type_traits>
#include <vector>

namespace seal_b200
{
    class CKKSEncoder
    {
    public:
        // shares the device context of an existing evaluator, which must outlive this object
        CKKSEncoder(const seal::SEALContext &context, const Evaluator &evaluator) : context_(context), ctx_(evaluator.native_handle())
        {
            if (!context_.parameters_set())
                throw std::invalid_argument("encryption parameters are not set correctly"); // ckks.cpp:16-19
            auto &parms = context_.first_context_data()->parms();
            if (parms.scheme() != seal::scheme_type::ckks)
                throw std::invalid_argument("unsupported scheme"); // ckks.cpp:22-25
            slots_ = parms.poly_modulus_degree() >> 1;
        }

        std::size_t slot_count() const noexcept { return slots_; }

        // ckks.h:172-178, 196-202
        template <typename T, typename = std::enable_if_t<std::is_same<std::remove_cv_t<T>, double>::value ||
                                                          std::is_same<std::remove_cv_t<T>, std::complex<double>>::value>>
        void encode(const std::vector<T> &values, seal::parms_id_type parms_id, double scale, seal::Plaintext &destination) const
        {
            encode_internal(values.data(), values.size(), parms_id, scale, destination);
        }
        template <typename T, typename = std::enable_if_t<std::is_same<std::remove_cv_t<T>, double>::value ||
                                                          std::is_same<std::remove_cv_t<T>, std::complex<double>>::value>>
        void encode(const std::vector<T> &values, double scale, seal::Plaintext &destination) const
        {
            encode_internal(values.data(), values.size(), context_.first_parms_id(), scale, destination);
        }
        // ---- one scalar in every slot (ckks.h:272-377): the reference's six declarations, so that calls written for seal::CKKSEncoder
        // select the same overload (encode(i + 1, plain) with a size_t takes the int64 one).  The pool is checked, as the reference
        // checks it, and not otherwise used: the plaintext is made on the device (sb200_ckks_encode_scalar_host)
        void encode(double value, seal::parms_id_type parms_id, double scale, seal::Plaintext &destination,
                    seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            auto cd = context_.get_context_data(parms_id);
            if (!cd)
                throw std::invalid_argument("parms_id is not valid for encryption parameters"); // ckks.cpp:79-88
            if (!pool)
                throw std::invalid_argument("pool is uninitialized");
            encode_scalar_internal(&value, SB200_CKKS_SCALAR_REAL, cd->parms().coeff_modulus().size(), parms_id, scale, destination);
        }
        void encode(double value, double scale, seal::Plaintext &destination, seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            encode(value, context_.first_parms_id(), scale, destination, std::move(pool));
        }
        void encode(std::complex<double> value, seal::parms_id_type parms_id, double scale, seal::Plaintext &destination,
                    seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            auto cd = context_.get_context_data(parms_id);
            if (!cd)
                throw std::invalid_argument("parms_id is not valid for encryption parameters"); // ckks.h:462-466
            if (!pool)
                throw std::invalid_argument("pool is uninitialized");
            encode_scalar_internal(&value, SB200_CKKS_SCALAR_COMPLEX, cd->parms().coeff_modulus().size(), parms_id, scale, destination);
        }
        void encode(std::complex<double> value, double scale, seal::Plaintext &destination,
                    seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            encode(value, context_.first_parms_id(), scale, destination, std::move(pool));
        }
        void encode(std::int64_t value, seal::parms_id_type parms_id, seal::Plaintext &destination) const
        {
            auto cd = context_.get_context_data(parms_id);
            if (!cd)
                throw std::invalid_argument("parms_id is not valid for encryption parameters"); // ckks.cpp:235-239
            encode_scalar_internal(&value, SB200_CKKS_SCALAR_INT64, cd->parms().coeff_modulus().size(), parms_id, 1.0, destination);
        }
        void encode(std::int64_t value, seal::Plaintext &destination) const { encode(value, context_.first_parms_id(), destination); }

        // ckks.h:365-372
        template <typename T, typename = std::enable_if_t<std::is_same<std::remove_cv_t<T>, double>::value ||
                                                          std::is_same<std::remove_cv_t<T>, std::complex<double>>::value>>
        void decode(const seal::Plaintext &plain, std::vector<T> &destination) const
        {
            if (!seal::is_valid_for(plain, context_))
                throw std::invalid_argument("plain is not valid for encryption parameters"); // ckks.h:700-703
            if (!plain.is_ntt_form())
                throw std::invalid_argument("plain is not in NTT form");
            const std::size_t L = context_.get_context_data(plain.parms_id())->parms().coeff_modulus().size();
            std::vector<std::complex<double>> out(slots_);
            status(sb200_ckks_decode_host(ctx_, L, 1, plain.data(), plain.scale(), reinterpret_cast<double *>(out.data())));
            destination.resize(slots_);
            for (std::size_t i = 0; i < slots_; i++)
                destination[i] = from_complex<T>(out[i]);
        }

        // ---- batches: B vectors -> B plaintexts in one call (one transform launch sequence for all of them) ----
        template <typename T>
        void encode(const std::vector<std::vector<T>> &values, seal::parms_id_type parms_id, double scale, std::vector<seal::Plaintext> &destination) const
        {
            auto cd = context_.get_context_data(parms_id);
            if (!cd)
                throw std::invalid_argument("parms_id is not valid for encryption parameters");
            const std::size_t B = values.size(), L = cd->parms().coeff_modulus().size(), n = slots_ * 2;
            std::size_t count = 0;
            for (auto &v : values)
                count = std::max(count, v.size());
            if (count > slots_)
                throw std::invalid_argument("values_size is too large");
            std::vector<T> flat(B * count, T(0));
            for (std::size_t b = 0; b < B; b++)
                std::copy(values[b].begin(), values[b].end(), flat.begin() + b * count);
            std::vector<std::uint64_t> words(B * L * n);
            if (B)
                status(sb200_ckks_encode_host(ctx_, L, B, reinterpret_cast<const double *>(flat.data()), count,
                                              std::is_same<T, std::complex<double>>::value ? 1 : 0, scale, words.data()));
            destination.resize(B);
            for (std::size_t b = 0; b < B; b++)
            {
                destination[b].parms_id() = seal::parms_id_zero;
                destination[b].resize(L * n);
                std::copy_n(words.data() + b * L * n, L * n, destination[b].data());
                destination[b].parms_id() = parms_id;
                destination[b].scale() = scale;
            }
        }

        // ---- device-resident plaintexts: B vectors -> a PlaintextBatch [B][L][n] in NTT form at parms_id, encoded on the device
        // (sb200_ckks_encode).  Build the encoder with the Evaluator (CKKSEncoder(context, evaluator)) for that Evaluator to accept it.
        template <typename T>
        void encode(const std::vector<std::vector<T>> &values, seal::parms_id_type parms_id, double scale, PlaintextBatch &destination) const
        {
            auto cd = context_.get_context_data(parms_id);
            if (!cd)
                throw std::invalid_argument("parms_id is not valid for encryption parameters");
            if (values.empty())
                throw std::invalid_argument("batch cannot be empty");
            const std::size_t B = values.size(), L = cd->parms().coeff_modulus().size(), n = slots_ * 2;
            std::size_t count = 0;
            for (auto &v : values)
                count = std::max(count, v.size());
            if (count > slots_)
                throw std::invalid_argument("values_size is too large");
            std::vector<T> flat(B * count, T(0));
            for (std::size_t b = 0; b < B; b++)
                std::copy(values[b].begin(), values[b].end(), flat.begin() + b * count);
            std::uint64_t *d_values = nullptr;
            int rc = SB200_OK;
            if (count)
            {
                status(sb200_device_malloc(ctx_, flat.size() * sizeof(T), &d_values));
                rc = sb200_memcpy_h2d(ctx_, d_values, flat.data(), flat.size() * sizeof(T), nullptr);
            }
            if (rc == SB200_OK)
                rc = destination.reserve(ctx_, B * L * n);
            if (rc == SB200_OK)
                rc = sb200_ckks_encode(ctx_, L, B, reinterpret_cast<const double *>(d_values), count,
                                       std::is_same<T, std::complex<double>>::value ? 1 : 0, scale, destination.d_, nullptr);
            if (d_values)
                sb200_device_free(ctx_, d_values);
            status(rc);
            destination.batch_ = B, destination.L_ = L, destination.n_ = n;
            destination.parms_id_ = parms_id, destination.ntt_ = true, destination.scale_ = scale;
        }

        // ---- device-resident scalar plaintexts (sb200_ckks_encode_scalar): encode(value, ..., PlaintextBatch &) makes a batch of one
        // plaintext, which every PlaintextBatch consumer applies to a whole CiphertextBatch; encode_scalars makes one plaintext per
        // value (a distinct name: encode(std::vector<double>, ...) means one slot vector).  Checks and messages as the Plaintext overloads.
        void encode(double value, seal::parms_id_type parms_id, double scale, PlaintextBatch &destination) const
        {
            encode_scalars_internal(&value, 1, SB200_CKKS_SCALAR_REAL, parms_id, scale, destination);
        }
        void encode(std::complex<double> value, seal::parms_id_type parms_id, double scale, PlaintextBatch &destination) const
        {
            encode_scalars_internal(&value, 1, SB200_CKKS_SCALAR_COMPLEX, parms_id, scale, destination);
        }
        void encode(std::int64_t value, seal::parms_id_type parms_id, PlaintextBatch &destination) const
        {
            encode_scalars_internal(&value, 1, SB200_CKKS_SCALAR_INT64, parms_id, 1.0, destination);
        }
        void encode_scalars(const std::vector<double> &values, seal::parms_id_type parms_id, double scale, PlaintextBatch &destination) const
        {
            encode_scalars_internal(values.data(), values.size(), SB200_CKKS_SCALAR_REAL, parms_id, scale, destination);
        }
        void encode_scalars(const std::vector<std::complex<double>> &values, seal::parms_id_type parms_id, double scale,
                            PlaintextBatch &destination) const
        {
            encode_scalars_internal(values.data(), values.size(), SB200_CKKS_SCALAR_COMPLEX, parms_id, scale, destination);
        }
        void encode_scalars(const std::vector<std::int64_t> &values, seal::parms_id_type parms_id, PlaintextBatch &destination) const
        {
            encode_scalars_internal(values.data(), values.size(), SB200_CKKS_SCALAR_INT64, parms_id, 1.0, destination);
        }

        // ---- device-resident plaintexts: a PlaintextBatch in NTT form -> B vectors of slot_count() values, decoded on the device
        // (sb200_ckks_decode) with the batch's scale; only the values cross PCIe.  The batch must come from this encoder's context.
        template <typename T, typename = std::enable_if_t<std::is_same<std::remove_cv_t<T>, double>::value ||
                                                          std::is_same<std::remove_cv_t<T>, std::complex<double>>::value>>
        void decode(const PlaintextBatch &plain, std::vector<std::vector<T>> &destination) const
        {
            if (plain.ctx_ != ctx_ || !plain.d_ || !plain.batch_ || (plain.ntt_ && !context_.get_context_data(plain.parms_id_)))
                throw std::invalid_argument("plain is not valid for encryption parameters");
            if (!plain.ntt_)
                throw std::invalid_argument("plain is not in NTT form");
            const std::size_t B = plain.batch_;
            std::vector<std::complex<double>> out(B * slots_);
            std::uint64_t *d_values = nullptr;
            status(sb200_device_malloc(ctx_, out.size() * sizeof(std::complex<double>), &d_values));
            int rc = sb200_ckks_decode(ctx_, plain.L_, B, plain.d_, plain.scale_, reinterpret_cast<double *>(d_values), nullptr);
            if (rc == SB200_OK)
                rc = sb200_memcpy_d2h(ctx_, out.data(), d_values, out.size() * sizeof(std::complex<double>), nullptr);
            if (rc == SB200_OK)
                rc = sb200_stream_synchronize(ctx_, nullptr);
            sb200_device_free(ctx_, d_values); // on success it leaves the last error alone
            status(rc);
            destination.resize(B);
            for (std::size_t b = 0; b < B; b++)
            {
                destination[b].resize(slots_);
                for (std::size_t i = 0; i < slots_; i++)
                    destination[b][i] = from_complex<T>(out[b * slots_ + i]);
            }
        }

    private:
        // one scalar (kind SB200_CKKS_SCALAR_*) -> destination, which changes only on success
        void encode_scalar_internal(const void *value, int kind, std::size_t L, seal::parms_id_type parms_id, double scale,
                                    seal::Plaintext &destination) const
        {
            const std::size_t n = slots_ * 2;
            std::vector<std::uint64_t> words(L * n);
            status(sb200_ckks_encode_scalar_host(ctx_, L, 1, kind, value, scale, words.data()));
            destination.parms_id() = seal::parms_id_zero; // ckks.cpp:129-132
            destination.resize(L * n);
            std::copy(words.begin(), words.end(), destination.data());
            destination.parms_id() = parms_id;
            destination.scale() = scale;
        }
        // B scalars (host) -> a PlaintextBatch [B][L][n] made on the device
        void encode_scalars_internal(const void *values, std::size_t B, int kind, seal::parms_id_type parms_id, double scale,
                                     PlaintextBatch &destination) const
        {
            auto cd = context_.get_context_data(parms_id);
            if (!cd)
                throw std::invalid_argument("parms_id is not valid for encryption parameters");
            if (!B)
                throw std::invalid_argument("batch cannot be empty");
            const std::size_t L = cd->parms().coeff_modulus().size(), n = slots_ * 2;
            const std::size_t bytes = B * (kind == SB200_CKKS_SCALAR_COMPLEX ? 16 : 8);
            std::uint64_t *d_values = nullptr;
            status(sb200_device_malloc(ctx_, bytes, &d_values));
            int rc = sb200_memcpy_h2d(ctx_, d_values, values, bytes, nullptr);
            if (rc == SB200_OK)
                rc = destination.reserve(ctx_, B * L * n);
            if (rc == SB200_OK)
                rc = sb200_ckks_encode_scalar(ctx_, L, B, kind, d_values, scale, destination.d_, nullptr);
            sb200_device_free(ctx_, d_values);
            status(rc);
            destination.batch_ = B, destination.L_ = L, destination.n_ = n;
            destination.parms_id_ = parms_id, destination.ntt_ = true, destination.scale_ = scale;
        }
        template <typename T>
        void encode_internal(const T *values, std::size_t values_size, seal::parms_id_type parms_id, double scale, seal::Plaintext &destination) const
        {
            auto cd = context_.get_context_data(parms_id);
            if (!cd)
                throw std::invalid_argument("parms_id is not valid for encryption parameters"); // ckks.h:462-466
            if (!values && values_size > 0)
                throw std::invalid_argument("values cannot be null");
            if (values_size > slots_)
                throw std::invalid_argument("values_size is too large");
            const std::size_t L = cd->parms().coeff_modulus().size(), n = slots_ * 2;
            std::vector<std::uint64_t> words(L * n);
            // scale bounds, finiteness and magnitude are checked by the library with the reference's messages
            status(sb200_ckks_encode_host(ctx_, L, 1, reinterpret_cast<const double *>(values), values_size,
                                          std::is_same<std::remove_cv_t<T>, std::complex<double>>::value ? 1 : 0, scale, words.data()));
            destination.parms_id() = seal::parms_id_zero; // ckks.h:561-562
            destination.resize(L * n);
            std::copy(words.begin(), words.end(), destination.data());
            destination.parms_id() = parms_id;
            destination.scale() = scale;
        }
        template <typename T>
        static T from_complex(std::complex<double> in) // ckks.h (from_complex): the real part for T = double
        {
            if constexpr (std::is_same<T, double>::value)
                return in.real();
            else
                return in;
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
        std::size_t slots_ = 0;
    };
} // namespace seal_b200
