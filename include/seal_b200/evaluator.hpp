// include/seal_b200/evaluator.hpp -- header-only C++17 drop-in for the hot-path members of seal::Evaluator.
//
// seal::Evaluator has no virtual members and cannot be subclassed (evaluator.h:79, copy/move deleted :1320-1326), so the
// drop-in is a class with the SAME member signatures (same seal::Ciphertext / RelinKeys / GaloisKeys / SEALContext
// types, same argument meaning, same exception types from the same prologue checks) that a SEAL user instantiates
// instead of seal::Evaluator for multiply / relinearize / rescale_to_next / mod_switch_to_next / apply_galois /
// rotate_rows / rotate_columns / rotate_vector / complex_conjugate / transform_{to,from}_ntt.  It is compiled against the
// user's own SEAL headers; all arithmetic happens in libseal_b200.so (include/seal_b200.h) on the GPU -- there is
// no CPU fallback.  Batch overloads (std::vector<Ciphertext>) are the extension the reference does not have.
//
// Reference members mirrored (native/src/seal/): evaluator.h:219-345, 510-545, 929-1316; evaluator.cpp:352-393, 569-708,
// 1144-1199, 1201-1294, 1404-1541, 2289-2559.
#pragma once
#include "../seal_b200.h"
#include "seal/seal.h"
#include "seal/util/numth.h"
#include "seal/util/uintarithsmallmod.h"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <deque>
#include <limits>
#include <map>
#include <mutex>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

namespace seal_b200
{
    class Evaluator;
    class Decryptor;
    class BatchEncoder;
    class CKKSEncoder;

    // ---- device-resident ciphertexts ---------------------------------------------------------------------------------
    // A batch of B ciphertexts of one shape that stays on the GPU between Evaluator calls.  It carries exactly the metadata
    // seal::Ciphertext carries (ciphertext.h:728-742: parms_id, is_ntt_form, size, poly_modulus_degree, coeff_modulus_size,
    // scale, correction_factor), shared by all members of the batch; Evaluator updates it the way the reference updates the
    // members of each Ciphertext.  Storage is one slab [B][size][L][n] laid out like Ciphertext::data(), allocated from the
    // Evaluator's context (sb200_device_malloc) -- the reference's counterpart is the MemoryPoolHandle behind a Ciphertext.
    // Usage: ev.upload(cts, batch); ev.multiply_relinearize_inplace(batch, other, rk); ev.rescale_to_next_inplace(batch); ...
    //        ev.download(batch, cts);      -- one H2D and one D2H for a whole chain of operations.
    class CiphertextBatch
    {
    public:
        CiphertextBatch() = default;
        ~CiphertextBatch() { release(); }
        CiphertextBatch(const CiphertextBatch &) = delete;
        CiphertextBatch &operator=(const CiphertextBatch &) = delete;
        CiphertextBatch(CiphertextBatch &&o) noexcept { *this = std::move(o); }
        CiphertextBatch &operator=(CiphertextBatch &&o) noexcept
        {
            if (this != &o)
            {
                release();
                ctx_ = o.ctx_, d_ = o.d_, cap_ = o.cap_, batch_ = o.batch_, size_ = o.size_, L_ = o.L_, n_ = o.n_;
                parms_id_ = o.parms_id_, ntt_ = o.ntt_, scale_ = o.scale_, cf_ = o.cf_;
                o.ctx_ = nullptr, o.d_ = nullptr, o.cap_ = o.batch_ = o.size_ = o.L_ = o.n_ = 0;
            }
            return *this;
        }
        std::size_t batch_size() const noexcept { return batch_; }
        std::size_t size() const noexcept { return size_; }                             // polynomials per ciphertext
        std::size_t coeff_modulus_size() const noexcept { return L_; }
        std::size_t poly_modulus_degree() const noexcept { return n_; }
        const seal::parms_id_type &parms_id() const noexcept { return parms_id_; }
        bool is_ntt_form() const noexcept { return ntt_; }
        double &scale() noexcept { return scale_; }
        double scale() const noexcept { return scale_; }
        std::uint64_t correction_factor() const noexcept { return cf_; }
        std::uint64_t *device_data() noexcept { return d_; }
        const std::uint64_t *device_data() const noexcept { return d_; }
        std::size_t words_per_ciphertext() const noexcept { return size_ * L_ * n_; }
        void release() noexcept
        {
            if (d_ && ctx_)
                sb200_device_free(ctx_, d_);
            d_ = nullptr, cap_ = 0;
        }

    private:
        friend class Evaluator;
        friend class Decryptor;
        friend class Encryptor;
        sb200_context *ctx_ = nullptr;
        std::uint64_t *d_ = nullptr;
        std::size_t cap_ = 0; // words
        std::size_t batch_ = 0, size_ = 0, L_ = 0, n_ = 0;
        seal::parms_id_type parms_id_ = seal::parms_id_zero;
        bool ntt_ = false;
        double scale_ = 1.0;
        std::uint64_t cf_ = 1;
    };

    // ---- device-resident plaintexts ----------------------------------------------------------------------------------
    // B plaintexts of one shape on the GPU, with seal::Plaintext's metadata (plaintext.h: parms_id, zero in coefficient form;
    // is_ntt_form; scale), shared by all members.  The slab is [B][L][n] in NTT form (Plaintext::data() at that parms_id) or [B][n]
    // in coefficient form (words below t, zero-padded above coeff_count).  B may be 1: one plaintext applied to every ciphertext
    // of a CiphertextBatch (the plaintext operations accept B = 1 or B = the ciphertext batch size).  Same ownership rules as
    // CiphertextBatch: allocated from the Evaluator's context (or an encoder sharing it), movable, not copyable.
    class PlaintextBatch
    {
    public:
        PlaintextBatch() = default;
        ~PlaintextBatch() { release(); }
        PlaintextBatch(const PlaintextBatch &) = delete;
        PlaintextBatch &operator=(const PlaintextBatch &) = delete;
        PlaintextBatch(PlaintextBatch &&o) noexcept { *this = std::move(o); }
        PlaintextBatch &operator=(PlaintextBatch &&o) noexcept
        {
            if (this != &o)
            {
                release();
                ctx_ = o.ctx_, d_ = o.d_, cap_ = o.cap_, batch_ = o.batch_, L_ = o.L_, n_ = o.n_;
                parms_id_ = o.parms_id_, ntt_ = o.ntt_, scale_ = o.scale_;
                o.ctx_ = nullptr, o.d_ = nullptr, o.cap_ = o.batch_ = o.L_ = o.n_ = 0;
            }
            return *this;
        }
        std::size_t batch_size() const noexcept { return batch_; }
        std::size_t coeff_modulus_size() const noexcept { return ntt_ ? L_ : 0; } // primes of an NTT-form plaintext
        std::size_t poly_modulus_degree() const noexcept { return n_; }
        const seal::parms_id_type &parms_id() const noexcept { return parms_id_; }
        bool is_ntt_form() const noexcept { return ntt_; }
        double scale() const noexcept { return scale_; }
        std::uint64_t *device_data() noexcept { return d_; }
        const std::uint64_t *device_data() const noexcept { return d_; }
        std::size_t words_per_plaintext() const noexcept { return ntt_ ? L_ * n_ : n_; }
        void release() noexcept
        {
            if (d_ && ctx_)
                sb200_device_free(ctx_, d_);
            d_ = nullptr, cap_ = 0;
        }

    private:
        friend class Evaluator;
        friend class BatchEncoder;
        friend class CKKSEncoder;
        friend class Encryptor;
        friend class Decryptor;
        // room for `words` words from the context ctx (a status code of include/seal_b200.h)
        int reserve(sb200_context *ctx, std::size_t words)
        {
            if (ctx_ != ctx)
            {
                release();
                ctx_ = ctx;
            }
            if (cap_ >= words)
                return SB200_OK;
            release();
            const int rc = sb200_device_malloc(ctx_, words * sizeof(std::uint64_t), &d_);
            cap_ = rc == SB200_OK ? words : 0;
            return rc;
        }
        sb200_context *ctx_ = nullptr;
        std::uint64_t *d_ = nullptr;
        std::size_t cap_ = 0; // words
        std::size_t batch_ = 0, L_ = 0, n_ = 0;
        seal::parms_id_type parms_id_ = seal::parms_id_zero;
        bool ntt_ = false;
        double scale_ = 1.0;
    };

    // ---- device-resident key sets ------------------------------------------------------------------------------------
    // RelinKeys / GaloisKeys whose key-switching keys live on the GPU, one key handle (sb200_kswitch_key) per non-empty slot of
    // KSwitchKeys::data(), owned by this object.  Filled by Evaluator::load (straight from a stream: none, zlib or seeded) or
    // Evaluator::upload (from a seal:: object), or by KeyGenerator on the device; the batch members of Evaluator take them wherever
    // they take seal::RelinKeys / seal::GaloisKeys.  Same ownership rules as CiphertextBatch: allocated from the Evaluator's context,
    // movable, not copyable, and they must not outlive that context.  They are never entered in the Evaluator's key cache and never
    // evicted.  device_bytes() is what the set holds on the device: at n >= 4096 a key holds its 64-bit words and the integer
    // key-switching path's copy, 3.5x the words (n = 65536, k = 32: 1.04 GB + 2.6 GB per key).
    class DeviceKSwitchKeys
    {
    public:
        DeviceKSwitchKeys() = default;
        ~DeviceKSwitchKeys() { release(); }
        DeviceKSwitchKeys(const DeviceKSwitchKeys &) = delete;
        DeviceKSwitchKeys &operator=(const DeviceKSwitchKeys &) = delete;
        DeviceKSwitchKeys(DeviceKSwitchKeys &&o) noexcept { *this = std::move(o); }
        DeviceKSwitchKeys &operator=(DeviceKSwitchKeys &&o) noexcept
        {
            if (this != &o)
            {
                release();
                ctx_ = o.ctx_, keys_ = std::move(o.keys_), parms_id_ = o.parms_id_;
                o.ctx_ = nullptr, o.keys_.clear(), o.parms_id_ = seal::parms_id_zero;
            }
            return *this;
        }
        // the key level (KSwitchKeys::parms_id)
        const seal::parms_id_type &parms_id() const noexcept { return parms_id_; }
        // non-empty slots (KSwitchKeys::size)
        std::size_t size() const noexcept
        {
            return static_cast<std::size_t>(std::count_if(keys_.begin(), keys_.end(), [](const sb200_kswitch_key *k) { return k != nullptr; }));
        }
        std::size_t device_bytes() const noexcept
        {
            std::size_t bytes = 0;
            for (const sb200_kswitch_key *k : keys_)
                bytes += sb200_kswitch_key_device_bytes(k);
            return bytes;
        }
        void release() noexcept
        {
            for (sb200_kswitch_key *k : keys_)
                if (k)
                    sb200_kswitch_key_destroy(k);
            keys_.clear();
            ctx_ = nullptr, parms_id_ = seal::parms_id_zero;
        }

    protected:
        bool has_slot(std::size_t index) const noexcept { return index < keys_.size() && keys_[index]; }

    private:
        friend class Evaluator;
        friend class KeyGenerator;
        // replaces the contents with `keys` (indexed by slot, nullptr = empty), which this object then owns
        void assign(sb200_context *ctx, const seal::parms_id_type &parms_id, std::vector<sb200_kswitch_key *> &&keys) noexcept
        {
            release();
            ctx_ = ctx, parms_id_ = parms_id, keys_ = std::move(keys);
        }
        sb200_context *ctx_ = nullptr;
        std::vector<sb200_kswitch_key *> keys_;
        seal::parms_id_type parms_id_ = seal::parms_id_zero;
    };
    // RelinKeys on the device: slot RelinKeys::get_index(key_power)
    class DeviceRelinKeys : public DeviceKSwitchKeys
    {
    public:
        bool has_key(std::size_t key_power) const { return has_slot(seal::RelinKeys::get_index(key_power)); }
    };
    // GaloisKeys on the device: slot GaloisKeys::get_index(galois_elt); has_key throws like GaloisKeys::has_key for an even element
    class DeviceGaloisKeys : public DeviceKSwitchKeys
    {
    public:
        bool has_key(std::uint32_t galois_elt) const { return has_slot(seal::GaloisKeys::get_index(galois_elt)); }
    };

    class Evaluator
    {
    public:
        explicit Evaluator(const seal::SEALContext &context, int device = 0) : context_(context)
        {
            if (!context_.parameters_set())
                throw std::invalid_argument("encryption parameters are not set correctly"); // evaluator.cpp:121-128
            auto &parms = context_.key_context_data()->parms();
            std::vector<std::uint64_t> q;
            for (auto &m : parms.coeff_modulus())
                q.push_back(m.value());
            scheme_ = parms.scheme();
            if (scheme_ != seal::scheme_type::bfv && scheme_ != seal::scheme_type::ckks && scheme_ != seal::scheme_type::bgv)
                throw std::invalid_argument("unsupported scheme");
            check(sb200_context_create(
                static_cast<int>(scheme_), parms.poly_modulus_degree(), q.data(), q.size(),
                scheme_ != seal::scheme_type::ckks ? parms.plain_modulus().value() : 0, device, &ctx_));
        }
        ~Evaluator()
        {
            for (auto &kv : keys_)
                sb200_kswitch_key_destroy(kv.second.handle);
            tmp_.release(); // before the context it was allocated from goes away
            if (ctx_)
                sb200_context_destroy(ctx_);
        }
        Evaluator(const Evaluator &) = delete;
        Evaluator &operator=(const Evaluator &) = delete;

        // ---- multiply (evaluator.cpp:352-393) ------------------------------------------------------------------
        void multiply_inplace(seal::Ciphertext &encrypted1, const seal::Ciphertext &encrypted2,
                              seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            validate(encrypted1, "encrypted1 is not valid for encryption parameters");
            validate(encrypted2, "encrypted2 is not valid for encryption parameters");
            const Meta r = multiply_meta(meta(encrypted1), meta(encrypted2), &pool);
            const std::size_t L = encrypted1.coeff_modulus_size(), n = encrypted1.poly_modulus_degree();
            const std::size_t s1 = encrypted1.size(), s2 = encrypted2.size(); // any sizes: :524-560, :664-700, :796-833
            std::vector<std::uint64_t> a(encrypted1.data(), encrypted1.data() + s1 * L * n);
            encrypted1.resize(context_, r.parms_id, r.size);
            check(sb200_multiply_sized_host(ctx_, L, s1, s2, 1, a.data(), encrypted2.data(), encrypted1.data()));
            encrypted1.scale() = r.scale;
            encrypted1.correction_factor() = r.cf;
            throw_if_transparent(encrypted1);
        }
        void multiply(const seal::Ciphertext &encrypted1, const seal::Ciphertext &encrypted2, seal::Ciphertext &destination,
                      seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            if (&encrypted2 == &destination)
            {
                multiply_inplace(destination, encrypted1, std::move(pool));
            }
            else
            {
                destination = encrypted1;
                multiply_inplace(destination, encrypted2, std::move(pool));
            }
        }

        // ---- square (evaluator.cpp:843-1142): same residues as multiply(x, x) -------------------------------------------
        void square_inplace(seal::Ciphertext &encrypted, seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            seal::Ciphertext copy = encrypted;
            multiply_inplace(encrypted, copy, std::move(pool));
        }
        void square(const seal::Ciphertext &encrypted, seal::Ciphertext &destination,
                    seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination = encrypted;
            square_inplace(destination, std::move(pool));
        }

        // ---- negate / add / sub (evaluator.cpp:130-350) ------------------------------------------------------------------
        void negate_inplace(seal::Ciphertext &encrypted) const
        {
            validate(encrypted, "encrypted is not valid for encryption parameters");
            check(sb200_negate_host(ctx_, encrypted.coeff_modulus_size(), encrypted.size(), 1, encrypted.data(), encrypted.data()));
            throw_if_transparent(encrypted);
        }
        void negate(const seal::Ciphertext &encrypted, seal::Ciphertext &destination) const
        {
            destination = encrypted;
            negate_inplace(destination);
        }
        void add_inplace(seal::Ciphertext &encrypted1, const seal::Ciphertext &encrypted2) const { linear(encrypted1, encrypted2, false); }
        void add(const seal::Ciphertext &encrypted1, const seal::Ciphertext &encrypted2, seal::Ciphertext &destination) const
        {
            if (&encrypted2 == &destination)
            {
                add_inplace(destination, encrypted1);
            }
            else
            {
                destination = encrypted1;
                add_inplace(destination, encrypted2);
            }
        }
        void sub_inplace(seal::Ciphertext &encrypted1, const seal::Ciphertext &encrypted2) const { linear(encrypted1, encrypted2, true); }
        void sub(const seal::Ciphertext &encrypted1, const seal::Ciphertext &encrypted2, seal::Ciphertext &destination) const
        {
            if (&encrypted2 == &destination)
            {
                sub_inplace(destination, encrypted1);
                negate_inplace(destination);
            }
            else
            {
                destination = encrypted1;
                sub_inplace(destination, encrypted2);
            }
        }

        // ---- multiply_plain (evaluator.cpp:1975-2019 dispatcher, :2157-2195 multiply_plain_ntt, :2021-2155 multiply_plain_normal) ----
        void multiply_plain_inplace(seal::Ciphertext &encrypted, const seal::Plaintext &plain,
                                    seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            validate(encrypted, "encrypted is not valid for encryption parameters");
            if (!seal::is_metadata_valid_for(plain, context_) || !seal::is_buffer_valid(plain))
                throw std::invalid_argument("plain is not valid for encryption parameters");
            if (!pool)
                throw std::invalid_argument("pool is uninitialized");
            const Meta r = multiply_plain_meta(meta(encrypted), meta(plain));
            if (!plain.is_ntt_form())
            {
                // multiply_plain_normal (:2021-2155) / transform + multiply_plain_ntt (:1999-2004)
                const std::vector<std::uint64_t> words = padded(plain);
                check(sb200_multiply_plain_coeff_host(ctx_, encrypted.coeff_modulus_size(), encrypted.size(), 1, encrypted.is_ntt_form() ? 1 : 0,
                                                      encrypted.data(), words.data(), encrypted.data()));
                throw_if_transparent(encrypted);
                return;
            }
            const bool back = !encrypted.is_ntt_form(); // :2006-2011: to NTT form, multiply, back
            if (back)
                transform_to_ntt_inplace(encrypted);
            check(sb200_multiply_plain_host(ctx_, encrypted.coeff_modulus_size(), encrypted.size(), 1, encrypted.data(), plain.data(),
                                            encrypted.data()));
            encrypted.scale() = r.scale;
            if (back)
                transform_from_ntt_inplace(encrypted);
            throw_if_transparent(encrypted);
        }
        void multiply_plain(const seal::Ciphertext &encrypted, const seal::Plaintext &plain, seal::Ciphertext &destination,
                            seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination = encrypted;
            multiply_plain_inplace(destination, plain, std::move(pool));
        }

        // ---- add_plain / sub_plain (evaluator.cpp:1759-1868, :1870-1975) ---------------------------------------------------
        void add_plain_inplace(seal::Ciphertext &encrypted, const seal::Plaintext &plain,
                               seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            plain_linear(encrypted, plain, false);
            (void)pool;
        }
        void add_plain(const seal::Ciphertext &encrypted, const seal::Plaintext &plain, seal::Ciphertext &destination,
                       seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination = encrypted;
            add_plain_inplace(destination, plain, std::move(pool));
        }
        void sub_plain_inplace(seal::Ciphertext &encrypted, const seal::Plaintext &plain,
                               seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            plain_linear(encrypted, plain, true);
            (void)pool;
        }
        void sub_plain(const seal::Ciphertext &encrypted, const seal::Plaintext &plain, seal::Ciphertext &destination,
                       seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination = encrypted;
            sub_plain_inplace(destination, plain, std::move(pool));
        }

        // ---- compositions the reference builds from the operations above ---------------------------------------------
        // add_many (evaluator.cpp:236-262)
        void add_many(const std::vector<seal::Ciphertext> &encrypteds, seal::Ciphertext &destination) const
        {
            if (encrypteds.empty())
                throw std::invalid_argument("encrypteds cannot be empty");
            for (auto &e : encrypteds)
                if (&e == &destination)
                    throw std::invalid_argument("encrypteds must be different from destination");
            destination = encrypteds[0];
            for (std::size_t i = 1; i < encrypteds.size(); i++)
                add_inplace(destination, encrypteds[i]);
        }
        // multiply_many (evaluator.cpp:1649-1724): pairwise products, each relinearized, appended until one is left
        void multiply_many(const std::vector<seal::Ciphertext> &encrypteds, const seal::RelinKeys &relin_keys, seal::Ciphertext &destination,
                           seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            if (encrypteds.empty())
                throw std::invalid_argument("encrypteds vector must not be empty");
            if (!pool)
                throw std::invalid_argument("pool is uninitialized");
            for (auto &e : encrypteds)
                if (&e == &destination)
                    throw std::invalid_argument("encrypteds must be different from destination");
            if (!context_.get_context_data(encrypteds[0].parms_id()))
                throw std::invalid_argument("encrypteds is not valid for encryption parameters");
            if (scheme_ != seal::scheme_type::bfv && scheme_ != seal::scheme_type::bgv)
                throw std::logic_error("unsupported scheme");
            if (encrypteds.size() == 1)
            {
                destination = encrypteds[0];
                return;
            }
            std::vector<seal::Ciphertext> products;
            for (std::size_t i = 0; i + 1 < encrypteds.size(); i += 2)
            {
                seal::Ciphertext temp;
                if (encrypteds[i].data() == encrypteds[i + 1].data())
                    square(encrypteds[i], temp);
                else
                    multiply(encrypteds[i], encrypteds[i + 1], temp);
                relinearize_inplace(temp, relin_keys, pool);
                products.emplace_back(std::move(temp));
            }
            if (encrypteds.size() & 1)
                products.emplace_back(encrypteds.back());
            for (std::size_t i = 0; i + 1 < products.size(); i += 2)
            {
                seal::Ciphertext temp;
                multiply(products[i], products[i + 1], temp);
                relinearize_inplace(temp, relin_keys, pool);
                products.emplace_back(std::move(temp));
            }
            destination = products.back();
        }
        // exponentiate (evaluator.cpp:1726-1757)
        void exponentiate_inplace(seal::Ciphertext &encrypted, std::uint64_t exponent, const seal::RelinKeys &relin_keys,
                                  seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            if (!context_.get_context_data(encrypted.parms_id()))
                throw std::invalid_argument("encrypted is not valid for encryption parameters");
            if (!context_.get_context_data(relin_keys.parms_id()))
                throw std::invalid_argument("relin_keys is not valid for encryption parameters");
            if (!pool)
                throw std::invalid_argument("pool is uninitialized");
            if (exponent == 0)
                throw std::invalid_argument("exponent cannot be 0");
            if (exponent == 1)
                return;
            std::vector<seal::Ciphertext> copies(static_cast<std::size_t>(exponent), encrypted);
            multiply_many(copies, relin_keys, encrypted, std::move(pool));
        }
        void exponentiate(const seal::Ciphertext &encrypted, std::uint64_t exponent, const seal::RelinKeys &relin_keys,
                          seal::Ciphertext &destination, seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination = encrypted;
            exponentiate_inplace(destination, exponent, relin_keys, std::move(pool));
        }
        // mod_switch_to / rescale_to (evaluator.cpp:1451-1473, :1543-1590): repeat the single step down to parms_id
        void mod_switch_to_inplace(seal::Ciphertext &encrypted, seal::parms_id_type parms_id,
                                   seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            check_target_level(encrypted.parms_id(), parms_id);
            while (encrypted.parms_id() != parms_id)
                mod_switch_to_next_inplace(encrypted, pool);
        }
        void mod_switch_to(const seal::Ciphertext &encrypted, seal::parms_id_type parms_id, seal::Ciphertext &destination,
                           seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination = encrypted;
            mod_switch_to_inplace(destination, parms_id, std::move(pool));
        }
        void rescale_to_inplace(seal::Ciphertext &encrypted, seal::parms_id_type parms_id,
                                seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            validate(encrypted, "encrypted is not valid for encryption parameters");
            check_target_level(encrypted.parms_id(), parms_id, true, &pool);
            while (encrypted.parms_id() != parms_id)
            {
                seal::Ciphertext next;
                mod_switch_impl(encrypted, next, true);
                encrypted = std::move(next);
            }
        }
        void rescale_to(const seal::Ciphertext &encrypted, seal::parms_id_type parms_id, seal::Ciphertext &destination,
                        seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination = encrypted;
            rescale_to_inplace(destination, parms_id, std::move(pool));
        }

        // ---- dropping RNS components without scaling: layout only, no arithmetic ----------------------------------------
        // mod_reduce_to_next / mod_reduce_to (evaluator.cpp:1598-1647 -> mod_switch_drop_to_next :1296-1366)
        void mod_reduce_to_next_inplace(seal::Ciphertext &encrypted, seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            validate(encrypted, "encrypted is not valid for encryption parameters");
            check_mod_switch_to_next(meta(encrypted), false, &pool);
            drop_last_component(encrypted);
            throw_if_transparent(encrypted);
        }
        void mod_reduce_to_next(const seal::Ciphertext &encrypted, seal::Ciphertext &destination,
                                seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination = encrypted;
            mod_reduce_to_next_inplace(destination, std::move(pool));
        }
        void mod_reduce_to_inplace(seal::Ciphertext &encrypted, seal::parms_id_type parms_id,
                                   seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            check_target_level(encrypted.parms_id(), parms_id);
            while (encrypted.parms_id() != parms_id)
                mod_reduce_to_next_inplace(encrypted, pool);
        }
        void mod_reduce_to(const seal::Ciphertext &encrypted, seal::parms_id_type parms_id, seal::Ciphertext &destination,
                           seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination = encrypted;
            mod_reduce_to_inplace(destination, parms_id, std::move(pool));
        }
        // NTT-form plaintexts one level down (evaluator.h:431-458, evaluator.cpp:1368-1402): the last component is cut off
        void mod_switch_to_next_inplace(seal::Plaintext &plain) const
        {
            if (!seal::is_valid_for(plain, context_))
                throw std::invalid_argument("plain is not valid for encryption parameters");
            auto &next = plain_next_level(meta(plain));
            const std::size_t words = next.parms().coeff_modulus().size() * next.parms().poly_modulus_degree();
            plain.parms_id() = seal::parms_id_zero;
            plain.resize(words);
            plain.parms_id() = next.parms_id();
        }
        void mod_switch_to_next(const seal::Plaintext &plain, seal::Plaintext &destination) const
        {
            destination = plain;
            mod_switch_to_next_inplace(destination);
        }
        void mod_switch_to_inplace(seal::Plaintext &plain, seal::parms_id_type parms_id) const
        {
            if (!context_.get_context_data(plain.parms_id()))
                throw std::invalid_argument("plain is not valid for encryption parameters");
            check_plain_target_level(meta(plain), parms_id);
            while (plain.parms_id() != parms_id)
                mod_switch_to_next_inplace(plain);
        }
        void mod_switch_to(const seal::Plaintext &plain, seal::parms_id_type parms_id, seal::Plaintext &destination) const
        {
            destination = plain;
            mod_switch_to_inplace(destination, parms_id);
        }

        // ---- relinearize (evaluator.cpp:1144-1199) ---------------------------------------------------------------
        void relinearize_inplace(seal::Ciphertext &encrypted, const seal::RelinKeys &relin_keys,
                                 seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            auto cd = context_.get_context_data(encrypted.parms_id());
            if (!cd)
                throw std::invalid_argument("encrypted is not valid for encryption parameters");
            check_relinearize(relin_keys, encrypted.size());
            if (encrypted.size() == 2)
                return;
            validate(encrypted, "encrypted is not valid for encryption parameters");
            check_switch_key(encrypted.is_ntt_form(), &pool);
            const std::size_t L = encrypted.coeff_modulus_size(), n = encrypted.poly_modulus_degree(), size = encrypted.size();
            std::lock_guard<std::mutex> lock(mu_);
            if (size == 3)
            {
                sb200_kswitch_key *key = key_for(relin_keys, seal::RelinKeys::get_index(2), L);
                std::vector<std::uint64_t> in(encrypted.data(), encrypted.data() + 3 * L * n);
                encrypted.resize(context_, cd->parms_id(), 2);
                check(sb200_relinearize_host(ctx_, L, 1, in.data(), key, encrypted.data()));
                throw_if_transparent(encrypted);
                return;
            }
            // size > 3, exactly as the reference's loop is written (evaluator.cpp:1176-1187): every step key-switches the LAST
            // polynomial (the iterator is not advanced) with the key of index size-1-I, then the ciphertext is cut to 2 polynomials
            std::vector<std::uint64_t> cur(encrypted.data(), encrypted.data() + size * L * n), next(cur.size());
            for (std::size_t I = 0; I < size - 2; I++)
            {
                sb200_kswitch_key *key = key_for(relin_keys, seal::RelinKeys::get_index(size - 1 - I), L);
                check(sb200_relinearize_sized_host(ctx_, L, size, 1, cur.data(), key, next.data()));
                cur.swap(next);
            }
            encrypted.resize(context_, cd->parms_id(), 2);
            std::memcpy(encrypted.data(), cur.data(), 2 * L * n * sizeof(std::uint64_t));
            throw_if_transparent(encrypted);
        }
        void relinearize(const seal::Ciphertext &encrypted, const seal::RelinKeys &relin_keys, seal::Ciphertext &destination,
                         seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination = encrypted;
            relinearize_inplace(destination, relin_keys, std::move(pool));
        }

        // ---- rescale / mod switch (evaluator.cpp:1404-1541, 1201-1358) --------------------------------------------
        void rescale_to_next(const seal::Ciphertext &encrypted, seal::Ciphertext &destination,
                             seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            validate(encrypted, "encrypted is not valid for encryption parameters");
            check_mod_switch_to_next(meta(encrypted), true, &pool);
            mod_switch_impl(encrypted, destination, true);
        }
        void rescale_to_next_inplace(seal::Ciphertext &encrypted, seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            rescale_to_next(encrypted, encrypted, std::move(pool));
        }
        void mod_switch_to_next(const seal::Ciphertext &encrypted, seal::Ciphertext &destination,
                                seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            validate(encrypted, "encrypted is not valid for encryption parameters");
            check_mod_switch_to_next(meta(encrypted), false, &pool);
            mod_switch_impl(encrypted, destination, false);
        }
        void mod_switch_to_next_inplace(seal::Ciphertext &encrypted, seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            mod_switch_to_next(encrypted, encrypted, std::move(pool));
        }

        // ---- Galois automorphisms and rotations (evaluator.cpp:2384-2559, evaluator.h:1006-1316) ---------------------
        void apply_galois_inplace(seal::Ciphertext &encrypted, std::uint32_t galois_elt, const seal::GaloisKeys &galois_keys,
                                  seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            validate(encrypted, "encrypted is not valid for encryption parameters");
            check_apply_galois(meta(encrypted), galois_elt, galois_keys, &pool);
            const std::size_t L = encrypted.coeff_modulus_size(), n = encrypted.poly_modulus_degree();
            std::lock_guard<std::mutex> lock(mu_); // the cached key stays valid (not evicted) while the operation uses it
            sb200_kswitch_key *key = key_for(galois_keys, seal::GaloisKeys::get_index(galois_elt), L);
            std::vector<std::uint64_t> in(encrypted.data(), encrypted.data() + 2 * L * n);
            check(sb200_apply_galois_host(ctx_, L, 1, in.data(), galois_elt, key, encrypted.data()));
            throw_if_transparent(encrypted);
        }
        void apply_galois(const seal::Ciphertext &encrypted, std::uint32_t galois_elt, const seal::GaloisKeys &galois_keys,
                          seal::Ciphertext &destination, seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination = encrypted;
            apply_galois_inplace(destination, galois_elt, galois_keys, std::move(pool));
        }
        void rotate_rows_inplace(seal::Ciphertext &encrypted, int steps, const seal::GaloisKeys &galois_keys,
                                 seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            if (scheme_ != seal::scheme_type::bfv && scheme_ != seal::scheme_type::bgv) // evaluator.h:1076-1080, 1145-1149
                throw std::logic_error("unsupported scheme");
            rotate_internal(encrypted, steps, galois_keys, std::move(pool));
        }
        void rotate_rows(const seal::Ciphertext &encrypted, int steps, const seal::GaloisKeys &galois_keys, seal::Ciphertext &destination,
                         seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination = encrypted;
            rotate_rows_inplace(destination, steps, galois_keys, std::move(pool));
        }
        void rotate_columns_inplace(seal::Ciphertext &encrypted, const seal::GaloisKeys &galois_keys,
                                    seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            if (scheme_ != seal::scheme_type::bfv && scheme_ != seal::scheme_type::bgv) // evaluator.h:1076-1080, 1145-1149
                throw std::logic_error("unsupported scheme");
            conjugate_internal(encrypted, galois_keys, std::move(pool));
        }
        void rotate_columns(const seal::Ciphertext &encrypted, const seal::GaloisKeys &galois_keys, seal::Ciphertext &destination,
                            seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination = encrypted;
            rotate_columns_inplace(destination, galois_keys, std::move(pool));
        }
        void rotate_vector_inplace(seal::Ciphertext &encrypted, int steps, const seal::GaloisKeys &galois_keys,
                                   seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            if (scheme_ != seal::scheme_type::ckks)
                throw std::logic_error("unsupported scheme");
            rotate_internal(encrypted, steps, galois_keys, std::move(pool));
        }
        void rotate_vector(const seal::Ciphertext &encrypted, int steps, const seal::GaloisKeys &galois_keys, seal::Ciphertext &destination,
                           seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination = encrypted;
            rotate_vector_inplace(destination, steps, galois_keys, std::move(pool));
        }
        void complex_conjugate_inplace(seal::Ciphertext &encrypted, const seal::GaloisKeys &galois_keys,
                                       seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            if (scheme_ != seal::scheme_type::ckks)
                throw std::logic_error("unsupported scheme");
            conjugate_internal(encrypted, galois_keys, std::move(pool));
        }
        void complex_conjugate(const seal::Ciphertext &encrypted, const seal::GaloisKeys &galois_keys, seal::Ciphertext &destination,
                               seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination = encrypted;
            complex_conjugate_inplace(destination, galois_keys, std::move(pool));
        }

        // ---- NTT form changes (evaluator.cpp:2289-2382) -------------------------------------------------------------
        void transform_to_ntt_inplace(seal::Ciphertext &encrypted) const
        {
            validate(encrypted, "encrypted is not valid for encryption parameters");
            if (encrypted.is_ntt_form())
                throw std::invalid_argument("encrypted is already in NTT form");
            check(sb200_ntt_forward_host(ctx_, encrypted.coeff_modulus_size(), encrypted.size(), 1, encrypted.data()));
            encrypted.is_ntt_form() = true;
            throw_if_transparent(encrypted);
        }
        void transform_to_ntt(const seal::Ciphertext &encrypted, seal::Ciphertext &destination_ntt) const
        {
            destination_ntt = encrypted;
            transform_to_ntt_inplace(destination_ntt);
        }
        void transform_from_ntt_inplace(seal::Ciphertext &encrypted_ntt) const
        {
            validate(encrypted_ntt, "encrypted is not valid for encryption parameters");
            if (!encrypted_ntt.is_ntt_form())
                throw std::invalid_argument("encrypted_ntt is not in NTT form");
            check(sb200_ntt_inverse_host(ctx_, encrypted_ntt.coeff_modulus_size(), encrypted_ntt.size(), 1, encrypted_ntt.data()));
            encrypted_ntt.is_ntt_form() = false;
            throw_if_transparent(encrypted_ntt);
        }
        void transform_from_ntt(const seal::Ciphertext &encrypted_ntt, seal::Ciphertext &destination) const
        {
            destination = encrypted_ntt;
            transform_from_ntt_inplace(destination);
        }

        // transform_to_ntt_inplace(Plaintext&, parms_id) (evaluator.cpp:2197-2287)
        void transform_to_ntt_inplace(seal::Plaintext &plain, seal::parms_id_type parms_id,
                                      seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            if (!seal::is_valid_for(plain, context_))
                throw std::invalid_argument("plain is not valid for encryption parameters");
            auto cd = context_.get_context_data(parms_id);
            if (!cd)
                throw std::invalid_argument("parms_id is not valid for the current context");
            if (plain.is_ntt_form())
                throw std::invalid_argument("plain is already in NTT form");
            if (!pool)
                throw std::invalid_argument("pool is uninitialized");
            const std::vector<std::uint64_t> words = padded(plain);
            const std::size_t L = cd->parms().coeff_modulus().size(), n = cd->parms().poly_modulus_degree();
            plain.resize(n * L);
            check(sb200_plain_to_ntt_host(ctx_, L, 1, words.data(), plain.data()));
            plain.parms_id() = parms_id;
        }
        void transform_to_ntt(const seal::Plaintext &plain, seal::parms_id_type parms_id, seal::Plaintext &destination_ntt,
                              seal::MemoryPoolHandle pool = seal::MemoryManager::GetPool()) const
        {
            destination_ntt = plain;
            transform_to_ntt_inplace(destination_ntt, parms_id, std::move(pool));
        }

        // ---- batch extension: destination[i] = relinearize(multiply(a[i], b[i])), one device pass over the batch ----
        // (upload through page-locked staging, fused multiply + relinearize on the device, download).  The checks are
        // multiply_inplace's for every entry, then relinearize_inplace's; the entries must have size 2 and share one level.  Scales and
        // BGV correction factors may differ from ciphertext to ciphertext; they are computed before anything is written, so
        // destination may alias a or b.
        void multiply_relinearize(const std::vector<seal::Ciphertext> &a, const std::vector<seal::Ciphertext> &b,
                                  const seal::RelinKeys &relin_keys, std::vector<seal::Ciphertext> &destination) const
        {
            if (a.size() != b.size() || a.empty())
                throw std::invalid_argument("batch size mismatch");
            const std::size_t B = a.size();
            std::vector<Meta> products;
            for (std::size_t i = 0; i < B; i++)
            {
                validate(a[i], "encrypted1 is not valid for encryption parameters");
                validate(b[i], "encrypted2 is not valid for encryption parameters");
                products.push_back(multiply_meta(meta(a[i]), meta(b[i])));
                if (a[i].size() != 2 || b[i].size() != 2 || a[i].parms_id() != a[0].parms_id())
                    throw std::invalid_argument("batch entries must be fresh size-2 ciphertexts in the scheme's native form");
            }
            check_relinearize(relin_keys, 3);
            check_switch_key(products[0].ntt);
            CiphertextBatch da, db;
            upload_rows(a.data(), B, da);
            upload_rows(b.data(), B, db);
            da.scale_ = db.scale_ = 1.0; // per-ciphertext metadata is applied below
            multiply_relinearize_inplace(da, db, relin_keys);
            download(da, destination);
            for (std::size_t i = 0; i < B; i++)
            {
                destination[i].scale() = products[i].scale;
                destination[i].correction_factor() = products[i].cf;
            }
        }

        // =================================== device-resident batches (CiphertextBatch) ===================================
        // Same members, same checks and metadata updates as the seal::Ciphertext overloads above; the data never leaves the GPU.
        void upload(const std::vector<seal::Ciphertext> &cts, CiphertextBatch &destination) const
        {
            upload(cts.data(), cts.size(), destination);
        }
        // a contiguous range of ciphertext objects (e.g. one slice of a larger vector: slices of a batch can be uploaded, processed and
        // downloaded by different host threads so that the copies of one slice overlap the kernels of another)
        void upload(const seal::Ciphertext *first, std::size_t count, CiphertextBatch &destination) const
        {
            if (!first || !count)
                throw std::invalid_argument("batch cannot be empty");
            const seal::Ciphertext &f = first[0];
            for (std::size_t i = 0; i < count; i++)
            {
                const seal::Ciphertext &c = first[i];
                validate(c, "encrypted is not valid for encryption parameters");
                const double s1 = c.scale(), s2 = f.scale();
                if (c.parms_id() != f.parms_id() || c.size() != f.size() || c.is_ntt_form() != f.is_ntt_form() ||
                    c.correction_factor() != f.correction_factor() || std::memcmp(&s1, &s2, sizeof(double)) != 0)
                    throw std::invalid_argument("batch members must share parms_id, size, NTT form, scale and correction factor");
            }
            upload_rows(first, count, destination);
        }
        void download(const CiphertextBatch &source, std::vector<seal::Ciphertext> &cts) const
        {
            cts.resize(source.batch_);
            download(source, cts.data());
        }
        void download(const CiphertextBatch &source, seal::Ciphertext *cts) const
        {
            owned(source);
            if (!cts)
                throw std::invalid_argument("destination cannot be null");
            std::vector<std::uint64_t *> rows(source.batch_);
            for (std::size_t i = 0; i < source.batch_; i++)
            {
                cts[i].resize(context_, source.parms_id_, source.size_);
                cts[i].is_ntt_form() = source.ntt_;
                cts[i].scale() = source.scale_;
                cts[i].correction_factor() = source.cf_;
                rows[i] = cts[i].data();
            }
            check(sb200_download_rows(ctx_, rows.data(), source.d_, source.words_per_ciphertext() * sizeof(std::uint64_t), source.batch_));
            for (std::size_t i = 0; i < source.batch_; i++)
                throw_if_transparent(cts[i]);
        }
        void copy(const CiphertextBatch &source, CiphertextBatch &destination) const
        {
            owned(source);
            std::lock_guard<std::mutex> lock(mu_);
            shape(destination, source.batch_, source.size_, source.L_, source.n_);
            assign(destination, meta(source));
            check(sb200_memcpy_d2d(ctx_, destination.d_, source.d_, source.batch_ * source.words_per_ciphertext() * sizeof(std::uint64_t), nullptr));
        }
        // Ciphertext::load / unsafe_load (ciphertext.cpp:249-395) of `count` streams into one batch: none, zlib and seeded streams,
        // words copied from the streams to the device and seeded c_1s expanded there (sb200_ciphertext_load).  The members must share
        // parms_id, size, NTT form, scale and correction factor (std::invalid_argument, raised before anything is written); a stream
        // the reference rejects throws what Ciphertext::load throws.  destination changes only on success.
        void load(const seal::seal_byte *const *streams, const std::size_t *sizes, std::size_t count, CiphertextBatch &destination) const
        {
            load_batch(streams, sizes, count, true, destination);
        }
        void unsafe_load(const seal::seal_byte *const *streams, const std::size_t *sizes, std::size_t count, CiphertextBatch &destination) const
        {
            load_batch(streams, sizes, count, false, destination);
        }
        // Ciphertext::save (ciphertext.cpp:190-247) of every member: streams[i] = the bytes seal::Ciphertext::save(compr_mode) writes for
        // member i.  compr_mode none is written from the device (sb200_ciphertext_save); other modes hand those members to
        // seal::Serialization::Save, as Ciphertext::save does.
        void save(const CiphertextBatch &source, std::vector<std::vector<seal::seal_byte>> &streams,
                  seal::compr_mode_type compr_mode = seal::Serialization::compr_mode_default) const
        {
            owned(source);
            const std::size_t plain = sb200_ciphertext_save_size(ctx_, source.L_, source.size_), B = source.batch_;
            std::vector<std::vector<seal::seal_byte>> out(B, std::vector<seal::seal_byte>(plain));
            std::vector<std::uint8_t *> ptrs(B);
            std::vector<sb200_ct_info> meta(B);
            for (std::size_t i = 0; i < B; i++)
            {
                ptrs[i] = reinterpret_cast<std::uint8_t *>(out[i].data());
                meta[i].is_ntt_form = source.ntt_ ? 1 : 0, meta[i].scale = source.scale_, meta[i].correction_factor = source.cf_;
            }
            {
                std::lock_guard<std::mutex> lock(mu_);
                check(sb200_ciphertext_save(ctx_, B, source.L_, source.size_, source.d_, meta.data(), ptrs.data(), plain, nullptr));
            }
            if (compr_mode != seal::compr_mode_type::none)
                for (auto &s : out)
                {
                    std::vector<seal::seal_byte> z(static_cast<std::size_t>(save_size_of(plain, compr_mode)));
                    const auto got = seal::Serialization::Save(
                        [&s](std::ostream &o) { o.write(reinterpret_cast<const char *>(s.data() + kSealHeader), static_cast<std::streamsize>(s.size() - kSealHeader)); },
                        static_cast<std::streamoff>(s.size()), z.data(), z.size(), compr_mode, false);
                    z.resize(static_cast<std::size_t>(got));
                    s = std::move(z);
                }
            streams = std::move(out);
        }
        // Ciphertext::save_size of one member (an upper bound for compressed modes, as the reference's)
        std::streamoff save_size(const CiphertextBatch &source, seal::compr_mode_type compr_mode = seal::Serialization::compr_mode_default) const
        {
            owned(source);
            return save_size_of(sb200_ciphertext_save_size(ctx_, source.L_, source.size_), compr_mode);
        }

        // ---- device-resident key sets (DeviceRelinKeys / DeviceGaloisKeys) ----
        // RelinKeys::load / GaloisKeys::load (kswitchkeys.cpp:42-160) straight onto the device, for streams saved with compr_mode none
        // or zlib and the seeded streams of KeyGenerator's Serializable overloads: the object is inflated and parsed once, and seeded
        // c_1s expand on the device (sb200_kswitch_keys_load).  A stream the reference rejects throws what its load throws.
        // destination changes only on success.
        void load(const seal::seal_byte *in, std::size_t size, DeviceRelinKeys &destination) const { load_keys(in, size, nullptr, 0, destination); }
        void load(const seal::seal_byte *in, std::size_t size, DeviceGaloisKeys &destination) const
        {
            load_keys(in, size, nullptr, context_.key_context_data()->parms().poly_modulus_degree(), destination);
        }
        // only the keys of galois_elts (any order, duplicates ignored): at n = 65536 a server loads the keys that fit on the device.  An
        // element without a key in the stream: std::invalid_argument.
        void load(const seal::seal_byte *in, std::size_t size, const std::vector<std::uint32_t> &galois_elts, DeviceGaloisKeys &destination) const
        {
            std::vector<std::size_t> slots;
            for (const std::uint32_t elt : galois_elts)
            {
                const std::size_t s = seal::GaloisKeys::get_index(elt);
                if (std::find(slots.begin(), slots.end(), s) == slots.end())
                    slots.push_back(s);
            }
            load_keys(in, size, &slots, context_.key_context_data()->parms().poly_modulus_degree(), destination);
        }
        // the non-empty slots of a seal:: key object, one device key each (sb200_kswitch_key_create)
        void upload(const seal::RelinKeys &keys, DeviceRelinKeys &destination) const { upload_keys(keys, destination); }
        void upload(const seal::GaloisKeys &keys, DeviceGaloisKeys &destination) const { upload_keys(keys, destination); }
        // Evaluator::multiply_inplace (evaluator.cpp:352-393), any sizes
        void multiply_inplace(CiphertextBatch &encrypted1, const CiphertextBatch &encrypted2) const
        {
            owned(encrypted1), owned(encrypted2);
            const Meta r = multiply_meta(meta(encrypted1), meta(encrypted2));
            std::lock_guard<std::mutex> lock(mu_);
            std::uint64_t *out = out_slab(encrypted1.batch_ * r.size * encrypted1.L_ * encrypted1.n_, encrypted1);
            check(sb200_multiply_sized(ctx_, encrypted1.L_, encrypted1.size_, encrypted2.size_, encrypted1.batch_, encrypted1.d_, encrypted2.d_, out,
                                       nullptr));
            adopt(encrypted1);
            assign(encrypted1, r);
        }
        void square_inplace(CiphertextBatch &encrypted) const { multiply_inplace(encrypted, encrypted); }
        // Evaluator::relinearize_inplace (evaluator.cpp:1144-1199).  Every key-switching member of a batch takes the keys as a seal::
        // object (uploaded through the key cache) or as a device key set; both overloads share one body, which differs only in key_for.
        void relinearize_inplace(CiphertextBatch &encrypted, const seal::RelinKeys &relin_keys) const { relinearize_batch(encrypted, relin_keys); }
        void relinearize_inplace(CiphertextBatch &encrypted, const DeviceRelinKeys &relin_keys) const { relinearize_batch(encrypted, relin_keys); }
        // multiply + relinearize in one device pass (both operands size 2); the result replaces encrypted1
        void multiply_relinearize_inplace(CiphertextBatch &encrypted1, const CiphertextBatch &encrypted2, const seal::RelinKeys &relin_keys) const
        {
            multiply_relinearize_batch(encrypted1, encrypted2, relin_keys);
        }
        void multiply_relinearize_inplace(CiphertextBatch &encrypted1, const CiphertextBatch &encrypted2, const DeviceRelinKeys &relin_keys) const
        {
            multiply_relinearize_batch(encrypted1, encrypted2, relin_keys);
        }

    private:
        template <class RelinKeys>
        void relinearize_batch(CiphertextBatch &encrypted, const RelinKeys &relin_keys) const
        {
            owned(encrypted);
            check_relinearize(relin_keys, encrypted.size_);
            if (encrypted.size_ == 2)
                return;
            check_switch_key(encrypted.ntt_);
            std::lock_guard<std::mutex> lock(mu_);
            const std::size_t size = encrypted.size_, poly = encrypted.L_ * encrypted.n_;
            if (size == 3)
            {
                sb200_kswitch_key *key = key_for(relin_keys, seal::RelinKeys::get_index(2), encrypted.L_);
                std::uint64_t *out = out_slab(encrypted.batch_ * 2 * poly, encrypted);
                check(sb200_relinearize(ctx_, encrypted.L_, encrypted.batch_, encrypted.d_, key, out, nullptr));
                adopt(encrypted);
                encrypted.size_ = 2;
                return;
            }
            // size > 3, as the reference's loop is written (evaluator.cpp:1176-1187): every step key-switches the LAST polynomial
            // with the key of index size-1-I; afterwards the ciphertexts are cut to 2 polynomials
            for (std::size_t I = 0; I < size - 2; I++)
            {
                sb200_kswitch_key *key = key_for(relin_keys, seal::RelinKeys::get_index(size - 1 - I), encrypted.L_);
                std::uint64_t *out = out_slab(encrypted.batch_ * size * poly, encrypted);
                check(sb200_relinearize_sized(ctx_, encrypted.L_, size, encrypted.batch_, encrypted.d_, key, out, nullptr));
                adopt(encrypted);
            }
            std::uint64_t *out = out_slab(encrypted.batch_ * 2 * poly, encrypted);
            check(sb200_memcpy_d2d_2d(ctx_, out, 2 * poly * sizeof(std::uint64_t), encrypted.d_, size * poly * sizeof(std::uint64_t),
                                      2 * poly * sizeof(std::uint64_t), encrypted.batch_, nullptr));
            adopt(encrypted);
            encrypted.size_ = 2;
        }
        template <class RelinKeys>
        void multiply_relinearize_batch(CiphertextBatch &encrypted1, const CiphertextBatch &encrypted2, const RelinKeys &relin_keys) const
        {
            owned(encrypted1), owned(encrypted2);
            if (encrypted1.size_ != 2 || encrypted2.size_ != 2)
            {
                multiply_inplace(encrypted1, encrypted2);
                relinearize_inplace(encrypted1, relin_keys);
                return;
            }
            Meta r = multiply_meta(meta(encrypted1), meta(encrypted2)); // the chain's checks: multiply_inplace's, relinearize_inplace's
            check_relinearize(relin_keys, r.size);
            check_switch_key(r.ntt);
            std::lock_guard<std::mutex> lock(mu_);
            sb200_kswitch_key *key = key_for(relin_keys, seal::RelinKeys::get_index(2), encrypted1.L_);
            check(sb200_multiply_relinearize(ctx_, encrypted1.L_, encrypted1.batch_, encrypted1.d_, encrypted2.d_, key, encrypted1.d_, nullptr));
            r.size = 2;
            assign(encrypted1, r);
        }

    public:
        // Evaluator::rescale_to_next_inplace / mod_switch_to_next_inplace (evaluator.cpp:1404-1541), any size
        void rescale_to_next_inplace(CiphertextBatch &encrypted) const
        {
            owned(encrypted);
            check_mod_switch_to_next(meta(encrypted), true);
            mod_switch_batch(encrypted, true);
        }
        void mod_switch_to_next_inplace(CiphertextBatch &encrypted) const
        {
            owned(encrypted);
            check_mod_switch_to_next(meta(encrypted), false);
            mod_switch_batch(encrypted, false);
        }
        // add / sub / negate (evaluator.cpp:130-350), any sizes and correction factors: the result takes the larger size, the longer
        // operand's tail is copied (add) or negated (sub), and BGV operands with different correction factors are first scaled by
        // the balancing factors -- all in one sb200_add_many pass
        void add_inplace(CiphertextBatch &encrypted1, const CiphertextBatch &encrypted2) const { linear_batch(encrypted1, encrypted2, false); }
        void sub_inplace(CiphertextBatch &encrypted1, const CiphertextBatch &encrypted2) const { linear_batch(encrypted1, encrypted2, true); }
        // add_many (evaluator.cpp:236-262), member-wise: member i of destination is add_many of member i of every operand.  One
        // sb200_add_many pass reads every operand once and writes destination once (the reference's chain of add_inplace calls
        // moves 3 (m - 1) slabs); the chain's correction factors are replayed on the host to fill the steps.
        void add_many(const std::vector<CiphertextBatch> &encrypteds, CiphertextBatch &destination) const
        {
            if (encrypteds.empty())
                throw std::invalid_argument("encrypteds cannot be empty");
            for (auto &e : encrypteds)
                if (&e == &destination)
                    throw std::invalid_argument("encrypteds must be different from destination");
            const CiphertextBatch &e0 = encrypteds[0];
            owned(e0);
            Fold f{ meta(e0), { e0.size_ }, {}, {} };
            std::vector<const std::uint64_t *> ptrs{ e0.d_ };
            for (std::size_t j = 1; j < encrypteds.size(); j++)
            {
                owned(encrypteds[j]);
                fold_in(f, meta(encrypteds[j]), SB200_FOLD_ADD);
                ptrs.push_back(encrypteds[j].d_);
            }
            std::lock_guard<std::mutex> lock(mu_);
            shape(destination, e0.batch_, f.result.size, e0.L_, e0.n_);
            assign(destination, f.result);
            check(sb200_add_many(ctx_, e0.L_, e0.batch_, ptrs.size(), f.sizes.data(), ptrs.data(), f.modes.data(),
                                 f.factors.empty() ? nullptr : f.factors.data(), destination.d_, nullptr));
        }
        // Sums of plaintext products, member-wise: destination j is add_many over i of multiply_plain(encrypteds[i], plains[j K + i])
        // (K = encrypteds.size()), with the chain's checks, messages and metadata: multiply_plain_inplace's for terms 0 .. K - 1 in
        // order, then add_many's (correction factors balanced as plan_fold balances them), output by output.  One
        // sb200_multiply_plain_sum pass reads every ciphertext once per tile of outputs and every plaintext once.  The plaintexts must
        // all be in NTT form or all in coefficient form.
        void multiply_plain_sum(const std::vector<CiphertextBatch> &encrypteds, const std::vector<PlaintextBatch> &plains,
                                CiphertextBatch &destination) const
        {
            if (encrypteds.empty())
                throw std::invalid_argument("encrypteds cannot be empty");
            for (auto &e : encrypteds)
                if (&e == &destination)
                    throw std::invalid_argument("encrypteds must be different from destination");
            if (plains.size() != encrypteds.size())
                throw std::invalid_argument("plains must hold one plaintext batch per encrypted");
            const PlainSum p = plan_plain_sum(encrypteds, plains, 1);
            std::lock_guard<std::mutex> lock(mu_);
            std::uint64_t *out = plain_sum_output(encrypteds[0], p, 0, destination);
            run_plain_sum(encrypteds, plains, p, &out);
        }
        void multiply_plain_sum(const std::vector<CiphertextBatch> &encrypteds, const std::vector<PlaintextBatch> &plains,
                                std::vector<CiphertextBatch> &destinations) const
        {
            if (encrypteds.empty())
                throw std::invalid_argument("encrypteds cannot be empty");
            if (&destinations == &encrypteds)
                throw std::invalid_argument("encrypteds must be different from destination");
            if (plains.empty() || plains.size() % encrypteds.size() != 0)
                throw std::invalid_argument("plains must hold K plaintext batches per destination");
            const std::size_t M = plains.size() / encrypteds.size();
            const PlainSum p = plan_plain_sum(encrypteds, plains, M);
            std::lock_guard<std::mutex> lock(mu_);
            destinations.resize(M);
            std::vector<std::uint64_t *> outs(M);
            for (std::size_t j = 0; j < M; j++)
                outs[j] = plain_sum_output(encrypteds[0], p, j, destinations[j]);
            run_plain_sum(encrypteds, plains, p, outs.data());
        }
        // Sums of ciphertext products, member-wise: destination j is add_many over i of multiply(encrypteds1[j K + i], encrypteds2[i])
        // (K = encrypteds2.size()), the size-3 products summed before any relinearization (the lazy-relinearization idiom of
        // inner products and encrypted matrix x encrypted vector by diagonals).  The chain's checks, messages and metadata:
        // multiply_inplace's for terms 0 .. K - 1 in order, then add_many's (correction factors cf(a) cf(b) mod t balanced as
        // plan_fold balances them), output by output, all before anything is written.  When every operand has size 2, one
        // sb200_multiply_sum call forms every output (one per output when BGV's balancing differs between outputs); other sizes take
        // the chain itself (a copy, multiply_inplace, then add_many).  An operand of encrypteds1 may be one of encrypteds2 (squares).
        void multiply_sum(const std::vector<CiphertextBatch> &encrypteds1, const std::vector<CiphertextBatch> &encrypteds2,
                          CiphertextBatch &destination) const
        {
            check_sum_destination(encrypteds1, encrypteds2, destination);
            if (encrypteds1.size() != encrypteds2.size())
                throw std::invalid_argument("encrypteds1 must hold K ciphertext batches per destination");
            const MultiplySum p = plan_multiply_sum(encrypteds1, encrypteds2, 1);
            CiphertextBatch *d = &destination;
            run_multiply_sum(encrypteds1, encrypteds2, p, &d);
        }
        void multiply_sum(const std::vector<CiphertextBatch> &encrypteds1, const std::vector<CiphertextBatch> &encrypteds2,
                          std::vector<CiphertextBatch> &destinations) const
        {
            const std::size_t M = sum_outputs(encrypteds1, encrypteds2, destinations);
            const MultiplySum p = plan_multiply_sum(encrypteds1, encrypteds2, M);
            destinations.resize(M);
            std::vector<CiphertextBatch *> d;
            for (auto &x : destinations)
                d.push_back(&x);
            run_multiply_sum(encrypteds1, encrypteds2, p, d.data());
        }
        // multiply_sum, then relinearize_inplace of every destination: one key switch per sum.  relinearize_inplace's checks run
        // with the others, before anything is written.
        void multiply_relinearize_sum(const std::vector<CiphertextBatch> &encrypteds1, const std::vector<CiphertextBatch> &encrypteds2,
                                      const seal::RelinKeys &relin_keys, CiphertextBatch &destination) const
        {
            multiply_relinearize_sum_one(encrypteds1, encrypteds2, relin_keys, destination);
        }
        void multiply_relinearize_sum(const std::vector<CiphertextBatch> &encrypteds1, const std::vector<CiphertextBatch> &encrypteds2,
                                      const DeviceRelinKeys &relin_keys, CiphertextBatch &destination) const
        {
            multiply_relinearize_sum_one(encrypteds1, encrypteds2, relin_keys, destination);
        }
        void multiply_relinearize_sum(const std::vector<CiphertextBatch> &encrypteds1, const std::vector<CiphertextBatch> &encrypteds2,
                                      const seal::RelinKeys &relin_keys, std::vector<CiphertextBatch> &destinations) const
        {
            multiply_relinearize_sum_many(encrypteds1, encrypteds2, relin_keys, destinations);
        }
        void multiply_relinearize_sum(const std::vector<CiphertextBatch> &encrypteds1, const std::vector<CiphertextBatch> &encrypteds2,
                                      const DeviceRelinKeys &relin_keys, std::vector<CiphertextBatch> &destinations) const
        {
            multiply_relinearize_sum_many(encrypteds1, encrypteds2, relin_keys, destinations);
        }
        // multiply_many (evaluator.cpp:1649-1724), member-wise, BFV and BGV.  The reference's queue of products is replayed on
        // operand ids (schedule_products); products that do not depend on each other run as one wave: their operand pairs are staged
        // into two slabs and multiplied and relinearized by one sb200_multiply_relinearize call, one pass over the relinearization
        // key per key-switching chunk.  Each product is a function of its two operands alone, so the words are the reference's.
        void multiply_many(const std::vector<CiphertextBatch> &encrypteds, const seal::RelinKeys &relin_keys, CiphertextBatch &destination) const
        {
            multiply_many_batch(encrypteds, relin_keys, destination);
        }
        void multiply_many(const std::vector<CiphertextBatch> &encrypteds, const DeviceRelinKeys &relin_keys, CiphertextBatch &destination) const
        {
            multiply_many_batch(encrypteds, relin_keys, destination);
        }
        // exponentiate (evaluator.cpp:1726-1757): multiply_many of `exponent` copies of encrypted, with the copies' queue kept in
        // run-length form so that the schedule costs O(log exponent) and equal products are computed once (4 products for exponent
        // 16, 5 for 13, against the reference's exponent - 1).  The reference allocates the copies and fails with std::bad_alloc
        // for an exponent it cannot allocate; this member allocates no copies and does not reproduce that failure.
        void exponentiate_inplace(CiphertextBatch &encrypted, std::uint64_t exponent, const seal::RelinKeys &relin_keys) const
        {
            exponentiate_batch(encrypted, exponent, relin_keys);
        }
        void exponentiate_inplace(CiphertextBatch &encrypted, std::uint64_t exponent, const DeviceRelinKeys &relin_keys) const
        {
            exponentiate_batch(encrypted, exponent, relin_keys);
        }
        void exponentiate(const CiphertextBatch &encrypted, std::uint64_t exponent, const seal::RelinKeys &relin_keys,
                          CiphertextBatch &destination) const
        {
            copy(encrypted, destination);
            exponentiate_inplace(destination, exponent, relin_keys);
        }
        void exponentiate(const CiphertextBatch &encrypted, std::uint64_t exponent, const DeviceRelinKeys &relin_keys,
                          CiphertextBatch &destination) const
        {
            copy(encrypted, destination);
            exponentiate_inplace(destination, exponent, relin_keys);
        }

    private:
        template <class RelinKeys>
        void multiply_many_batch(const std::vector<CiphertextBatch> &encrypteds, const RelinKeys &relin_keys, CiphertextBatch &destination) const
        {
            if (encrypteds.empty())
                throw std::invalid_argument("encrypteds vector must not be empty");
            for (auto &e : encrypteds)
                if (&e == &destination)
                    throw std::invalid_argument("encrypteds must be different from destination");
            if (!context_.get_context_data(encrypteds[0].parms_id_))
                throw std::invalid_argument("encrypteds is not valid for encryption parameters");
            if (scheme_ != seal::scheme_type::bfv && scheme_ != seal::scheme_type::bgv)
                throw std::logic_error("unsupported scheme");
            std::vector<const CiphertextBatch *> leaves;
            std::vector<std::pair<std::size_t, std::uint64_t>> runs;
            for (auto &e : encrypteds)
            {
                runs.emplace_back(leaves.size(), 1);
                leaves.push_back(&e);
            }
            run_products(leaves, schedule_products(leaves.size(), runs), relin_keys, destination);
        }
        template <class RelinKeys>
        void exponentiate_batch(CiphertextBatch &encrypted, std::uint64_t exponent, const RelinKeys &relin_keys) const
        {
            if (!context_.get_context_data(encrypted.parms_id_))
                throw std::invalid_argument("encrypted is not valid for encryption parameters");
            if (!context_.get_context_data(relin_keys.parms_id()))
                throw std::invalid_argument("relin_keys is not valid for encryption parameters");
            if (exponent == 0)
                throw std::invalid_argument("exponent cannot be 0");
            if (exponent == 1)
                return;
            if (scheme_ != seal::scheme_type::bfv && scheme_ != seal::scheme_type::bgv)
                throw std::logic_error("unsupported scheme");
            CiphertextBatch result;
            run_products({ &encrypted }, schedule_products(1, { { 0, exponent } }), relin_keys, result);
            encrypted = std::move(result);
        }

    public:
        // mod_switch_to / rescale_to (evaluator.cpp:1451-1473, :1543-1590): the reference's checks, then single steps down to parms_id
        void mod_switch_to_inplace(CiphertextBatch &encrypted, seal::parms_id_type parms_id) const
        {
            owned(encrypted);
            check_target_level(encrypted.parms_id_, parms_id);
            while (encrypted.parms_id_ != parms_id)
                mod_switch_to_next_inplace(encrypted);
        }
        void rescale_to_inplace(CiphertextBatch &encrypted, seal::parms_id_type parms_id) const
        {
            owned(encrypted);
            check_target_level(encrypted.parms_id_, parms_id, true);
            while (encrypted.parms_id_ != parms_id)
                rescale_to_next_inplace(encrypted);
        }
        void negate_inplace(CiphertextBatch &encrypted) const
        {
            owned(encrypted);
            std::lock_guard<std::mutex> lock(mu_);
            check(sb200_negate(ctx_, encrypted.L_, encrypted.size_, encrypted.batch_, encrypted.d_, encrypted.d_, nullptr));
        }
        // apply_galois / rotations (evaluator.cpp:2384-2559)
        void apply_galois_inplace(CiphertextBatch &encrypted, std::uint32_t galois_elt, const seal::GaloisKeys &galois_keys) const
        {
            apply_galois_batch(encrypted, galois_elt, galois_keys);
        }
        void apply_galois_inplace(CiphertextBatch &encrypted, std::uint32_t galois_elt, const DeviceGaloisKeys &galois_keys) const
        {
            apply_galois_batch(encrypted, galois_elt, galois_keys);
        }
        void rotate_rows_inplace(CiphertextBatch &encrypted, int steps, const seal::GaloisKeys &galois_keys) const
        {
            rotate_rows_batch(encrypted, steps, galois_keys);
        }
        void rotate_rows_inplace(CiphertextBatch &encrypted, int steps, const DeviceGaloisKeys &galois_keys) const
        {
            rotate_rows_batch(encrypted, steps, galois_keys);
        }
        void rotate_vector_inplace(CiphertextBatch &encrypted, int steps, const seal::GaloisKeys &galois_keys) const
        {
            rotate_vector_batch(encrypted, steps, galois_keys);
        }
        void rotate_vector_inplace(CiphertextBatch &encrypted, int steps, const DeviceGaloisKeys &galois_keys) const
        {
            rotate_vector_batch(encrypted, steps, galois_keys);
        }
        void rotate_columns_inplace(CiphertextBatch &encrypted, const seal::GaloisKeys &galois_keys) const
        {
            rotate_columns_batch(encrypted, galois_keys);
        }
        void rotate_columns_inplace(CiphertextBatch &encrypted, const DeviceGaloisKeys &galois_keys) const
        {
            rotate_columns_batch(encrypted, galois_keys);
        }
        void complex_conjugate_inplace(CiphertextBatch &encrypted, const seal::GaloisKeys &galois_keys) const
        {
            complex_conjugate_batch(encrypted, galois_keys);
        }
        void complex_conjugate_inplace(CiphertextBatch &encrypted, const DeviceGaloisKeys &galois_keys) const
        {
            complex_conjugate_batch(encrypted, galois_keys);
        }
        // Sums of rotations.  apply_galois_add_inplace: destination += apply_galois(encrypted), the words of
        //     t = encrypted (a copy); apply_galois_inplace(t, galois_elt, galois_keys); add_inplace(destination, t);
        // with the addition in the key switch's last pass (sb200_apply_galois_add): no copy and no add pass.  destination may be
        // encrypted.  The chain's checks and messages run first, apply_galois_inplace's then add_inplace's; BGV operands with
        // different correction factors, or a destination of another size than 2, take the chain itself.
        void apply_galois_add_inplace(CiphertextBatch &destination, const CiphertextBatch &encrypted, std::uint32_t galois_elt,
                                      const seal::GaloisKeys &galois_keys) const
        {
            apply_galois_add_batch(destination, encrypted, galois_elt, galois_keys);
        }
        void apply_galois_add_inplace(CiphertextBatch &destination, const CiphertextBatch &encrypted, std::uint32_t galois_elt,
                                      const DeviceGaloisKeys &galois_keys) const
        {
            apply_galois_add_batch(destination, encrypted, galois_elt, galois_keys);
        }
        // rotate_sum_inplace: slot i becomes the sum over m < count of slot i + m step (cyclic within a row), the words of
        //     for (j = 0; (1 << j) < count; j++) { t = encrypted; rotate_X_inplace(t, step << j, galois_keys); add_inplace(encrypted, t); }
        // with rotate_X = rotate_vector (CKKS) or rotate_rows (BFV / BGV), in one sb200_rotate_sum call.  count is a power of two
        // (1 leaves the batch unchanged); step = 0 throws std::invalid_argument.  Scheme and batching errors, "step count too large"
        // and missing keys throw what the chain throws, before anything is written; when a step's key is absent but the reference's
        // NAF decomposition of it is covered by other keys, the chain itself runs.  No key of the call is evicted from the key cache
        // while it runs.
        // Every slot of a BFV batch (n slots, two rows of n / 2): rotate_sum_inplace(y, 1, n / 2, gk) sums each row, then
        // apply_galois_add_inplace(y, y, 2 n - 1, gk) adds the other row (element 2n - 1 swaps the rows, rotate_columns).
        void rotate_sum_inplace(CiphertextBatch &encrypted, int step, std::size_t count, const seal::GaloisKeys &galois_keys) const
        {
            rotate_sum_batch(encrypted, step, count, galois_keys);
        }
        void rotate_sum_inplace(CiphertextBatch &encrypted, int step, std::size_t count, const DeviceGaloisKeys &galois_keys) const
        {
            rotate_sum_batch(encrypted, step, count, galois_keys);
        }
        // Plaintext matrix times encrypted vector by diagonals.  apply_galois_multiply_plain_add_inplace: destination +=
        // plain * apply_galois(encrypted), the words and metadata of
        //     t = encrypted; apply_galois_inplace(t, galois_elt, galois_keys); multiply_plain_inplace(t, plain); add_inplace(destination, t);
        // CKKS / BGV with an NTT-form plaintext: one sb200_apply_galois_multiply_plain_add, the product and the addition in the key
        // switch's last pass.  destination may be encrypted.  The chain's checks and messages run first (apply_galois_inplace's,
        // multiply_plain_inplace's, then add_inplace's, "scale mismatch" included); a coefficient-form plaintext, BFV, BGV operands
        // whose correction factors need balancing, or a destination of another size than 2 take the chain itself.
        void apply_galois_multiply_plain_add_inplace(CiphertextBatch &destination, const CiphertextBatch &encrypted, std::uint32_t galois_elt,
                                                     const PlaintextBatch &plain, const seal::GaloisKeys &galois_keys) const
        {
            apply_galois_multiply_plain_add_batch(destination, encrypted, galois_elt, plain, galois_keys);
        }
        void apply_galois_multiply_plain_add_inplace(CiphertextBatch &destination, const CiphertextBatch &encrypted, std::uint32_t galois_elt,
                                                     const PlaintextBatch &plain, const DeviceGaloisKeys &galois_keys) const
        {
            apply_galois_multiply_plain_add_batch(destination, encrypted, galois_elt, plain, galois_keys);
        }
        // diagonal_sum: destination = sum_i diagonals[i] * rotate(encrypted, steps[i]), the words and metadata of
        //     for each i: t = encrypted; if (steps[i]) rotate_X_inplace(t, steps[i], galois_keys); multiply_plain_inplace(t, diagonals[i]);
        //                 i == 0 ? destination = t : add_inplace(destination, t)
        // with rotate_X = rotate_vector (CKKS) or rotate_rows (BFV / BGV); step 0 is no rotation, as in rotate_internal.  The
        // destination's scale is the first term's (CKKS: the ciphertext's times the diagonal's, and every term's must match it or
        // "scale mismatch" is thrown); BGV's correction factor is the ciphertext's.  One sb200_diagonal_sum call: every step-0 term in
        // one multiply_plain_sum pass, every other term one key switch with the product and the addition in its last pass (CKKS /
        // BGV); BFV runs the chain on the device through one key-switching chunk of temporary.  Every check of the chain, term by
        // term in its order, runs before anything is written.  The chain itself runs when a step's key exists only through SEAL's
        // NAF decomposition, when encrypted's size is not 2, when the diagonals mix NTT and coefficient form, or when BGV correction
        // factors would need balancing.  No key of the call is evicted from the key cache while it runs.  destination must not be
        // encrypted.
        // A small matrix M (d x d, d dividing the slot count) times a vector v replicated across the slots, CKKS:
        //     std::vector<int> steps(d); std::vector<PlaintextBatch> diags(d);
        //     for (int i = 0; i < d; i++) { steps[i] = i; diags[i] = encode(slot j -> M[j % d][(j + i) % d]); }
        //     evaluator.diagonal_sum(v, steps, diags, gk, y);     // slot j of y holds (M v)[j % d]
        // Larger matrices by baby-step giant-step compose from the existing calls: the baby-step rotations once, each giant step's
        // inner sum with multiply_plain_sum, and the giant-step rotations accumulated with apply_galois_add_inplace.
        void diagonal_sum(const CiphertextBatch &encrypted, const std::vector<int> &steps, const std::vector<PlaintextBatch> &diagonals,
                          const seal::GaloisKeys &galois_keys, CiphertextBatch &destination) const
        {
            diagonal_sum_batch(encrypted, steps, diagonals, galois_keys, destination);
        }
        void diagonal_sum(const CiphertextBatch &encrypted, const std::vector<int> &steps, const std::vector<PlaintextBatch> &diagonals,
                          const DeviceGaloisKeys &galois_keys, CiphertextBatch &destination) const
        {
            diagonal_sum_batch(encrypted, steps, diagonals, galois_keys, destination);
        }

    private:
        template <class GaloisKeys>
        void apply_galois_add_batch(CiphertextBatch &destination, const CiphertextBatch &encrypted, std::uint32_t galois_elt,
                                    const GaloisKeys &galois_keys) const
        {
            owned(encrypted);
            check_apply_galois(meta(encrypted), galois_elt, galois_keys);
            {
                std::lock_guard<std::mutex> lock(mu_);
                sb200_kswitch_key *key = key_for(galois_keys, seal::GaloisKeys::get_index(galois_elt), encrypted.L_);
                owned(destination);
                const Fold f = plan_fold({ meta(destination), meta(encrypted) }, SB200_FOLD_ADD); // add_inplace(destination, t)
                if (f.factors.empty() && destination.size_ == 2)
                {
                    const bool same = &destination == &encrypted; // out must not be the input: through the result slab
                    std::uint64_t *out = same ? out_slab(destination.batch_ * destination.words_per_ciphertext(), destination) : destination.d_;
                    check(sb200_apply_galois_add(ctx_, encrypted.L_, encrypted.batch_, encrypted.d_, galois_elt, key, destination.d_, out, nullptr));
                    if (same)
                        adopt(destination);
                    return;
                }
            }
            CiphertextBatch t;
            copy(encrypted, t);
            apply_galois_batch(t, galois_elt, galois_keys);
            add_inplace(destination, t);
        }
        template <class GaloisKeys>
        void rotate_sum_batch(CiphertextBatch &encrypted, int step, std::size_t count, const GaloisKeys &galois_keys) const
        {
            if (step == 0)
                throw std::invalid_argument("step must be nonzero");
            if (count == 0 || (count & (count - 1)))
                throw std::invalid_argument("count must be a power of two");
            if (count == 1)
                return;
            const bool ckks = scheme_ == seal::scheme_type::ckks;
            if (!ckks && scheme_ != seal::scheme_type::bfv && scheme_ != seal::scheme_type::bgv)
                throw std::logic_error("unsupported scheme");
            auto cd = batching_level(encrypted);
            if (galois_keys.parms_id() != context_.key_parms_id())
                throw std::invalid_argument("galois_keys is not valid for encryption parameters");
            std::vector<std::uint32_t> elts;
            bool naf = false;
            for (std::size_t j = 0; (std::size_t(1) << j) < count; j++)
            {
                const long long s = static_cast<long long>(step) * (1ll << j);
                if (s > std::numeric_limits<int>::max() || s < std::numeric_limits<int>::min())
                    throw std::invalid_argument("step count too large");
                const std::uint32_t elt = cd->galois_tool()->get_elt_from_step(static_cast<int>(s)); // "step count too large"
                if (!galois_keys.has_key(elt))
                {
                    if (seal::util::naf(static_cast<int>(s)).size() == 1)
                        throw std::invalid_argument("Galois key not present");
                    naf = true;
                }
                elts.push_back(elt);
            }
            if (naf)
            {
                for (std::size_t j = 0; j < elts.size(); j++)
                {
                    CiphertextBatch t;
                    copy(encrypted, t);
                    rotate_internal(t, static_cast<int>(static_cast<long long>(step) * (1ll << j)), galois_keys);
                    add_inplace(encrypted, t);
                }
                return;
            }
            check_apply_galois(meta(encrypted), elts[0], galois_keys);
            std::lock_guard<std::mutex> lock(mu_);
            std::vector<const sb200_kswitch_key *> keys;
            struct Unpin // the keys of this call stay in the cache until it returns
            {
                std::vector<const sb200_kswitch_key *> &pinned;
                ~Unpin() { pinned.clear(); }
            } unpin{ pinned_ };
            for (std::uint32_t elt : elts)
            {
                sb200_kswitch_key *k = key_for(galois_keys, seal::GaloisKeys::get_index(elt), encrypted.L_);
                pinned_.push_back(k);
                keys.push_back(k);
            }
            check(sb200_rotate_sum(ctx_, encrypted.L_, encrypted.batch_, encrypted.d_, elts.size(), elts.data(), keys.data(), encrypted.d_, nullptr));
        }
        template <class GaloisKeys>
        void apply_galois_multiply_plain_add_batch(CiphertextBatch &destination, const CiphertextBatch &encrypted, std::uint32_t galois_elt,
                                                   const PlaintextBatch &plain, const GaloisKeys &galois_keys) const
        {
            owned(encrypted);
            check_apply_galois(meta(encrypted), galois_elt, galois_keys);
            owned(plain);
            plain_count(encrypted, plain);
            const Meta t = multiply_plain_meta(meta(encrypted), meta(plain)); // apply_galois leaves the metadata alone
            {
                std::lock_guard<std::mutex> lock(mu_);
                sb200_kswitch_key *key = key_for(galois_keys, seal::GaloisKeys::get_index(galois_elt), encrypted.L_);
                owned(destination);
                const Fold f = plan_fold({ meta(destination), t }, SB200_FOLD_ADD); // add_inplace(destination, t)
                if (scheme_ != seal::scheme_type::bfv && plain.ntt_ && f.factors.empty() && destination.size_ == 2)
                {
                    const bool same = &destination == &encrypted; // out must not be the input: through the result slab
                    std::uint64_t *out = same ? out_slab(destination.batch_ * destination.words_per_ciphertext(), destination) : destination.d_;
                    check(sb200_apply_galois_multiply_plain_add(ctx_, encrypted.L_, encrypted.batch_, encrypted.d_, galois_elt, key, plain.batch_,
                                                                plain.d_, destination.d_, out, nullptr));
                    if (same)
                        adopt(destination);
                    return;
                }
            }
            CiphertextBatch tmp;
            copy(encrypted, tmp);
            apply_galois_batch(tmp, galois_elt, galois_keys);
            multiply_plain_inplace(tmp, plain);
            add_inplace(destination, tmp);
        }
        template <class GaloisKeys>
        void diagonal_sum_batch(const CiphertextBatch &encrypted, const std::vector<int> &steps, const std::vector<PlaintextBatch> &diagonals,
                                const GaloisKeys &galois_keys, CiphertextBatch &destination) const
        {
            if (steps.empty())
                throw std::invalid_argument("steps cannot be empty");
            if (diagonals.size() != steps.size())
                throw std::invalid_argument("diagonals must hold one plaintext batch per step");
            if (&destination == &encrypted)
                throw std::invalid_argument("encrypted must be different from destination");
            const bool ckks = scheme_ == seal::scheme_type::ckks;
            if (!ckks && scheme_ != seal::scheme_type::bfv && scheme_ != seal::scheme_type::bgv)
                throw std::logic_error("unsupported scheme");
            // the chain's checks, term by term: rotate_internal's, multiply_plain_inplace's, add_inplace's
            std::vector<std::uint32_t> elts;
            bool naf = false;
            Fold f;
            for (std::size_t i = 0; i < steps.size(); i++)
            {
                auto cd = batching_level(encrypted);
                if (galois_keys.parms_id() != context_.key_parms_id())
                    throw std::invalid_argument("galois_keys is not valid for encryption parameters");
                std::uint32_t elt = 1;
                if (steps[i] != 0)
                {
                    elt = cd->galois_tool()->get_elt_from_step(steps[i]); // "step count too large"
                    if (galois_keys.has_key(elt))
                        check_apply_galois(meta(encrypted), elt, galois_keys);
                    else if (seal::util::naf(steps[i]).size() == 1)
                        throw std::invalid_argument("Galois key not present");
                    else
                        naf = true;
                }
                elts.push_back(elt);
                owned(diagonals[i]);
                plain_count(encrypted, diagonals[i]);
                const Meta t = multiply_plain_meta(meta(encrypted), meta(diagonals[i]));
                if (i == 0)
                    f = Fold{ t, { t.size }, {}, {} };
                else
                    fold_in(f, t, SB200_FOLD_ADD);
            }
            bool mixed = false;
            for (auto &d : diagonals)
                mixed |= d.ntt_ != diagonals[0].ntt_;
            if (naf || mixed || encrypted.size_ != 2 || !f.factors.empty() || encrypted.ntt_ != (scheme_ != seal::scheme_type::bfv))
            {
                for (std::size_t i = 0; i < steps.size(); i++)
                {
                    CiphertextBatch t;
                    copy(encrypted, t);
                    rotate_internal(t, steps[i], galois_keys);
                    multiply_plain_inplace(t, diagonals[i]);
                    if (i == 0)
                        destination = std::move(t);
                    else
                        add_inplace(destination, t);
                }
                return;
            }
            std::lock_guard<std::mutex> lock(mu_);
            struct Unpin // the keys of this call stay in the cache until it returns
            {
                std::vector<const sb200_kswitch_key *> &pinned;
                ~Unpin() { pinned.clear(); }
            } unpin{ pinned_ };
            std::vector<const sb200_kswitch_key *> keys;
            std::vector<std::size_t> counts;
            std::vector<const std::uint64_t *> plains;
            for (std::size_t i = 0; i < steps.size(); i++)
            {
                sb200_kswitch_key *k = elts[i] == 1 ? nullptr : key_for(galois_keys, seal::GaloisKeys::get_index(elts[i]), encrypted.L_);
                if (k)
                    pinned_.push_back(k);
                keys.push_back(k);
                counts.push_back(diagonals[i].batch_);
                plains.push_back(diagonals[i].d_);
            }
            shape(destination, encrypted.batch_, 2, encrypted.L_, encrypted.n_);
            assign(destination, f.result);
            check(sb200_diagonal_sum(ctx_, encrypted.L_, encrypted.batch_, encrypted.d_, steps.size(), elts.data(), keys.data(), counts.data(),
                                     plains.data(), diagonals[0].ntt_ ? 1 : 0, destination.d_, nullptr));
        }
        template <class GaloisKeys>
        void apply_galois_batch(CiphertextBatch &encrypted, std::uint32_t galois_elt, const GaloisKeys &galois_keys) const
        {
            owned(encrypted);
            check_apply_galois(meta(encrypted), galois_elt, galois_keys);
            std::lock_guard<std::mutex> lock(mu_);
            sb200_kswitch_key *key = key_for(galois_keys, seal::GaloisKeys::get_index(galois_elt), encrypted.L_);
            std::uint64_t *out = out_slab(encrypted.batch_ * encrypted.words_per_ciphertext(), encrypted);
            check(sb200_apply_galois(ctx_, encrypted.L_, encrypted.batch_, encrypted.d_, galois_elt, key, out, nullptr));
            adopt(encrypted);
        }
        template <class GaloisKeys>
        void rotate_rows_batch(CiphertextBatch &encrypted, int steps, const GaloisKeys &galois_keys) const
        {
            if (scheme_ != seal::scheme_type::bfv && scheme_ != seal::scheme_type::bgv)
                throw std::logic_error("unsupported scheme");
            rotate_internal(encrypted, steps, galois_keys);
        }
        template <class GaloisKeys>
        void rotate_vector_batch(CiphertextBatch &encrypted, int steps, const GaloisKeys &galois_keys) const
        {
            if (scheme_ != seal::scheme_type::ckks)
                throw std::logic_error("unsupported scheme");
            rotate_internal(encrypted, steps, galois_keys);
        }
        template <class GaloisKeys>
        void rotate_columns_batch(CiphertextBatch &encrypted, const GaloisKeys &galois_keys) const
        {
            if (scheme_ != seal::scheme_type::bfv && scheme_ != seal::scheme_type::bgv)
                throw std::logic_error("unsupported scheme");
            conjugate_internal(encrypted, galois_keys);
        }
        template <class GaloisKeys>
        void complex_conjugate_batch(CiphertextBatch &encrypted, const GaloisKeys &galois_keys) const
        {
            if (scheme_ != seal::scheme_type::ckks)
                throw std::logic_error("unsupported scheme");
            conjugate_internal(encrypted, galois_keys);
        }

    public:
        // transform_to_ntt_inplace / transform_from_ntt_inplace (evaluator.cpp:2289-2382)
        void transform_to_ntt_inplace(CiphertextBatch &encrypted) const
        {
            owned(encrypted);
            if (encrypted.ntt_)
                throw std::invalid_argument("encrypted is already in NTT form");
            std::lock_guard<std::mutex> lock(mu_);
            check(sb200_ntt_forward(ctx_, encrypted.L_, encrypted.size_, encrypted.batch_, encrypted.d_, nullptr));
            encrypted.ntt_ = true;
        }
        void transform_from_ntt_inplace(CiphertextBatch &encrypted_ntt) const
        {
            owned(encrypted_ntt);
            if (!encrypted_ntt.ntt_)
                throw std::invalid_argument("encrypted_ntt is not in NTT form");
            std::lock_guard<std::mutex> lock(mu_);
            check(sb200_ntt_inverse(ctx_, encrypted_ntt.L_, encrypted_ntt.size_, encrypted_ntt.batch_, encrypted_ntt.d_, nullptr));
            encrypted_ntt.ntt_ = false;
        }
        // ---- device-resident plaintexts (PlaintextBatch): the same checks, exception types and metadata updates as the
        // seal::Plaintext overloads above, all made before anything is written; between upload and download only the stream
        // entry points run.  A PlaintextBatch of size 1 is applied to every ciphertext of the batch (read once per call).
        void upload(const std::vector<seal::Plaintext> &plains, PlaintextBatch &destination) const
        {
            upload(plains.data(), plains.size(), destination);
        }
        void upload(const seal::Plaintext *first, std::size_t count, PlaintextBatch &destination) const
        {
            if (!first || !count)
                throw std::invalid_argument("batch cannot be empty");
            const seal::Plaintext &f = first[0];
            for (std::size_t i = 0; i < count; i++)
            {
                const seal::Plaintext &p = first[i];
                if (!seal::is_metadata_valid_for(p, context_) || !seal::is_buffer_valid(p))
                    throw std::invalid_argument("plain is not valid for encryption parameters");
                const double s1 = p.scale(), s2 = f.scale();
                if (p.parms_id() != f.parms_id() || std::memcmp(&s1, &s2, sizeof(double)) != 0)
                    throw std::invalid_argument("batch members must share parms_id, NTT form and scale");
            }
            const bool ntt = f.is_ntt_form();
            const std::size_t n = context_.first_context_data()->parms().poly_modulus_degree();
            const std::size_t L = ntt ? context_.get_context_data(f.parms_id())->parms().coeff_modulus().size() : 1, words = L * n;
            std::vector<std::uint64_t> flat(count * words, 0); // coefficient form: zero above coeff_count
            for (std::size_t i = 0; i < count; i++)
                std::copy_n(first[i].data(), std::min(first[i].coeff_count(), words), flat.data() + i * words);
            std::lock_guard<std::mutex> lock(mu_);
            check(destination.reserve(ctx_, flat.size()));
            check(sb200_memcpy_h2d(ctx_, destination.d_, flat.data(), flat.size() * sizeof(std::uint64_t), nullptr));
            destination.batch_ = count, destination.L_ = L, destination.n_ = n;
            destination.parms_id_ = f.parms_id(), destination.ntt_ = ntt, destination.scale_ = f.scale();
        }
        void download(const PlaintextBatch &source, std::vector<seal::Plaintext> &plains) const
        {
            owned(source);
            const std::size_t words = source.words_per_plaintext();
            std::vector<std::uint64_t> flat(source.batch_ * words);
            check(sb200_memcpy_d2h(ctx_, flat.data(), source.d_, flat.size() * sizeof(std::uint64_t), nullptr));
            check(sb200_stream_synchronize(ctx_, nullptr));
            plains.resize(source.batch_);
            for (std::size_t i = 0; i < source.batch_; i++)
            {
                plains[i].parms_id() = seal::parms_id_zero;
                plains[i].resize(words);
                std::copy_n(flat.data() + i * words, words, plains[i].data());
                plains[i].parms_id() = source.parms_id_;
                plains[i].scale() = source.scale_;
            }
        }
        // transform_to_ntt_inplace(Plaintext&, parms_id) (evaluator.cpp:2196-2287)
        void transform_to_ntt_inplace(PlaintextBatch &plain, seal::parms_id_type parms_id) const
        {
            owned(plain);
            auto cd = context_.get_context_data(parms_id);
            if (!cd)
                throw std::invalid_argument("parms_id is not valid for the current context");
            if (plain.ntt_)
                throw std::invalid_argument("plain is already in NTT form");
            const std::size_t L = cd->parms().coeff_modulus().size();
            std::lock_guard<std::mutex> lock(mu_);
            PlaintextBatch out;
            check(out.reserve(ctx_, plain.batch_ * L * plain.n_));
            check(sb200_plain_to_ntt(ctx_, L, plain.batch_, plain.d_, out.d_, nullptr));
            std::swap(plain.d_, out.d_), std::swap(plain.cap_, out.cap_);
            plain.L_ = L, plain.ntt_ = true, plain.parms_id_ = parms_id;
        }
        // mod_switch_to_next_inplace / mod_switch_to_inplace(Plaintext&) (evaluator.cpp:1369-1402, :1475-1501): NTT-form plaintexts
        // lose their last prime -- a 2-D copy of the first L - 1 rows of every plaintext
        void mod_switch_to_next_inplace(PlaintextBatch &plain) const
        {
            owned(plain);
            auto &next = plain_next_level(meta(plain));
            const std::size_t L = plain.L_, n = plain.n_, row = (L - 1) * n * sizeof(std::uint64_t);
            std::lock_guard<std::mutex> lock(mu_);
            PlaintextBatch out;
            check(out.reserve(ctx_, plain.batch_ * (L - 1) * n));
            check(sb200_memcpy_d2d_2d(ctx_, out.d_, row, plain.d_, L * n * sizeof(std::uint64_t), row, plain.batch_, nullptr));
            std::swap(plain.d_, out.d_), std::swap(plain.cap_, out.cap_);
            plain.L_ = L - 1, plain.parms_id_ = next.parms_id();
        }
        void mod_switch_to_inplace(PlaintextBatch &plain, seal::parms_id_type parms_id) const
        {
            owned(plain);
            check_plain_target_level(meta(plain), parms_id);
            while (plain.parms_id_ != parms_id)
                mod_switch_to_next_inplace(plain);
        }
        // multiply_plain_inplace (evaluator.cpp:1975-2019): the four-way dispatch on the NTT forms
        void multiply_plain_inplace(CiphertextBatch &encrypted, const PlaintextBatch &plain) const
        {
            owned(encrypted), owned(plain);
            plain_count(encrypted, plain);
            const Meta r = multiply_plain_meta(meta(encrypted), meta(plain));
            const std::size_t L = encrypted.L_, size = encrypted.size_, B = encrypted.batch_;
            if (!plain.ntt_)
            {
                // multiply_plain_normal (:2021-2155) / transform + multiply_plain_ntt (:1999-2004)
                std::lock_guard<std::mutex> lock(mu_);
                check(sb200_multiply_plain_coeff_n(ctx_, L, size, B, plain.batch_, encrypted.ntt_ ? 1 : 0, encrypted.d_, plain.d_, encrypted.d_,
                                                   nullptr));
                return;
            }
            const bool back = !encrypted.ntt_; // :2006-2011: to NTT form, multiply, back
            std::lock_guard<std::mutex> lock(mu_);
            if (back)
                check(sb200_ntt_forward(ctx_, L, size, B, encrypted.d_, nullptr));
            check(sb200_multiply_plain_n(ctx_, L, size, B, plain.batch_, encrypted.d_, plain.d_, encrypted.d_, nullptr));
            if (back)
                check(sb200_ntt_inverse(ctx_, L, size, B, encrypted.d_, nullptr));
            encrypted.scale_ = r.scale;
        }
        // add_plain_inplace / sub_plain_inplace (evaluator.cpp:1759-1866, :1867-1974)
        void add_plain_inplace(CiphertextBatch &encrypted, const PlaintextBatch &plain) const { plain_linear_batch(encrypted, plain, false); }
        void sub_plain_inplace(CiphertextBatch &encrypted, const PlaintextBatch &plain) const { plain_linear_batch(encrypted, plain, true); }

        // waits for all device work queued by this Evaluator (the batch members above only enqueue)
        void synchronize() const { check(sb200_stream_synchronize(ctx_, nullptr)); }

        // ---- key cache control: uploaded key-switching keys are cached by CONTENT (a fingerprint of the key words), never by
        // address; least recently used entries are evicted above the byte budget ----
        void set_key_cache_limit(std::size_t bytes) const
        {
            std::lock_guard<std::mutex> lock(mu_);
            key_cache_limit_ = bytes;
            evict(nullptr);
        }
        void clear_key_cache() const
        {
            std::lock_guard<std::mutex> lock(mu_);
            for (auto &kv : keys_)
                sb200_kswitch_key_destroy(kv.second.handle);
            keys_.clear();
            key_cache_bytes_ = 0;
        }
        std::size_t key_cache_entries() const
        {
            std::lock_guard<std::mutex> lock(mu_);
            return keys_.size();
        }

        sb200_context *native_handle() const noexcept { return ctx_; }

    private:
        // evaluator.cpp:154-262 / 264-350
        void linear(seal::Ciphertext &encrypted1, const seal::Ciphertext &encrypted2, bool subtract) const
        {
            validate(encrypted1, "encrypted1 is not valid for encryption parameters");
            validate(encrypted2, "encrypted2 is not valid for encryption parameters");
            const Fold f = plan_fold({ meta(encrypted1), meta(encrypted2) }, subtract ? SB200_FOLD_SUB : SB200_FOLD_ADD);
            auto cd = context_.get_context_data(encrypted1.parms_id());
            const std::size_t L = encrypted1.coeff_modulus_size(), n = encrypted1.poly_modulus_degree();
            if (!f.factors.empty())
            {
                // BGV: bring both operands to a common correction factor first
                seal::Ciphertext copy = encrypted2;
                scale_by(encrypted1, f.factors[0], *cd);
                scale_by(copy, f.factors[1], *cd);
                encrypted1.correction_factor() = f.result.cf;
                copy.correction_factor() = f.result.cf;
                linear(encrypted1, copy, subtract);
                return;
            }
            const std::size_t s1 = encrypted1.size(), s2 = encrypted2.size(), lo = std::min(s1, s2);
            encrypted1.resize(context_, cd->parms_id(), std::max(s1, s2));
            check(subtract ? sb200_sub_host(ctx_, L, lo, 1, encrypted1.data(), encrypted2.data(), encrypted1.data())
                           : sb200_add_host(ctx_, L, lo, 1, encrypted1.data(), encrypted2.data(), encrypted1.data()));
            if (s1 < s2)
            {
                // the longer operand's tail is copied (add, :228-233) or negated (sub, :336-341)
                if (subtract)
                    check(sb200_negate_host(ctx_, L, s2 - lo, 1, encrypted2.data(lo), encrypted1.data(lo)));
                else
                    std::memcpy(encrypted1.data(lo), encrypted2.data(lo), (s2 - lo) * L * n * sizeof(std::uint64_t));
            }
            throw_if_transparent(encrypted1);
        }
        // every polynomial times the scalar e (multiply_poly_scalar_coeffmod, evaluator.cpp:192-200): a dyadic product with the
        // constant vector e mod q_i, valid in either form
        void scale_by(seal::Ciphertext &ct, std::uint64_t e, const seal::SEALContext::ContextData &cd) const
        {
            const std::size_t L = ct.coeff_modulus_size(), n = ct.poly_modulus_degree();
            std::vector<std::uint64_t> v(L * n);
            for (std::size_t i = 0; i < L; i++)
                std::fill(v.begin() + i * n, v.begin() + (i + 1) * n, seal::util::barrett_reduce_64(e, cd.parms().coeff_modulus()[i]));
            check(sb200_multiply_plain_host(ctx_, L, ct.size(), 1, ct.data(), v.data(), ct.data()));
        }
        // (f, e1, e2) with e1*factor1 = e2*factor2 = f mod t, both e invertible mod t, and |e1| + |e2| (balanced
        // representatives) minimal over the remainder sequence of (t, factor2/factor1) -- evaluator.cpp:50-118
        static void balance_factors(std::uint64_t factor1, std::uint64_t factor2, const seal::Modulus &plain, std::uint64_t &f,
                                    std::uint64_t &e1, std::uint64_t &e2)
        {
            using namespace seal::util;
            const std::uint64_t t = plain.value();
            auto weight = [t](std::uint64_t x, std::uint64_t y) {
                auto mag = [t](std::uint64_t v) { return static_cast<std::int64_t>(v > t / 2 ? t - v : v); };
                return mag(x) + mag(y);
            };
            auto residue = [&plain](std::int64_t v) {
                std::uint64_t r = barrett_reduce_64(static_cast<std::uint64_t>(v < 0 ? -v : v), plain);
                return v < 0 ? negate_uint_mod(r, plain) : r;
            };
            std::uint64_t ratio = 1;
            if (!try_invert_uint_mod(factor1, plain, ratio))
                throw std::logic_error("invalid correction factor1");
            ratio = multiply_uint_mod(ratio, factor2, plain);
            e1 = ratio, e2 = 1;
            std::int64_t best = weight(e1, e2);
            std::int64_t r0 = static_cast<std::int64_t>(t), r1 = static_cast<std::int64_t>(ratio), c0 = 0, c1 = 1;
            while (r1 != 0)
            {
                const std::int64_t quo = r0 / r1, r2 = r0 % r1, c2 = sub_safe(c0, mul_safe(c1, quo));
                r0 = r1, r1 = r2, c0 = c1, c1 = c2;
                const std::uint64_t a = residue(r1), b = residue(c1);
                if (a != 0 && gcd(a, t) == 1)
                {
                    const std::int64_t w = weight(a, b);
                    if (w < best)
                        best = w, e1 = a, e2 = b;
                }
            }
            f = multiply_uint_mod(e1, factor1, plain);
        }
        // a coefficient-form plaintext as n words (Plaintext::coeff_count() may be smaller; the rest is zero)
        std::vector<std::uint64_t> padded(const seal::Plaintext &plain) const
        {
            const std::size_t n = context_.key_context_data()->parms().poly_modulus_degree();
            std::vector<std::uint64_t> w(n, 0);
            std::copy(plain.data(), plain.data() + std::min(n, plain.coeff_count()), w.begin());
            return w;
        }
        // mod_switch_drop_to_next (evaluator.cpp:1296-1366): every polynomial keeps its first L-1 components
        void drop_last_component(seal::Ciphertext &encrypted) const
        {
            const Meta r = mod_switch_to_next_meta(meta(encrypted), true);
            const std::size_t L = encrypted.coeff_modulus_size(), n = encrypted.poly_modulus_degree(), size = encrypted.size();
            std::vector<std::uint64_t> kept(size * (L - 1) * n);
            for (std::size_t p = 0; p < size; p++)
                std::memcpy(kept.data() + p * (L - 1) * n, encrypted.data(p), (L - 1) * n * sizeof(std::uint64_t));
            encrypted.resize(context_, r.parms_id, size);
            std::memcpy(encrypted.data(), kept.data(), kept.size() * sizeof(std::uint64_t));
            encrypted.is_ntt_form() = r.ntt, encrypted.scale() = r.scale, encrypted.correction_factor() = r.cf;
        }
        // the checks of mod_switch_to_inplace / rescale_to_inplace (evaluator.cpp:1451-1473, :1543-1590) and
        // mod_reduce_to_inplace (:1625-1647) before their single steps; pool is the seal::Ciphertext members' pool
        void check_target_level(const seal::parms_id_type &current, const seal::parms_id_type &parms_id, bool rescale = false,
                                const seal::MemoryPoolHandle *pool = nullptr) const
        {
            auto cur = context_.get_context_data(current);
            auto target = context_.get_context_data(parms_id);
            if (!cur)
                throw std::invalid_argument("encrypted is not valid for encryption parameters");
            if (!target)
                throw std::invalid_argument("parms_id is not valid for encryption parameters");
            if (cur->chain_index() < target->chain_index())
                throw std::invalid_argument("cannot switch to higher level modulus");
            check_pool(pool);
            if (rescale && scheme_ != seal::scheme_type::ckks)
                throw std::invalid_argument("unsupported operation for scheme type");
        }
        void plain_linear(seal::Ciphertext &encrypted, const seal::Plaintext &plain, bool subtract) const
        {
            validate(encrypted, "encrypted is not valid for encryption parameters");
            if (!seal::is_metadata_valid_for(plain, context_) || !seal::is_buffer_valid(plain))
                throw std::invalid_argument("plain is not valid for encryption parameters");
            check_add_plain(meta(encrypted), meta(plain));
            if (scheme_ != seal::scheme_type::ckks)
            {
                // BFV: scaling variant on c_0 (util/scalingvariant.cpp:70-160); BGV: correction factor, lift, NTT (:1838-1849)
                const bool bfv = scheme_ == seal::scheme_type::bfv;
                const std::vector<std::uint64_t> words = padded(plain);
                const std::uint64_t cf = encrypted.correction_factor();
                check(sb200_add_plain_coeff_host(ctx_, encrypted.coeff_modulus_size(), encrypted.size(), 1, subtract ? 1 : 0, encrypted.data(),
                                                 words.data(), bfv ? nullptr : &cf, encrypted.data()));
                throw_if_transparent(encrypted);
                return;
            }
            const std::size_t L = encrypted.coeff_modulus_size();
            // c_0 +/- plain: a one-polynomial slab (add_poly_coeffmod / sub_poly_coeffmod on encrypted[0], :1831-1836)
            check(subtract ? sb200_sub_host(ctx_, L, 1, 1, encrypted.data(), plain.data(), encrypted.data())
                           : sb200_add_host(ctx_, L, 1, 1, encrypted.data(), plain.data(), encrypted.data()));
            throw_if_transparent(encrypted);
        }
        static void check(int status)
        {
            if (status == SB200_OK)
                return;
            const std::string msg = sb200_last_error();
            switch (status)
            {
            case SB200_E_INVALID_ARG:
            case SB200_E_POINTER: throw std::invalid_argument(msg);
            case SB200_E_LOGIC: throw std::logic_error(msg);
            case SB200_E_OUT_OF_RANGE: throw std::out_of_range(msg);
            case SB200_E_NOMEM: throw std::bad_alloc();
            default: throw std::runtime_error(msg);
            }
        }
        void validate(const seal::Ciphertext &ct, const char *msg) const
        {
            if (!seal::is_metadata_valid_for(ct, context_) || !seal::is_buffer_valid(ct))
                throw std::invalid_argument(msg);
        }
        static void throw_if_transparent(const seal::Ciphertext &ct)
        {
#ifdef SEAL_THROW_ON_TRANSPARENT_CIPHERTEXT
            if (ct.is_transparent())
                throw std::logic_error("result ciphertext is transparent");
#else
            (void)ct;
#endif
        }
        // evaluator.cpp:29-48
        static bool scale_within_bounds(double scale, const seal::SEALContext::ContextData &cd) noexcept
        {
            int bound = cd.parms().scheme() == seal::scheme_type::ckks ? cd.total_coeff_modulus_bit_count()
                                                                        : cd.parms().plain_modulus().bit_count();
            return !(!std::isnormal(scale) || scale <= 0 || (static_cast<int>(std::log2(scale)) >= bound));
        }

        // ---- the reference's preconditions, one function per rule, shared by the seal::Ciphertext and CiphertextBatch members ----
        // Each runs its checks in the reference's order on the operands' metadata, after the member's own operand checks (validate()
        // and the pool for a seal::Ciphertext, owned() and the batch counts for a batch), and returns the result's metadata where the
        // operation changes it.  pool is the seal::Ciphertext members' pool, checked where they check it; batches pass none.
        struct Meta
        {
            seal::parms_id_type parms_id = seal::parms_id_zero;
            std::size_t size = 0;
            bool ntt = false;
            double scale = 1.0;
            std::uint64_t cf = 1;  // correction factor
            std::size_t batch = 1; // 1 for a seal::Ciphertext
        };
        static Meta meta(const seal::Ciphertext &c)
        {
            return { c.parms_id(), c.size(), c.is_ntt_form(), c.scale(), c.correction_factor(), 1 };
        }
        static Meta meta(const CiphertextBatch &b) { return { b.parms_id_, b.size_, b.ntt_, b.scale_, b.cf_, b.batch_ }; }
        static Meta meta(const seal::Plaintext &p) { return { p.parms_id(), 0, p.is_ntt_form(), p.scale() }; }
        static Meta meta(const PlaintextBatch &p) { return { p.parms_id_, 0, p.ntt_, p.scale_, 1, p.batch_ }; }
        static void assign(CiphertextBatch &b, const Meta &m)
        {
            b.parms_id_ = m.parms_id, b.size_ = m.size, b.ntt_ = m.ntt, b.scale_ = m.scale, b.cf_ = m.cf;
        }
        static void check_pool(const seal::MemoryPoolHandle *pool)
        {
            if (pool && !*pool)
                throw std::invalid_argument("pool is uninitialized");
        }
        // the per-scheme form of an operand (mod_switch_scale_to_next, evaluator.cpp:1205-1217; mod_switch_drop_to_next :1300-1312;
        // add_plain_inplace :1774-1808; switch_key_inplace :2601-2611)
        void check_ntt_form(bool ntt) const
        {
            if (scheme_ == seal::scheme_type::bfv && ntt)
                throw std::invalid_argument("BFV encrypted cannot be in NTT form");
            if (scheme_ == seal::scheme_type::ckks && !ntt)
                throw std::invalid_argument("CKKS encrypted must be in NTT form");
            if (scheme_ == seal::scheme_type::bgv && !ntt)
                throw std::invalid_argument("BGV encrypted must be in NTT form");
        }
        // multiply_inplace (evaluator.cpp:352-393; bfv_multiply :397-400, ckks_multiply :571-574, :703-707 with the resize's size
        // check first, bgv_multiply :712-715, :838-840)
        Meta multiply_meta(const Meta &a, const Meta &b, const seal::MemoryPoolHandle *pool = nullptr) const
        {
            if (a.parms_id != b.parms_id || a.batch != b.batch)
                throw std::invalid_argument("encrypted1 and encrypted2 parameter mismatch");
            check_pool(pool);
            const bool bfv = scheme_ == seal::scheme_type::bfv;
            if (bfv && (a.ntt || b.ntt))
                throw std::invalid_argument("encrypted1 or encrypted2 cannot be in NTT form");
            if (!bfv && !(a.ntt && b.ntt))
                throw std::invalid_argument("encrypted1 or encrypted2 must be in NTT form");
            Meta r = a;
            r.size = a.size + b.size - 1;
            if (r.size > SEAL_CIPHERTEXT_SIZE_MAX)
                throw std::invalid_argument("invalid size");
            auto &cd = *context_.get_context_data(a.parms_id);
            if (scheme_ == seal::scheme_type::ckks)
            {
                r.scale = a.scale * b.scale;
                if (!scale_within_bounds(r.scale, cd))
                    throw std::invalid_argument("scale out of bounds");
            }
            if (scheme_ == seal::scheme_type::bgv)
                r.cf = seal::util::multiply_uint_mod(a.cf, b.cf, cd.parms().plain_modulus());
            return r;
        }
        // multiply_plain_inplace (evaluator.cpp:1975-2019): a coefficient-form plaintext (never CKKS) leaves the metadata alone;
        // multiply_plain_ntt (:2157-2195) checks the level and the product's scale
        Meta multiply_plain_meta(const Meta &encrypted, const Meta &plain) const
        {
            if (!plain.ntt)
            {
                if (scheme_ == seal::scheme_type::ckks)
                    throw std::invalid_argument("plain is not valid for encryption parameters"); // CKKS plaintexts are always in NTT form
                return encrypted;
            }
            if (encrypted.parms_id != plain.parms_id)
                throw std::invalid_argument("encrypted_ntt and plain_ntt parameter mismatch"); // :2164-2167
            Meta r = encrypted;
            r.scale = encrypted.scale * plain.scale;
            if (!scale_within_bounds(r.scale, *context_.get_context_data(encrypted.parms_id)))
                throw std::invalid_argument("scale out of bounds"); // :2189-2193
            return r;
        }
        // add_plain_inplace / sub_plain_inplace (evaluator.cpp:1759-1866, :1867-1974)
        void check_add_plain(const Meta &encrypted, const Meta &plain) const
        {
            check_ntt_form(encrypted.ntt);
            if (scheme_ == seal::scheme_type::bfv && plain.ntt)
                throw std::invalid_argument("BFV plain cannot be in NTT form");
            if (scheme_ == seal::scheme_type::bgv && plain.ntt)
                throw std::invalid_argument("BGV plain cannot be in NTT form");
            if (scheme_ != seal::scheme_type::ckks)
                return;
            if (!plain.ntt)
                throw std::invalid_argument("CKKS plain must be in NTT form");
            if (encrypted.parms_id != plain.parms_id)
                throw std::invalid_argument("encrypted and plain parameter mismatch");
            if (!seal::util::are_close<double>(encrypted.scale, plain.scale))
                throw std::invalid_argument("scale mismatch");
        }
        // relinearize_internal down to size 2 (evaluator.cpp:1144-1168): the key level, the size and the number of keys
        template <class RelinKeys>
        void check_relinearize(const RelinKeys &relin_keys, std::size_t size) const
        {
            if (relin_keys.parms_id() != context_.key_parms_id())
                throw std::invalid_argument("relin_keys is not valid for encryption parameters");
            if (size < 2)
                throw std::invalid_argument("destination_size must be at least 2 and less than or equal to current count");
            if (relin_keys.size() < size - 2)
                throw std::invalid_argument("not enough relinearization keys");
        }
        // the parts of switch_key_inplace's prologue that concern the operand (evaluator.cpp:2573-2611)
        void check_switch_key(bool ntt, const seal::MemoryPoolHandle *pool = nullptr) const
        {
            if (!context_.using_keyswitching())
                throw std::logic_error("keyswitching is not supported by the context");
            check_pool(pool);
            check_ntt_form(ntt);
        }
        // apply_galois_inplace (evaluator.cpp:2384-2430), up to the key lookup
        template <class GaloisKeys>
        void check_apply_galois(const Meta &encrypted, std::uint32_t galois_elt, const GaloisKeys &galois_keys,
                                const seal::MemoryPoolHandle *pool = nullptr) const
        {
            if (galois_keys.parms_id() != context_.key_parms_id())
                throw std::invalid_argument("galois_keys is not valid for encryption parameters");
            if (!galois_keys.has_key(galois_elt))
                throw std::invalid_argument("Galois key not present");
            if (!(galois_elt & 1) || galois_elt >= 2 * context_.get_context_data(encrypted.parms_id)->parms().poly_modulus_degree())
                throw std::invalid_argument("Galois element is not valid");
            if (encrypted.size != 2)
                throw std::invalid_argument("encrypted size must be 2");
            check_switch_key(encrypted.ntt, pool);
        }
        // the first checks of rotate_internal / conjugate_internal (evaluator.cpp:2507-2515, evaluator.h:1358-1369): the operand's
        // level, which must support batching
        template <class Encrypted>
        std::shared_ptr<const seal::SEALContext::ContextData> batching_level(const Encrypted &encrypted) const
        {
            if constexpr (std::is_same_v<Encrypted, CiphertextBatch>)
                owned(encrypted);
            auto cd = context_.get_context_data(meta(encrypted).parms_id);
            if (!cd)
                throw std::invalid_argument("encrypted is not valid for encryption parameters");
            if (!cd->qualifiers().using_batching)
                throw std::logic_error("encryption parameters do not support batching");
            return cd;
        }
        // the entry of mod_switch_to_next / rescale_to_next (evaluator.cpp:1404-1440, :1503-1532) and mod_reduce_to_next (:1597-1623)
        void check_mod_switch_to_next(const Meta &encrypted, bool rescale, const seal::MemoryPoolHandle *pool = nullptr) const
        {
            if (context_.last_parms_id() == encrypted.parms_id)
                throw std::invalid_argument("end of modulus switching chain reached");
            check_pool(pool);
            if (rescale && scheme_ != seal::scheme_type::ckks)
                throw std::invalid_argument("unsupported operation for scheme type");
        }
        // one level down: mod_switch_drop_to_next (evaluator.cpp:1296-1322) when drop, else mod_switch_scale_to_next (:1201-1294),
        // which rescales CKKS and updates BGV's correction factor
        Meta mod_switch_to_next_meta(const Meta &encrypted, bool drop) const
        {
            auto cd = context_.get_context_data(encrypted.parms_id);
            auto &next = *cd->next_context_data();
            check_ntt_form(encrypted.ntt);
            Meta r = encrypted;
            r.parms_id = next.parms_id();
            if (drop)
            {
                if (!scale_within_bounds(encrypted.scale, next))
                    throw std::invalid_argument("scale out of bounds");
                return r;
            }
            if (scheme_ == seal::scheme_type::ckks)
            {
                if (!scale_within_bounds(encrypted.scale, *cd))
                    throw std::invalid_argument("scale out of bounds");
                r.scale = encrypted.scale / static_cast<double>(cd->parms().coeff_modulus().back().value());
                if (!scale_within_bounds(r.scale, next))
                    throw std::invalid_argument("scale out of bounds");
            }
            if (scheme_ == seal::scheme_type::bgv)
                r.cf = seal::util::multiply_uint_mod(encrypted.cf, cd->rns_tool()->inv_q_last_mod_t(), next.parms().plain_modulus());
            return r;
        }
        // mod_switch_drop_to_next(Plaintext &) (evaluator.cpp:1369-1392): the level below an NTT-form plaintext's
        const seal::SEALContext::ContextData &plain_next_level(const Meta &plain) const
        {
            if (!plain.ntt)
                throw std::invalid_argument("plain is not in NTT form");
            auto cd = context_.get_context_data(plain.parms_id);
            if (!cd->next_context_data())
                throw std::invalid_argument("end of modulus switching chain reached");
            auto &next = *cd->next_context_data();
            if (!scale_within_bounds(plain.scale, next))
                throw std::invalid_argument("scale out of bounds");
            return next;
        }
        // mod_switch_to_inplace(Plaintext &, parms_id) (evaluator.cpp:1475-1501) after the plaintext's own check
        void check_plain_target_level(const Meta &plain, const seal::parms_id_type &parms_id) const
        {
            auto target = context_.get_context_data(parms_id);
            if (!target)
                throw std::invalid_argument("parms_id is not valid for encryption parameters");
            if (!plain.ntt)
                throw std::invalid_argument("plain is not in NTT form");
            if (context_.get_context_data(plain.parms_id)->chain_index() < target->chain_index())
                throw std::invalid_argument("cannot switch to higher level modulus");
        }
        // the arguments of one sb200_add_many call folding operands 0, 1, ... in order (the caller supplies their device words), each
        // step one add_inplace / sub_inplace of the reference's chain, with its checks and its correction factors (fold_in)
        struct Fold
        {
            Meta result;                        // the chain's result so far
            std::vector<std::size_t> sizes;     // every operand's
            std::vector<int> modes;             // [count - 1]
            std::vector<std::uint64_t> factors; // [count - 1][2], empty when no step is scaled
        };
        // add_inplace / sub_inplace (evaluator.cpp:155-350) of b into the fold; BGV operands with different correction factors are
        // both scaled by the balancing factors first (:188-209, :305-326)
        void fold_in(Fold &f, const Meta &b, int mode) const
        {
            const Meta &a = f.result;
            if (a.parms_id != b.parms_id || a.batch != b.batch)
                throw std::invalid_argument("encrypted1 and encrypted2 parameter mismatch");
            if (a.ntt != b.ntt)
                throw std::invalid_argument("NTT form mismatch");
            if (!seal::util::are_close<double>(a.scale, b.scale))
                throw std::invalid_argument("scale mismatch");
            std::uint64_t e1 = 0, e2 = 0;
            const bool scaled = a.cf != b.cf;
            if (scaled)
            {
                balance_factors(a.cf, b.cf, context_.get_context_data(a.parms_id)->parms().plain_modulus(), f.result.cf, e1, e2);
                mode |= SB200_FOLD_SCALED;
                f.factors.resize(2 * f.modes.size(), 0); // the earlier steps' (unscaled) entries
            }
            if (scaled || !f.factors.empty())
                f.factors.push_back(e1), f.factors.push_back(e2);
            f.modes.push_back(mode);
            f.sizes.push_back(b.size);
            f.result.size = std::max(f.result.size, b.size);
        }
        Fold plan_fold(const std::vector<Meta> &ops, int mode) const
        {
            Fold f{ ops[0], { ops[0].size }, {}, {} };
            for (std::size_t j = 1; j < ops.size(); j++)
                fold_in(f, ops[j], mode);
            return f;
        }
        // uploads KSwitchKeys::data()[index] (evaluator.cpp:2586-2648) and caches the device copy under a fingerprint of the
        // key's CONTENT (leading / trailing / strided words of every digit + its shape): a regenerated or reloaded key object
        // that happens to reuse a freed pool address can never be served another key's device copy.  Caller holds mu_.
        struct KeyEntry
        {
            sb200_kswitch_key *handle = nullptr;
            std::size_t bytes = 0;
            std::uint64_t last_use = 0;
        };
        static std::uint64_t fingerprint(const std::vector<seal::PublicKey> &kv, std::size_t row_words, std::size_t index)
        {
            std::uint64_t h = 0x9E3779B97F4A7C15ull ^ (row_words * 0xD6E8FEB86659FD93ull) ^ (kv.size() << 48) ^ (index << 32);
            auto mix = [&h](std::uint64_t v) {
                h ^= v + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
                h *= 0xFF51AFD7ED558CCDull;
                h ^= h >> 33;
            };
            const std::size_t edge = std::min<std::size_t>(64, row_words), stride = std::max<std::size_t>(1, row_words / 96) | 1;
            for (auto &pk : kv)
            {
                const std::uint64_t *p = pk.data().data();
                for (std::size_t i = 0; i < edge; i++)
                    mix(p[i]), mix(p[row_words - 1 - i]);
                for (std::size_t i = 0; i < row_words; i += stride)
                    mix(p[i]);
            }
            return h;
        }
        void evict(const sb200_kswitch_key *keep) const
        {
            while (key_cache_bytes_ > key_cache_limit_ && keys_.size() > (keep ? 1u : 0u))
            {
                auto victim = keys_.end();
                for (auto it = keys_.begin(); it != keys_.end(); ++it)
                    if (it->second.handle != keep && std::find(pinned_.begin(), pinned_.end(), it->second.handle) == pinned_.end() &&
                        (victim == keys_.end() || it->second.last_use < victim->second.last_use))
                        victim = it;
                if (victim == keys_.end())
                    break;
                sb200_kswitch_key_destroy(victim->second.handle);
                key_cache_bytes_ -= victim->second.bytes;
                keys_.erase(victim);
            }
        }
        sb200_kswitch_key *key_for(const seal::KSwitchKeys &keys, std::size_t index, std::size_t L) const
        {
            if (keys.parms_id() != context_.key_parms_id())
                throw std::invalid_argument("parameter mismatch");
            if (index >= keys.data().size())
                throw std::out_of_range("kswitch_keys_index");
            auto &kv = keys.data(index); // throws on an empty slot, like the reference's checked accessor
            if (kv.size() < L)
                throw std::invalid_argument("kswitch_keys inner dimension is too small");
            for (auto &each : kv)
                if (!seal::is_metadata_valid_for(each, context_) || !seal::is_buffer_valid(each))
                    throw std::invalid_argument("kswitch_keys is not valid for encryption parameters");
            const std::size_t K = context_.key_context_data()->parms().coeff_modulus().size();
            const std::size_t n = context_.key_context_data()->parms().poly_modulus_degree(), row = 2 * K * n;
            const std::uint64_t id = fingerprint(kv, row, index);
            auto it = keys_.find(id);
            if (it != keys_.end())
            {
                it->second.last_use = ++key_clock_;
                return it->second.handle;
            }
            std::vector<std::uint64_t> flat(kv.size() * row);
            for (std::size_t j = 0; j < kv.size(); j++)
                std::memcpy(flat.data() + j * row, kv[j].data().data(), row * sizeof(std::uint64_t));
            sb200_kswitch_key *h = nullptr;
            check(sb200_kswitch_key_create(ctx_, flat.data(), kv.size(), &h));
            KeyEntry e;
            e.handle = h, e.bytes = flat.size() * sizeof(std::uint64_t), e.last_use = ++key_clock_;
            keys_[id] = e;
            key_cache_bytes_ += e.bytes;
            evict(h);
            return h;
        }
        // a device key set's handle, with the checks of the overload above (its keys always have k - 1 >= L digits)
        sb200_kswitch_key *key_for(const DeviceKSwitchKeys &keys, std::size_t index, std::size_t) const
        {
            if (keys.parms_id_ != context_.key_parms_id())
                throw std::invalid_argument("parameter mismatch");
            if (keys.ctx_ != ctx_)
                throw std::invalid_argument("keys are not on this evaluator's device context");
            if (index >= keys.keys_.size())
                throw std::out_of_range("kswitch_keys_index");
            if (!keys.keys_[index])
                throw std::invalid_argument("keyswitching key does not exist");
            return keys.keys_[index];
        }
        // ---- helpers of the stream and key-set members ----
        static constexpr std::size_t kSealHeader = sizeof(seal::Serialization::SEALHeader);
        // Ciphertext::save_size from the uncompressed size: header + ComprSizeEstimate(members)
        static std::streamoff save_size_of(std::size_t plain, seal::compr_mode_type compr_mode)
        {
            return static_cast<std::streamoff>(kSealHeader + seal::Serialization::ComprSizeEstimate(plain - kSealHeader, compr_mode));
        }
        void load_batch(const seal::seal_byte *const *streams, const std::size_t *sizes, std::size_t count, bool validate,
                        CiphertextBatch &destination) const
        {
            if (!streams || !sizes || !count)
                throw std::invalid_argument("batch cannot be empty");
            std::vector<const std::uint8_t *> in(count);
            sb200_ct_info f{};
            for (std::size_t i = 0; i < count; i++)
            {
                if (!streams[i])
                    throw std::invalid_argument("in cannot be null");
                in[i] = reinterpret_cast<const std::uint8_t *>(streams[i]);
                sb200_ct_info info{};
                check(sb200_ciphertext_inspect(in[i], sizes[i], &info));
                if (i == 0)
                    f = info;
                else if (std::memcmp(info.parms_id, f.parms_id, sizeof(f.parms_id)) != 0 || info.size != f.size ||
                         info.is_ntt_form != f.is_ntt_form || info.correction_factor != f.correction_factor ||
                         std::memcmp(&info.scale, &f.scale, sizeof(double)) != 0)
                    throw std::invalid_argument("batch members must share parms_id, size, NTT form, scale and correction factor");
            }
            seal::parms_id_type pid;
            std::memcpy(pid.data(), f.parms_id, sizeof(f.parms_id));
            auto cd = context_.get_context_data(pid);
            if (!cd || cd->parms().coeff_modulus().size() != f.coeff_modulus_size) // is_metadata_valid_for (ciphertext.cpp:299-302)
                throw std::logic_error("ciphertext data is invalid");
            CiphertextBatch loaded;
            std::lock_guard<std::mutex> lock(mu_);
            shape(loaded, count, f.size, f.coeff_modulus_size, f.poly_modulus_degree);
            check(sb200_ciphertext_load(ctx_, count, in.data(), sizes, f.coeff_modulus_size, f.size, validate ? 1 : 0, loaded.d_, nullptr, nullptr));
            loaded.parms_id_ = pid, loaded.ntt_ = f.is_ntt_form != 0, loaded.scale_ = f.scale, loaded.cf_ = f.correction_factor;
            destination = std::move(loaded);
        }
        // slots == nullptr: every non-empty slot; min_slots = the slot count the set reports at least (GaloisKeys: n)
        void load_keys(const seal::seal_byte *in, std::size_t size, const std::vector<std::size_t> *slots, std::size_t min_slots,
                       DeviceKSwitchKeys &destination) const
        {
            if (!in)
                throw std::invalid_argument("in cannot be null");
            const std::size_t cap = slots ? slots->size() : std::max<std::size_t>(context_.key_context_data()->parms().poly_modulus_degree(), 64);
            const std::size_t none = 0;
            std::vector<sb200_kswitch_key *> out(std::max<std::size_t>(cap, 1), nullptr);
            std::vector<std::size_t> got(out.size());
            std::size_t made = 0;
            check(sb200_kswitch_keys_load(ctx_, reinterpret_cast<const std::uint8_t *>(in), size, slots ? (slots->empty() ? &none : slots->data()) : nullptr,
                                          cap, out.data(), got.data(), &made));
            adopt_keys(out.data(), got.data(), made, min_slots, destination);
        }
        // takes ownership of `count` handles for the slots `slots` (destroyed if this throws)
        void adopt_keys(sb200_kswitch_key **handles, const std::size_t *slots, std::size_t count, std::size_t min_slots,
                        DeviceKSwitchKeys &destination) const
        {
            try
            {
                std::size_t n_slots = min_slots;
                for (std::size_t i = 0; i < count; i++)
                    n_slots = std::max(n_slots, slots[i] + 1);
                std::vector<sb200_kswitch_key *> by_slot(n_slots, nullptr);
                for (std::size_t i = 0; i < count; i++)
                    by_slot[slots[i]] = handles[i];
                destination.assign(ctx_, context_.key_parms_id(), std::move(by_slot));
            }
            catch (...)
            {
                for (std::size_t i = 0; i < count; i++)
                    sb200_kswitch_key_destroy(handles[i]);
                throw;
            }
        }
        void upload_keys(const seal::KSwitchKeys &keys, DeviceKSwitchKeys &destination) const
        {
            if (keys.parms_id() != context_.key_parms_id())
                throw std::invalid_argument("keys is not valid for encryption parameters");
            const std::size_t K = context_.key_context_data()->parms().coeff_modulus().size();
            const std::size_t n = context_.key_context_data()->parms().poly_modulus_degree(), row = 2 * K * n;
            for (auto &kv : keys.data()) // is_valid_for(KSwitchKeys) (valcheck.cpp:292-323): k - 1 valid public keys per non-empty slot
            {
                if (!kv.empty() && kv.size() != K - 1)
                    throw std::invalid_argument("keys is not valid for encryption parameters");
                for (auto &each : kv)
                    if (!seal::is_metadata_valid_for(each, context_) || !seal::is_buffer_valid(each))
                        throw std::invalid_argument("keys is not valid for encryption parameters");
            }
            std::vector<sb200_kswitch_key *> handles;
            std::vector<std::size_t> slots;
            handles.reserve(keys.data().size()), slots.reserve(keys.data().size());
            try
            {
                std::vector<std::uint64_t> flat;
                for (std::size_t i = 0; i < keys.data().size(); i++)
                {
                    auto &kv = keys.data()[i];
                    if (kv.empty())
                        continue;
                    flat.resize(kv.size() * row);
                    for (std::size_t j = 0; j < kv.size(); j++)
                        std::memcpy(flat.data() + j * row, kv[j].data().data(), row * sizeof(std::uint64_t));
                    sb200_kswitch_key *h = nullptr;
                    check(sb200_kswitch_key_create(ctx_, flat.data(), kv.size(), &h));
                    handles.push_back(h);
                    slots.push_back(i);
                }
            }
            catch (...)
            {
                for (sb200_kswitch_key *h : handles)
                    sb200_kswitch_key_destroy(h);
                throw;
            }
            adopt_keys(handles.data(), slots.data(), handles.size(), keys.data().size(), destination);
        }
        // ---- helpers of the CiphertextBatch members ----
        // data of already validated ciphertexts of one shape -> one device slab; metadata of the first member
        void upload_rows(const seal::Ciphertext *cts, std::size_t count, CiphertextBatch &destination) const
        {
            const seal::Ciphertext &f = cts[0];
            {
                std::lock_guard<std::mutex> lock(mu_);
                shape(destination, count, f.size(), f.coeff_modulus_size(), f.poly_modulus_degree());
            }
            destination.parms_id_ = f.parms_id(), destination.ntt_ = f.is_ntt_form(), destination.scale_ = f.scale();
            destination.cf_ = f.correction_factor();
            // the transfer itself runs outside the lock (its own staging lane and stream in the library): uploads of one batch
            // overlap the operations another thread enqueues on other batches
            std::vector<const std::uint64_t *> rows(count);
            for (std::size_t i = 0; i < count; i++)
                rows[i] = cts[i].data();
            check(sb200_upload_rows(ctx_, destination.d_, rows.data(), destination.words_per_ciphertext() * sizeof(std::uint64_t), count));
        }
        void owned(const PlaintextBatch &p) const
        {
            if (p.ctx_ != ctx_ || !p.d_ || !p.batch_ || (p.ntt_ && !context_.get_context_data(p.parms_id_)))
                throw std::invalid_argument("plain is not valid for encryption parameters");
        }
        static void plain_count(const CiphertextBatch &encrypted, const PlaintextBatch &plain)
        {
            if (plain.batch_ != 1 && plain.batch_ != encrypted.batch_)
                throw std::invalid_argument("plain batch size must be 1 or the ciphertext batch size");
        }
        void plain_linear_batch(CiphertextBatch &encrypted, const PlaintextBatch &plain, bool subtract) const
        {
            owned(encrypted), owned(plain);
            plain_count(encrypted, plain);
            check_add_plain(meta(encrypted), meta(plain));
            const std::size_t L = encrypted.L_, size = encrypted.size_, B = encrypted.batch_;
            if (scheme_ != seal::scheme_type::ckks)
            {
                const bool bfv = scheme_ == seal::scheme_type::bfv;
                // the batch's one correction factor, once per plaintext (BGV, :1840-1843)
                const std::vector<std::uint64_t> cf(plain.batch_, encrypted.cf_);
                std::lock_guard<std::mutex> lock(mu_);
                check(sb200_add_plain_coeff_n(ctx_, L, size, B, plain.batch_, subtract ? 1 : 0, encrypted.d_, plain.d_, bfv ? nullptr : cf.data(),
                                              encrypted.d_, nullptr));
                return;
            }
            std::lock_guard<std::mutex> lock(mu_);
            check(sb200_add_plain_ntt(ctx_, L, size, B, plain.batch_, subtract ? 1 : 0, encrypted.d_, plain.d_, encrypted.d_, nullptr));
        }
        void owned(const CiphertextBatch &b) const
        {
            if (b.ctx_ != ctx_ || !b.d_ || !b.batch_)
                throw std::invalid_argument("encrypted is not valid for encryption parameters");
            if (!context_.get_context_data(b.parms_id_))
                throw std::invalid_argument("encrypted is not valid for encryption parameters");
        }
        void reserve(CiphertextBatch &b, std::size_t words) const
        {
            if (b.ctx_ != ctx_)
            {
                b.release();
                b.ctx_ = ctx_;
            }
            if (b.cap_ < words)
            {
                b.release();
                check(sb200_device_malloc(ctx_, words * sizeof(std::uint64_t), &b.d_));
                b.cap_ = words;
            }
        }
        void shape(CiphertextBatch &b, std::size_t batch, std::size_t size, std::size_t L, std::size_t n) const
        {
            reserve(b, batch * size * L * n);
            b.batch_ = batch, b.size_ = size, b.L_ = L, b.n_ = n;
        }
        // result slab of a layout-changing operation; adopt() swaps it with the operand's storage, so a chain of operations
        // allocates nothing once the largest shape has been seen.  Caller holds mu_.
        // (never smaller than the slab it will be swapped with: every buffer in circulation then fits every level of a chain,
        // and a later upload into the same batch object finds room without reallocating)
        std::uint64_t *out_slab(std::size_t words, const CiphertextBatch &operand) const
        {
            reserve(tmp_, std::max(words, operand.cap_));
            return tmp_.d_;
        }
        void adopt(CiphertextBatch &b) const
        {
            std::swap(b.d_, tmp_.d_);
            std::swap(b.cap_, tmp_.cap_);
        }
        void mod_switch_batch(CiphertextBatch &e, bool rescale) const
        {
            const Meta r = mod_switch_to_next_meta(meta(e), scheme_ == seal::scheme_type::ckks && !rescale);
            std::lock_guard<std::mutex> lock(mu_);
            std::uint64_t *out = out_slab(e.batch_ * e.size_ * (e.L_ - 1) * e.n_, e);
            check(rescale ? sb200_rescale_to_next_sized(ctx_, e.L_, e.size_, e.batch_, e.d_, out, nullptr)
                          : sb200_mod_switch_to_next_sized(ctx_, e.L_, e.size_, e.batch_, e.d_, out, nullptr));
            adopt(e);
            e.L_ -= 1;
            assign(e, r);
        }
        // ---- multiply_plain_sum: the chain's checks replayed on the products' metadata, before anything is written ----
        struct PlainSum
        {
            Fold fold;                  // the add_many of every output (the factors depend on the ciphertexts only)
            std::vector<double> scales; // [M] the result's scale: the first product's
        };
        PlainSum plan_plain_sum(const std::vector<CiphertextBatch> &encrypteds, const std::vector<PlaintextBatch> &plains, std::size_t M) const
        {
            const std::size_t K = encrypteds.size();
            PlainSum p;
            for (std::size_t j = 0; j < M; j++)
            {
                std::vector<Meta> prods; // the products t_i
                for (std::size_t i = 0; i < K; i++)
                {
                    // multiply_plain_inplace (evaluator.cpp:1975-2019), as the batch member above checks it
                    owned(encrypteds[i]), owned(plains[j * K + i]);
                    plain_count(encrypteds[i], plains[j * K + i]);
                    prods.push_back(multiply_plain_meta(meta(encrypteds[i]), meta(plains[j * K + i])));
                }
                p.fold = plan_fold(prods, SB200_FOLD_ADD); // add_many (evaluator.cpp:236-262)
                p.scales.push_back(prods[0].scale);
            }
            for (auto &pl : plains)
                if (pl.ntt_ != plains[0].ntt_)
                    throw std::invalid_argument("plains must all be in NTT form or all in coefficient form");
            return p;
        }
        // destination j shaped and given the chain's metadata; caller holds mu_
        std::uint64_t *plain_sum_output(const CiphertextBatch &e0, const PlainSum &p, std::size_t j, CiphertextBatch &d) const
        {
            shape(d, e0.batch_, p.fold.result.size, e0.L_, e0.n_);
            assign(d, p.fold.result);
            d.scale_ = p.scales[j];
            return d.d_;
        }
        void run_plain_sum(const std::vector<CiphertextBatch> &encrypteds, const std::vector<PlaintextBatch> &plains, const PlainSum &p,
                           std::uint64_t *const *outs) const
        {
            const CiphertextBatch &e0 = encrypteds[0];
            std::vector<std::size_t> counts;
            std::vector<const std::uint64_t *> cts, ptrs;
            for (auto &e : encrypteds)
                cts.push_back(e.d_);
            for (auto &pl : plains)
                counts.push_back(pl.batch_), ptrs.push_back(pl.d_);
            check(sb200_multiply_plain_sum(ctx_, e0.L_, e0.batch_, encrypteds.size(), p.scales.size(), p.fold.sizes.data(), cts.data(),
                                           counts.data(), ptrs.data(), e0.ntt_ ? 1 : 0, plains[0].ntt_ ? 1 : 0, p.fold.modes.data(),
                                           p.fold.factors.empty() ? nullptr : p.fold.factors.data(), outs, nullptr));
        }
        // ---- multiply_sum: the chain's checks replayed on the products' metadata, before anything is written ----
        struct MultiplySum
        {
            std::vector<Fold> folds; // [M] the add_many of every output (BGV's factors depend on both operands)
            bool fused = true;       // every operand has size 2: sb200_multiply_sum
        };
        void check_sum_destination(const std::vector<CiphertextBatch> &e1, const std::vector<CiphertextBatch> &e2, const CiphertextBatch &d) const
        {
            if (e2.empty())
                throw std::invalid_argument("encrypteds cannot be empty");
            for (auto *v : { &e1, &e2 })
                for (auto &e : *v)
                    if (&e == &d)
                        throw std::invalid_argument("encrypteds must be different from destination");
        }
        static std::size_t sum_outputs(const std::vector<CiphertextBatch> &e1, const std::vector<CiphertextBatch> &e2,
                                       const std::vector<CiphertextBatch> &d)
        {
            if (e2.empty())
                throw std::invalid_argument("encrypteds cannot be empty");
            if (&d == &e1 || &d == &e2)
                throw std::invalid_argument("encrypteds must be different from destination");
            if (e1.empty() || e1.size() % e2.size() != 0)
                throw std::invalid_argument("encrypteds1 must hold K ciphertext batches per destination");
            return e1.size() / e2.size();
        }
        MultiplySum plan_multiply_sum(const std::vector<CiphertextBatch> &e1, const std::vector<CiphertextBatch> &e2, std::size_t M) const
        {
            const std::size_t K = e2.size();
            MultiplySum p;
            for (std::size_t j = 0; j < M; j++)
            {
                std::vector<Meta> prods; // the products t_i
                for (std::size_t i = 0; i < K; i++)
                {
                    const CiphertextBatch &a = e1[j * K + i], &b = e2[i];
                    // multiply_inplace (evaluator.cpp:352-393), as the batch member above checks it
                    owned(a), owned(b);
                    prods.push_back(multiply_meta(meta(a), meta(b)));
                    p.fused = p.fused && a.size_ == 2 && b.size_ == 2;
                }
                p.folds.push_back(plan_fold(prods, SB200_FOLD_ADD)); // add_many (evaluator.cpp:236-262)
            }
            return p;
        }
        void run_multiply_sum(const std::vector<CiphertextBatch> &e1, const std::vector<CiphertextBatch> &e2, const MultiplySum &p,
                              CiphertextBatch *const *dest) const
        {
            const std::size_t K = e2.size(), M = p.folds.size();
            if (!p.fused) // other sizes: the chain itself
            {
                for (std::size_t j = 0; j < M; j++)
                {
                    std::vector<CiphertextBatch> terms(K);
                    for (std::size_t i = 0; i < K; i++)
                    {
                        copy(e1[j * K + i], terms[i]);
                        multiply_inplace(terms[i], e2[i]);
                    }
                    add_many(terms, *dest[j]);
                }
                return;
            }
            const CiphertextBatch &b0 = e2[0];
            std::lock_guard<std::mutex> lock(mu_);
            for (std::size_t j = 0; j < M; j++)
            {
                CiphertextBatch &d = *dest[j];
                shape(d, b0.batch_, 3, b0.L_, b0.n_);
                assign(d, p.folds[j].result);
            }
            std::vector<const std::uint64_t *> lhs, rhs;
            std::vector<std::uint64_t *> outs;
            for (auto &e : e1)
                lhs.push_back(e.d_);
            for (auto &e : e2)
                rhs.push_back(e.d_);
            for (std::size_t j = 0; j < M; j++)
                outs.push_back(dest[j]->d_);
            // one call for every output when the outputs share the fold's steps (always, but for BGV with differing correction factors)
            bool same = true;
            for (auto &f : p.folds)
                same = same && f.modes == p.folds[0].modes && f.factors == p.folds[0].factors;
            for (std::size_t j0 = 0, m = same ? M : 1; j0 < M; j0 += m)
            {
                const Fold &f = p.folds[j0];
                check(sb200_multiply_sum(ctx_, b0.L_, b0.batch_, K, m, lhs.data() + j0 * K, rhs.data(), f.modes.empty() ? nullptr : f.modes.data(),
                                         f.factors.empty() ? nullptr : f.factors.data(), outs.data() + j0, nullptr));
            }
        }
        template <class RelinKeys>
        void multiply_relinearize_sum_one(const std::vector<CiphertextBatch> &e1, const std::vector<CiphertextBatch> &e2, const RelinKeys &relin_keys,
                                          CiphertextBatch &destination) const
        {
            check_sum_destination(e1, e2, destination);
            if (e1.size() != e2.size())
                throw std::invalid_argument("encrypteds1 must hold K ciphertext batches per destination");
            const MultiplySum p = plan_multiply_sum(e1, e2, 1);
            check_relinearize(relin_keys, p.folds[0].result.size);
            if (p.folds[0].result.size > 2)
                check_switch_key(p.folds[0].result.ntt);
            CiphertextBatch *d = &destination;
            run_multiply_sum(e1, e2, p, &d);
            relinearize_inplace(destination, relin_keys);
        }
        template <class RelinKeys>
        void multiply_relinearize_sum_many(const std::vector<CiphertextBatch> &e1, const std::vector<CiphertextBatch> &e2, const RelinKeys &relin_keys,
                                           std::vector<CiphertextBatch> &destinations) const
        {
            const std::size_t M = sum_outputs(e1, e2, destinations);
            const MultiplySum p = plan_multiply_sum(e1, e2, M);
            for (const Fold &f : p.folds) // relinearize_inplace's checks of every sum
            {
                check_relinearize(relin_keys, f.result.size);
                if (f.result.size > 2)
                    check_switch_key(f.result.ntt);
            }
            destinations.resize(M);
            std::vector<CiphertextBatch *> d;
            for (auto &x : destinations)
                d.push_back(&x);
            run_multiply_sum(e1, e2, p, d.data());
            for (auto &x : destinations)
                relinearize_inplace(x, relin_keys);
        }
        void linear_batch(CiphertextBatch &a, const CiphertextBatch &b, bool subtract) const
        {
            owned(a), owned(b);
            const Fold f = plan_fold({ meta(a), meta(b) }, subtract ? SB200_FOLD_SUB : SB200_FOLD_ADD);
            const std::uint64_t *ptrs[2] = { a.d_, b.d_ };
            std::lock_guard<std::mutex> lock(mu_);
            // in place when the result keeps a's size and b is another slab; otherwise into the result slab
            const bool in_place = a.size_ == f.result.size && a.d_ != b.d_;
            std::uint64_t *out = in_place ? a.d_ : out_slab(a.batch_ * f.result.size * a.L_ * a.n_, a);
            check(sb200_add_many(ctx_, a.L_, a.batch_, 2, f.sizes.data(), ptrs, f.modes.data(), f.factors.empty() ? nullptr : f.factors.data(),
                                 out, nullptr));
            if (!in_place)
                adopt(a);
            assign(a, f.result);
        }
        // ---- the product schedule of multiply_many / exponentiate ----
        // The reference's queue (evaluator.cpp:1649-1724): products of operand pairs (0,1), (2,3), ... with an odd operand appended
        // at the end, then pairs taken from the front with each product appended at the back, until one is left.  It is replayed on
        // ids: leaves are 0 .. leaves-1, product p is id leaves + p.  The queue holds runs (id, count) of equal ids, so e copies of
        // one operand cost O(log e) steps; a product is hash-consed on (left id, right id) and made once, and products are grouped
        // into waves by their depth (a wave's products depend only on earlier waves).
        struct ProductSchedule
        {
            std::size_t leaves = 0, root = 0;
            std::vector<std::pair<std::size_t, std::size_t>> products; // (left id, right id)
            std::vector<std::vector<std::size_t>> waves;               // product indices
        };
        static ProductSchedule schedule_products(std::size_t leaves, const std::vector<std::pair<std::size_t, std::uint64_t>> &operand_runs)
        {
            ProductSchedule s;
            s.leaves = leaves;
            std::map<std::pair<std::size_t, std::size_t>, std::size_t> made;
            std::vector<std::size_t> depth(leaves, 0);
            auto product = [&](std::size_t l, std::size_t r) {
                auto it = made.find({ l, r });
                if (it != made.end())
                    return it->second;
                const std::size_t id = leaves + s.products.size(), d = std::max(depth[l], depth[r]) + 1;
                s.products.emplace_back(l, r);
                depth.push_back(d);
                if (s.waves.size() < d)
                    s.waves.resize(d);
                s.waves[d - 1].push_back(id - leaves);
                return made[{ l, r }] = id;
            };
            std::deque<std::pair<std::size_t, std::uint64_t>> q;
            auto push = [&q](std::size_t id, std::uint64_t count) {
                if (!q.empty() && q.back().first == id)
                    q.back().second += count;
                else
                    q.emplace_back(id, count);
            };
            // first level: consecutive operand pairs, the odd operand last
            bool pending = false;
            std::size_t odd = 0;
            for (auto [id, count] : operand_runs)
            {
                if (pending && count)
                    push(product(odd, id), 1), count--, pending = false;
                if (count / 2)
                    push(product(id, id), count / 2);
                if (count & 1)
                    pending = true, odd = id;
            }
            if (pending)
                push(odd, 1);
            // then pairs from the front of the queue, products to the back
            while (q.size() > 1 || q.front().second > 1)
            {
                auto [id, count] = q.front();
                q.pop_front();
                if (count / 2)
                    push(product(id, id), count / 2);
                if (count & 1)
                {
                    const std::size_t other = q.front().first;
                    if (--q.front().second == 0)
                        q.pop_front();
                    push(product(id, other), 1);
                }
            }
            s.root = q.front().first;
            return s;
        }
        // runs a schedule over the leaf batches; the result goes to destination with the reference's metadata
        template <class RelinKeys>
        void run_products(const std::vector<const CiphertextBatch *> &leaves, const ProductSchedule &s, const RelinKeys &relin_keys,
                          CiphertextBatch &destination) const
        {
            const CiphertextBatch &f = *leaves[0];
            for (auto *l : leaves)
                owned(*l);
            if (s.products.empty())
            {
                copy(*leaves[s.root], destination);
                return;
            }
            // every check of every product's multiply_inplace and relinearize_inplace, in the chain's order, before the first write
            const std::size_t P = s.products.size();
            std::vector<Meta> prods(P); // each product's metadata, relinearized
            auto id_meta = [&](std::size_t id) { return id < s.leaves ? meta(*leaves[id]) : prods[id - s.leaves]; };
            for (std::size_t p = 0; p < P; p++)
            {
                prods[p] = multiply_meta(id_meta(s.products[p].first), id_meta(s.products[p].second));
                check_relinearize(relin_keys, prods[p].size);
                check_switch_key(prods[p].ntt);
                prods[p].size = 2;
            }
            const std::size_t B = f.batch_, L = f.L_, ct = 2 * L * f.n_, bytes = B * ct * sizeof(std::uint64_t);
            std::vector<const std::uint64_t *> data(P);     // device words of each product, [B][2][L][n]
            std::vector<CiphertextBatch> slabs;              // owners of the wave outputs
            auto id_data = [&](std::size_t id) { return id < s.leaves ? leaves[id]->d_ : data[id - s.leaves]; };
            auto id_size = [&](std::size_t id) { return id < s.leaves ? leaves[id]->size_ : std::size_t(2); };
            for (const auto &wave : s.waves)
            {
                std::vector<std::size_t> fused, single; // size-2 pairs run together; other sizes one by one
                for (std::size_t p : wave)
                    (id_size(s.products[p].first) == 2 && id_size(s.products[p].second) == 2 ? fused : single).push_back(p);
                for (std::size_t p : single)
                {
                    CiphertextBatch x, y;
                    const CiphertextBatch *l = s.products[p].first < s.leaves ? leaves[s.products[p].first] : nullptr;
                    const CiphertextBatch *r = s.products[p].second < s.leaves ? leaves[s.products[p].second] : nullptr;
                    wrap(x, l, id_data(s.products[p].first), f);
                    wrap(y, r, id_data(s.products[p].second), f);
                    multiply_inplace(x, y);
                    relinearize_inplace(x, relin_keys);
                    data[p] = x.d_;
                    slabs.push_back(std::move(x));
                }
                std::lock_guard<std::mutex> lock(mu_);
                const std::size_t chunk = sb200_keyswitch_chunk(ctx_, L, fused.size() * B, 1);
                const std::size_t group = std::max<std::size_t>(1, chunk / B);
                for (std::size_t g0 = 0; g0 < fused.size(); g0 += group)
                {
                    const std::size_t G = std::min(group, fused.size() - g0);
                    CiphertextBatch a, b;
                    shape(a, G * B, 2, L, f.n_);
                    shape(b, G * B, 2, L, f.n_);
                    for (std::size_t i = 0; i < G; i++)
                    {
                        const auto &pr = s.products[fused[g0 + i]];
                        check(sb200_memcpy_d2d(ctx_, a.d_ + i * B * ct, id_data(pr.first), bytes, nullptr));
                        check(sb200_memcpy_d2d(ctx_, b.d_ + i * B * ct, id_data(pr.second), bytes, nullptr));
                    }
                    sb200_kswitch_key *key = key_for(relin_keys, seal::RelinKeys::get_index(2), L);
                    check(sb200_multiply_relinearize(ctx_, L, G * B, a.d_, b.d_, key, a.d_, nullptr));
                    for (std::size_t i = 0; i < G; i++)
                        data[fused[g0 + i]] = a.d_ + i * B * ct;
                    slabs.push_back(std::move(a));
                }
            }
            const std::size_t r = s.root - s.leaves;
            {
                std::lock_guard<std::mutex> lock(mu_);
                shape(destination, B, 2, L, f.n_);
                assign(destination, prods[r]);
                check(sb200_memcpy_d2d(ctx_, destination.d_, data[r], bytes, nullptr));
            }
        }
        // a batch object over a leaf (a copy) or over product words (size 2), with the leaves' metadata, for the one-by-one products
        void wrap(CiphertextBatch &x, const CiphertextBatch *leaf, const std::uint64_t *words, const CiphertextBatch &like) const
        {
            if (leaf)
            {
                copy(*leaf, x);
                return;
            }
            std::lock_guard<std::mutex> lock(mu_);
            assign(x, meta(like));
            shape(x, like.batch_, 2, like.L_, like.n_);
            check(sb200_memcpy_d2d(ctx_, x.d_, words, like.batch_ * 2 * like.L_ * like.n_ * sizeof(std::uint64_t), nullptr));
        }
        void mod_switch_impl(const seal::Ciphertext &encrypted, seal::Ciphertext &destination, bool rescale) const
        {
            const Meta r = mod_switch_to_next_meta(meta(encrypted), scheme_ == seal::scheme_type::ckks && !rescale);
            const std::size_t L = encrypted.coeff_modulus_size(), n = encrypted.poly_modulus_degree(), size = encrypted.size();
            std::vector<std::uint64_t> in(encrypted.data(), encrypted.data() + size * L * n);
            destination.resize(context_, r.parms_id, size);
            check(rescale ? sb200_rescale_to_next_sized_host(ctx_, L, size, 1, in.data(), destination.data())
                          : sb200_mod_switch_to_next_sized_host(ctx_, L, size, 1, in.data(), destination.data()));
            destination.is_ntt_form() = r.ntt;
            destination.scale() = r.scale;
            if (scheme_ == seal::scheme_type::bgv) // :1288-1293
                destination.correction_factor() = r.cf;
            throw_if_transparent(destination);
        }
        // rotate_internal (evaluator.cpp:2504-2559) of a seal::Ciphertext (pool: its pool) or a batch (no pool)
        template <class Encrypted, class GaloisKeys, class... Pool>
        void rotate_internal(Encrypted &encrypted, int steps, const GaloisKeys &galois_keys, const Pool &...pool) const
        {
            auto cd = batching_level(encrypted);
            if (galois_keys.parms_id() != context_.key_parms_id())
                throw std::invalid_argument("galois_keys is not valid for encryption parameters");
            if (steps == 0)
                return;
            const std::size_t n = cd->parms().poly_modulus_degree();
            const std::uint32_t elt = cd->galois_tool()->get_elt_from_step(steps);
            if (galois_keys.has_key(elt))
            {
                apply_galois_inplace(encrypted, elt, galois_keys, pool...);
                return;
            }
            std::vector<int> naf_steps = seal::util::naf(steps);
            if (naf_steps.size() == 1)
                throw std::invalid_argument("Galois key not present");
            for (int s : naf_steps)
                if (static_cast<std::size_t>(std::abs(s)) != (n >> 1))
                    rotate_internal(encrypted, s, galois_keys, pool...);
        }
        // conjugate_internal (evaluator.h:1354-1377)
        template <class Encrypted, class GaloisKeys, class... Pool>
        void conjugate_internal(Encrypted &encrypted, const GaloisKeys &galois_keys, const Pool &...pool) const
        {
            apply_galois_inplace(encrypted, batching_level(encrypted)->galois_tool()->get_elt_from_step(0), galois_keys, pool...);
        }

        seal::SEALContext context_;
        seal::scheme_type scheme_;
        sb200_context *ctx_ = nullptr;
        mutable std::mutex mu_;
        mutable std::map<std::uint64_t, KeyEntry> keys_;
        mutable std::vector<const sb200_kswitch_key *> pinned_; // keys of a running call that evict() must keep (rotate_sum_inplace)
        mutable std::size_t key_cache_bytes_ = 0, key_cache_limit_ = std::size_t(24) << 30;
        mutable std::uint64_t key_clock_ = 0;
        mutable CiphertextBatch tmp_; // result slab of layout-changing batch operations
    };
} // namespace seal_b200
