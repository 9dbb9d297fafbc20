// seal_b200/csrc/sb_engine.cuh -- device context + operation drivers (declarations).
#pragma once
#include "sb_host.hpp"
#include "sb_mem.cuh"
#include "sb_ntt.cuh"
#include "sb_ksint.cuh"
#include "sb_wire.hpp"
#include <array>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

namespace sb
{
    // device copy of sbh::BehzLevel (BFV multiply), see sb_bfv.cu
    struct BehzDev;
    // decryption constants of one prime (sb_engine.cu)
    struct DecConst;

    // the secret key on the device for decryption: powers s^1 .. s^powers in NTT form at the key level, [powers][k][n]
    struct SecretKey
    {
        struct Context *ctx = nullptr;
        DevBuf<u64> d_pow; // made with wipe set: zeroed before it is freed
        size_t powers = 0;
    };

    // PublicKey::data() on the device: [2][k][n], NTT form at the key level
    struct PublicKey
    {
        struct Context *ctx = nullptr;
        DevBuf<u64> d_key;
    };

    struct KSwitchKey
    {
        struct Context *ctx = nullptr;
        DevBuf<u64> d_key;        // [digits][2][k][n]
        DevBuf<uint32_t> d_key32; // [S][digits][2][k][n]: the key modulo the auxiliary primes, transformed (sb_ksint.cuh)
        size_t digits = 0;
    };

    // staging for the host-buffer entry points (sb_api.cu: HostPipe)
    struct IoArena
    {
        Stream s_in, s_comp, s_out;
        Event ev_in[2], ev_comp[2], ev_out[2];
        DevBuf<u64> buf[2][3];
        // page-locked staging of sb200_upload_rows ([0]) / sb200_download_rows ([1]): separate double buffers, streams and locks,
        // so that an upload, a download and the kernels of a third batch overlap (three host threads, or one thread per direction)
        struct Lane
        {
            PinnedBuf pin[2];
            Event ev[2], order;
            Stream st;
            std::mutex mu;
        } lane[2];
    };

    struct Context
    {
        int scheme = 0, device = 0, logn = 0;
        bool fast_q = true;                  // every q prime < 2^57: guard-free forward butterflies (sb_device.cuh)
        size_t n = 0, k = 0;
        u64 t = 0;
        std::vector<u64> q;                  // key-level primes
        std::vector<sbh::PrimeTables> tabs;  // host tables; ids [0,k) = q primes, [k, ...) = BEHZ auxiliary primes
        std::vector<u64> aux;                // auxiliary prime list [m_sk, gamma, B_0, B_1, ...] (BFV)
        std::vector<DevBuf<Tw>> d_fwd, d_inv; // per prime id
        DevBuf<PrimeDev> d_primes;           // [nprimes]
        size_t nprimes = 0;
        DevBuf<Tw> d_invq;                   // [k][k]: d_invq[j*k+i] = q_j^-1 mod q_i  (i != j)
        DevBuf<Tw> d_qmod;                   // BGV, [k][k]: d_qmod[j*k+i] = q_j mod q_i
        u64 t_ratio = 0;                     // BGV: floor(2^64 / t)
        std::vector<u64> inv_q_mod_t;        // BGV: q_j^-1 mod t
        // decryption constants per level (sb_engine.cu: decrypt_level)
        struct DecryptLevel
        {
            DevBuf<DecConst> d_consts; // [L]
            u64 neg_inv_q_mod_t = 0, neg_inv_q_mod_g = 0, q_mod_t = 0;
        };
        std::map<size_t, DecryptLevel> decrypt_levels;
        // BatchEncoder on the device (BFV / BGV with an NTT-friendly plain modulus): prime id of t and the inverse slot map
        int t_pid = -1;
        DevBuf<uint32_t> d_batch_inv_map;    // coefficient index -> matrix slot
        // coefficient-form plaintext operations (BFV / BGV): per-level constants, built on first use (sb_engine.cu: plain_level)
        struct PlainLevel
        {
            DevBuf<Tw> d_delta;     // [L]: floor(q / t) mod q_i (ContextData::coeff_div_plain_modulus, context.cpp:300-318)
            u64 q_mod_t = 0;        // ContextData::coeff_modulus_mod_plain_modulus
        };
        std::map<size_t, PlainLevel> plain_levels;
        // CKKSEncoder on the device (sb_ckks.cu): complex root tables + slot map, built on first use
        struct CkksEncoder
        {
            DevBuf<double2> d_roots, d_inv_roots; // [n]
            DevBuf<uint32_t> d_map;               // matrix_reps_index_map_
            DevBuf<u64> d_stat;                   // { max |coefficient| bits, flags }
        } ckks;
        // per-level big integers of the CRT composition (crt_compose, sb_device.cuh), built on first use (crt_level); they depend on
        // the primes only: CKKS decode and the BFV / BGV invariant noise budget share them
        struct CrtLevel
        {
            int total_bits = 0;
            DevBuf<u64> d_big; // [Q | (Q+1)/2 | Q/q_j ...] words
            DevBuf<Tw> d_invp; // (Q/q_j)^-1 mod q_j
        };
        std::map<size_t, CrtLevel> crt_levels;
        DevBuf<u64> d_t_mod_q;      // [k]: t mod q_i
        u64 t_ratio_lo = 0, t_ratio_hi = 0; // floor(2^128 / t)
        std::vector<std::array<u64, 4>> parms_ids; // parms_ids[L-1] = parms_id of the level with L primes (sb_wire.hpp)
        std::map<uint32_t, DevBuf<uint32_t>> galois_tables; // NTT-form permutation tables
        std::map<size_t, std::shared_ptr<BehzDev>> behz; // per level L
        DevBuf<unsigned char> scratch;
        DevBuf<int> d_flag;                  // result word of the range check (op_residues_in_range)
        DevBuf<unsigned char> aux_buf;       // second grow-only arena (size-3 intermediate of BFV multiply+relinearize)
        size_t scratch_used = 0, aux_used = 0; // bytes of the latest ensure_scratch / ensure_aux request (what wipe_* clears)
        size_t table_bytes = 0, scratch_budget = size_t(8) << 30;
        size_t ks_chunk_max = 0;                       // 0 = derived from scratch_budget (sb200_context_set_limit)
        size_t host_stage_bytes = size_t(640) << 20;   // per pipeline slot of the *_host entry points
        LaunchStats stats;
        KsInt ksint;                         // integer key-switching path (sb_ksint.cuh); ready = tables built
        // key switching: 0 = 64-bit digit transforms, 1 = automatic (the integer path from ks_min_digits digits on: below that the
        // L (L+1) large transforms are cheaper than S L + 2 S (L+1) small ones plus the reconstruction), 2 = integer path always.
        // In both modes 1 and 2, levels with more than ksint.max_digits digits (65 and up at n = 4096) take the 64-bit path: the
        // unreduced 64-bit sums of the integer path's product kernels would overflow there.
        int ks_algo = 1;
        size_t ks_min_digits = 16; // H100: the 64-bit path is still ahead at 15 digits, the integer path at 31 (DESIGN.md 3.2)
        bool ksint_on(size_t L) const
        {
            return ksint.ready && L <= ksint.max_digits && (ks_algo == 2 || (ks_algo == 1 && L >= ks_min_digits));
        }
        IoArena io;
        std::mutex mu;
        // cross-stream ordering of calls that share the scratch arenas (sb_api.cu: StreamOrder)
        Event order_event;
        cudaStream_t order_stream = nullptr;
        bool order_valid = false;

        ~Context() { cudaSetDevice(device); } // the members free their memory on this device
        void *ensure_scratch(size_t bytes);
        void *ensure_aux(size_t bytes);
        // secret-dependent intermediates (decryption phases, encryption noise) do not stay in the arenas: the reference keeps them in
        // clear-on-destruction pools (decryptor.cpp:106-109, util/rlwe.cpp:195, 292)
        void wipe_scratch(cudaStream_t st);
        void wipe_aux(cudaStream_t st);
        const uint32_t *galois_table(uint32_t elt);
        size_t prime_id_aux(size_t aux_index) const { return k + aux_index; }
    };

    // a host array as a device table of the context, counted in table_bytes.  T is the device type of the same bytes (Tw for
    // sbh::TwPair, uint2 for pairs of uint32_t, ...)
    template <class T, class S>
    DevBuf<T> upload(Context &c, const std::vector<S> &h)
    {
        static_assert(sizeof(T) % sizeof(S) == 0, "layout");
        DevBuf<T> d(h.size() * sizeof(S) / sizeof(T));
        if (d)
            cuda_check(cudaMemcpy(d.get(), h.data(), d.bytes(), cudaMemcpyHostToDevice), "upload table");
        c.table_bytes += d.bytes();
        return d;
    }

    std::unique_ptr<Context> make_context(int scheme, size_t n, const u64 *moduli, size_t k, u64 t, int device);

    // drivers (all stream-ordered, no synchronisation); slabs as documented in include/seal_b200.h
    void op_ntt(Context &c, bool inverse, size_t L, size_t size, size_t batch, u64 *d, cudaStream_t st);
    void op_linear(Context &c, int mode, size_t L, size_t size, size_t batch, const u64 *a, const u64 *b, u64 *out, cudaStream_t st);
    // add_many (sb200_add_many): count operands [B][sizes[j]][L][n] folded left into out [B][max size][L][n]; modes[j - 1] is step j's
    // mode (bit 0 sub, bit 1 scaled by the pair factors[2 (j - 1)], factors[2 (j - 1) + 1]).  One launch takes kFoldMaxOperands operands;
    // longer folds continue from the partial result in out.  ops[0] may be out when sizes[0] is the largest size.
    constexpr int kFoldMaxOperands = 16;
    void op_add_many(Context &c, size_t L, size_t batch, size_t count, const size_t *sizes, const u64 *const *ops, const int *modes,
                     const u64 *factors, u64 *out, cudaStream_t st);
    // sums of plaintext products (sb_plainsum.cu, sb200_multiply_plain_sum): outs[j] [B][max sizes][L][n] = the fold (modes /
    // factors as op_add_many) over t < K of multiply_plain(cts[t] [B][sizes[t]][L][n], plains[j K + t]), plains[j K + t] =
    // [plain_counts[j K + t]][L][n] (NTT form) or [..][n] (coefficient form), a count of 1 shared by the batch.  Operands not in
    // NTT form are transformed into scratch; the 128-bit sums are reduced once per kPlainSumWindow terms.
    constexpr int kPlainSumWindow = 256;
    void op_multiply_plain_sum(Context &c, size_t L, size_t batch, size_t K, size_t M, const size_t *sizes, const u64 *const *cts,
                               const size_t *plain_counts, const u64 *const *plains, bool ct_ntt, bool plain_ntt, const int *modes,
                               const u64 *factors, u64 *const *outs, cudaStream_t st);
    // sums of ciphertext products (sb_plainsum.cu, sb200_multiply_sum): outs[j] [B][3][L][n] = the fold (modes / factors as
    // op_add_many) over t < K of multiply(lhs[j K + t], rhs[t]), every operand [B][2][L][n].  CKKS and BGV: one multiply_sum_kernel
    // pass, output tiles of kMultiplySumTile, the 128-bit sums reduced once per window of at most kMultiplySumWindow terms.  BFV:
    // op_bfv_multiply into the aux arena, a chunk of terms at a time, each chunk folded into the output by op_add_many.
    constexpr int kMultiplySumWindow = 128;
    constexpr int kMultiplySumTile = 2; // 72 / 102 / 178 registers at tiles of 1 / 2 / 4; a tile of 4 ran slower (DESIGN 3.4)
    void op_multiply_sum(Context &c, size_t L, size_t batch, size_t K, size_t M, const u64 *const *lhs, const u64 *const *rhs, const int *modes,
                         const u64 *factors, u64 *const *outs, cudaStream_t st);
    // Plaintext operations take one plaintext per ciphertext, or (shared) one plaintext for the whole batch.
    // NTT-form plaintexts [B][L][n] or [L][n]: multiply_plain of NTT-form ciphertexts; CKKS add_plain / sub_plain (c_0 only)
    void op_multiply_plain(Context &c, size_t L, size_t size, size_t batch, bool shared, const u64 *a, const u64 *plain, u64 *out,
                           cudaStream_t st);
    void op_add_plain_ntt(Context &c, size_t L, size_t size, size_t batch, bool shared, bool subtract, const u64 *ct, const u64 *plain, u64 *out,
                          cudaStream_t st);
    // Decryptor::decrypt (decryptor.cpp:62-197): ct [B][size][L][n] -> CKKS: NTT-form plaintexts [B][L][n]; BFV / BGV:
    // coefficient-form plaintexts [B][n].  h_cf: BGV correction factors per ciphertext (nullptr = 1).
    void secret_key_create(Context &c, const u64 *h_sk, SecretKey &out);
    void op_decrypt(Context &c, SecretKey &sk, size_t L, size_t size, size_t batch, const u64 *ct, const u64 *h_cf, u64 *plain, cudaStream_t st);
    // Decryptor::invariant_noise_budget (decryptor.cpp:409-486) for a batch of BFV (coefficient form) / BGV (NTT form) ciphertexts
    // [B][size][L][n] -> budgets [B] (device ints).  check_noise_budget throws what op_invariant_noise_budget would before any launch:
    // a foreign key or a size outside 2..16 (invalid_argument), a CKKS context (logic_error), more than 60 primes (invalid_argument,
    // the decryption limit).  Stream-ordered, no host synchronisation (beyond scratch growth).
    void check_noise_budget(const Context &c, const SecretKey &sk, size_t L, size_t size);
    void op_invariant_noise_budget(Context &c, SecretKey &sk, size_t L, size_t size, size_t batch, const u64 *ct, int *budgets, cudaStream_t st);
    // the CRT composition tables of the level with L primes (Context::CrtLevel)
    Context::CrtLevel &crt_level(Context &c, size_t L);
    // BatchEncoder::encode / decode (batchencoder.cpp:84-330): values [B][n] (< t) <-> coefficient-form plaintexts [B][n]
    void op_batch_encode(Context &c, size_t batch, const u64 *values, u64 *plain, cudaStream_t st);
    void op_batch_decode(Context &c, size_t batch, const u64 *plain, u64 *values, cudaStream_t st);
    // coefficient-form plaintexts [B][n] or [n] (words < t): lift + NTT, multiply_plain, add_plain / sub_plain (BFV, BGV);
    // h_cf: BGV correction factors on the host, one per plaintext (nullptr = 1)
    void op_plain_to_ntt(Context &c, size_t L, size_t batch, const u64 *plain, const u64 *h_cf, u64 *out, cudaStream_t st);
    void op_multiply_plain_coeff(Context &c, size_t L, size_t size, size_t batch, bool shared, bool ct_ntt, const u64 *ct, const u64 *plain,
                                 u64 *out, cudaStream_t st);
    void op_add_plain_coeff(Context &c, size_t L, size_t size, size_t batch, bool shared, bool subtract, const u64 *ct, const u64 *plain,
                            const u64 *h_cf, u64 *out, cudaStream_t st);
    // the constants of the level with L primes for coefficient-form plaintexts (BFV / BGV; builds c.d_t_mod_q and the t ratio too);
    // std::invalid_argument for CKKS
    const Context::PlainLevel &plain_level(Context &c, size_t L);
    void op_ckks_multiply(Context &c, size_t L, size_t batch, const u64 *a, const u64 *b, u64 *out3, cudaStream_t st);
    void op_bfv_multiply(Context &c, size_t L, size_t batch, const u64 *a, const u64 *b, u64 *out3, cudaStream_t st);
    // general ciphertext sizes s1 x s2 -> s1+s2-1 (2 x 2 forwards to the specialised kernels above)
    void op_ckks_multiply(Context &c, size_t L, size_t s1, size_t s2, size_t batch, const u64 *a, const u64 *b, u64 *out, cudaStream_t st);
    void op_bfv_multiply(Context &c, size_t L, size_t s1, size_t s2, size_t batch, const u64 *a, const u64 *b, u64 *out, cudaStream_t st);
    void check_sizes(size_t s1, size_t s2);
    // BFV multiplication accumulates its FastBConv sums unreduced in 128 bits: at most 64 products of words below 2^61 each, so a
    // level whose base B would hold more than 64 primes (more than 64 primes in the level, or 64 with B enlarged) is rejected.
    // check_bfv_multiply_level throws std::invalid_argument for such a level of a BFV context and does nothing otherwise.
    constexpr size_t kBfvMultiplyMaxBase = 64;
    void check_bfv_multiply_level(const Context &c, size_t L);
    void launch_tensor_general(Context &c, const u64 *xa, long long xa_bs, const u64 *xb, long long xb_bs, u64 *out, const int *pid_tab,
                               size_t nb, size_t s1, size_t s2, size_t B, cudaStream_t st);
    void op_relinearize(Context &c, size_t L, size_t batch, const u64 *in3, const KSwitchKey &key, u64 *out2, cudaStream_t st);
    void op_multiply_relinearize(Context &c, size_t L, size_t batch, const u64 *a, const u64 *b, const KSwitchKey &key,
                                 u64 *out2, cudaStream_t st);
    // polys = batch * size polynomials of L components each (any ciphertext size)
    void op_rescale(Context &c, size_t L, size_t polys, const u64 *in, u64 *out, cudaStream_t st);
    void op_mod_switch(Context &c, size_t L, size_t polys, const u64 *in, u64 *out, cudaStream_t st);
    void op_relinearize_sized(Context &c, size_t L, size_t size, size_t batch, const u64 *in, const KSwitchKey &key, u64 *out, cudaStream_t st);
    void op_apply_galois(Context &c, size_t L, size_t batch, const u64 *in2, uint32_t elt, const KSwitchKey &key, u64 *out2,
                         cudaStream_t st);
    // out = addend + apply_galois(in), the addition in the key switch's epilogue.  out may be addend (accumulate), addend may be in,
    // out == in is rejected
    void op_apply_galois_add(Context &c, size_t L, size_t batch, const u64 *in2, uint32_t elt, const KSwitchKey &key, const u64 *addend2,
                             u64 *out2, cudaStream_t st);
    // y_0 = in, y_{j+1} = y_j + apply_galois(y_j, elts[j]) with keys[j]; out = y_steps (out may be in; steps = 0 copies)
    void check_rotate_sum_args(const Context &c, size_t L, size_t steps, const uint32_t *elts, const KSwitchKey *const *keys);
    void op_rotate_sum(Context &c, size_t L, size_t batch, const u64 *in2, size_t steps, const uint32_t *elts, const KSwitchKey *const *keys,
                       u64 *out2, cudaStream_t st);
    // out = addend + plain * apply_galois(in), NTT-form plaintexts [P][L][n] (shared: P = 1).  CKKS / BGV: the product and the addition
    // in the key switch's last pass; BFV: the chain through one chunk-sized temporary.  out may be addend, addend may be in, out == in
    // is rejected
    void op_apply_galois_multiply_plain_add(Context &c, size_t L, size_t batch, const u64 *in2, uint32_t elt, const KSwitchKey &key, bool shared,
                                            const u64 *plain, const u64 *addend2, u64 *out2, cudaStream_t st);
    // out = sum_t plains[t] * apply_galois(in, elts[t]); element 1 is no rotation (its key may be NULL).  plain_counts[t]: 1 or batch;
    // plains NTT form [P][L][n] or (plain_ntt = false, BFV / BGV) coefficient form [P][n].  out must not alias in
    void check_diagonal_sum_args(const Context &c, size_t L, size_t count, const uint32_t *elts, const KSwitchKey *const *keys);
    void op_diagonal_sum(Context &c, size_t L, size_t batch, const u64 *in2, size_t count, const uint32_t *elts, const KSwitchKey *const *keys,
                         const size_t *plain_counts, const u64 *const *plains, bool plain_ntt, u64 *out2, cudaStream_t st);
    size_t keyswitch_chunk(const Context &c, size_t L, size_t batch, bool fused);
    // arithmetic ceilings measured in process: warp-level butterflies (kind 0-2) / multiply-accumulates (kind 3) per second
    double selftest_rate(Context &c, int kind, cudaStream_t st);
    // SEAL's prng_type (randomgen.h:29-36) of a PRNG whose stream the device generates (sb_prng.cu); anything else is rejected by
    // check_prng_type (std::invalid_argument)
    constexpr int kPrngBlake2xb = 1, kPrngShake256 = 2;
    void check_prng_type(int type);
    // Ciphertext::expand_seed on the device (sb_prng.cu): seeds [B][8] host words, types [B] their prng_type, dst_off [B] host word
    // offsets into d_out of the polynomial ([L][n]) each seed expands into; returns after the expansion has been enqueued and the
    // host arrays are free
    void op_expand_seeded(Context &c, size_t L, size_t B, const u64 *h_seeds, const int *h_types, const long long *h_dst_off, u64 *d_out,
                          cudaStream_t st);
    // Encryptor::encrypt_zero_symmetric on the device (sb_prng.cu): bootstrap seeds [B][8] on the host, out [B][2][L][n]; boot_prng =
    // the type of the bootstrap PRNG (parms.random_generator()), ct_prng = the type c_1 is expanded with (the DefaultFactory's)
    void op_encrypt_zero_symmetric(Context &c, const SecretKey &sk, size_t L, size_t B, const u64 *h_boot_seeds, int boot_prng, int ct_prng,
                                   bool save_seed, u64 *d_out, u64 *h_public_seeds, cudaStream_t st);
    // Encryptor::encrypt_symmetric on the device: op_encrypt_zero_symmetric with one plaintext per ciphertext added as c_0 is written.
    // d_plain: CKKS [B][L][n] NTT form at the level; BFV / BGV [B][n] words < t (L = the first level).  d_plain must not alias d_out.
    void op_encrypt_symmetric(Context &c, const SecretKey &sk, size_t L, size_t B, const u64 *d_plain, const u64 *h_boot_seeds, int boot_prng,
                              int ct_prng, bool save_seed, u64 *d_out, u64 *h_public_seeds, cudaStream_t st);
    // KeyGenerator on the device (sb_prng.cu), for a secret key the caller supplies.  What turns a key-level encryption of zero into
    // digit digit0 + b of a key-switching key: s'_j[i] = new_key[j][perm ? perm[i] : i] (sb_prng.cu: enc_kernel MODE 7)
    struct KsFactor
    {
        const u64 *new_key = nullptr;   // [k][n], NTT form
        const uint32_t *perm = nullptr; // NTT-form Galois table, or nullptr
        long long digit0 = 0;
    };
    // KeyGenerator::create_public_key: h_boot_seed [8], d_out [2][k][n]; h_public_seed: nullptr or [8], the seed c_1 expands from
    // (the stream synchronised on return)
    void op_generate_public_key(Context &c, const SecretKey &sk, int boot_prng, int ct_prng, const u64 *h_boot_seed, u64 *d_out, cudaStream_t st,
                                u64 *h_public_seed = nullptr);
    // KeyGenerator::create_relin_keys (galois_elt = 0) / the key of one Galois element: h_boot_seeds [k-1][8] (one per digit),
    // d_out [k-1][2][k][n].  Returns once the host seeds have been consumed (they may be wiped then).  h_public_seeds: nullptr or
    // [k-1][8], each digit's public seed; with it, on_chunk(d0, count) (if set) runs after each chunk of digits is complete on the device.
    void op_generate_kswitch_key(Context &c, SecretKey &sk, uint32_t galois_elt, int boot_prng, int ct_prng, const u64 *h_boot_seeds, u64 *d_out,
                                 cudaStream_t st, u64 *h_public_seeds = nullptr, const std::function<void(size_t, size_t)> &on_chunk = {});
    // Decryptor::compute_secret_key_array (sb_engine.cu): s^1 .. s^powers at the key level in sk.d_pow
    void ensure_key_powers(Context &c, SecretKey &sk, size_t powers, cudaStream_t st);
    // Encryptor(public key)::encrypt_zero on the device (sb_prng.cu): seeds [B][8] on the host for PRNGs of type prng, out [B][2][L][n]
    void public_key_create(Context &c, const u64 *h_pk, PublicKey &out);
    void op_encrypt_zero_asymmetric(Context &c, const PublicKey &pk, size_t L, size_t B, const u64 *h_seeds, int prng, u64 *d_out, cudaStream_t st);
    // Encryptor(public key)::encrypt: op_encrypt_zero_asymmetric, then the plaintexts (layout as op_encrypt_symmetric) added to c_0
    void op_encrypt_asymmetric(Context &c, const PublicKey &pk, size_t L, size_t B, const u64 *d_plain, const u64 *h_seeds, int prng, u64 *d_out,
                               cudaStream_t st);
    // CKKSEncoder::encode / decode (sb_ckks.cu): values = device doubles, [B][count] complex pairs (or reals); plain = [B][L][n] NTT form.
    // broadcast: values holds one value per member, encoded into every one of count slots
    void op_ckks_encode(Context &c, size_t L, size_t B, const double *values, size_t count, bool is_complex, double scale, u64 *plain,
                        cudaStream_t st, bool broadcast = false);
    // CKKSEncoder::encode of one scalar per member (ckks.h:272-377): values = device words [B] (kind real: a double, int64: an int64_t)
    // or [B][2] (complex: re, im); plain = [B][L][n] NTT form.  Real and int64 synchronise the stream once to check the values on the
    // host, then one fill kernel writes the constant polynomials; complex is the vector encode of n/2 copies.  scale is ignored for int64.
    constexpr int kCkksScalarReal = 0, kCkksScalarComplex = 1, kCkksScalarInt64 = 2; // SB200_CKKS_SCALAR_*
    void op_ckks_encode_scalar(Context &c, size_t L, size_t B, int kind, const u64 *values, double scale, u64 *plain, cudaStream_t st);
    // the checks of op_ckks_encode_scalar that need no values (kind, scheme, level, scale), and those of B host values (real, int64),
    // each in the reference's order and with its messages (std::invalid_argument)
    void check_ckks_scalar(const Context &c, size_t L, int kind, double scale);
    void check_ckks_scalar_values(const Context &c, size_t L, size_t B, int kind, const u64 *h_values, double scale);
    void op_ckks_decode(Context &c, size_t L, size_t B, const u64 *plain, double scale, double *values, cudaStream_t st);
    const sbh::BehzLevel &behz_host(Context &c, size_t L);
    // wire format support (sb_api.cu): 1 if any residue of data [rows][n] (prime of a row = row % L) is >= its modulus
    bool op_residues_in_range(Context &c, size_t L, size_t rows, const u64 *d, cudaStream_t st);
} // namespace sb
