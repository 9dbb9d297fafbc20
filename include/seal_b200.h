/* include/seal_b200.h -- C-ABI of libseal_b200.so: the H100 (sm_90a) drop-in for the RNS-polynomial hot path of
 * microsoft/SEAL 4.4.3 (negacyclic NTT/INTT, dyadic products, hybrid key switching, rescale / BEHZ base conversion)
 * that backs Evaluator::multiply / relinearize_inplace / rotate_rows / rotate_vector / rescale_to_next.
 *
 * Style follows the reference's own C layer (native/src/seal/c/defines.h:34-96): extern "C", opaque handles, plain
 * pointers and sizes, an integer status instead of exceptions, a last-error string.  Unlike the reference's C layer
 * the data arguments are raw uint64 slabs laid out exactly like seal::Ciphertext::data() (ciphertext.h:24-37):
 *
 *      [batch][poly (size)][rns prime (L)][coefficient (n)]       8*n*L*size bytes per ciphertext
 *
 * so a binding marshals `ct.data()` with one memcpy (see INTEGRATION.md).  `L` = number of RNS primes the
 * ciphertexts carry = parms.coeff_modulus().size() at that level of the modulus-switching chain; the key level has
 * k primes, ciphertexts have L <= k-1 (context.cpp:513-535).  Device entry points (d_ prefix on arguments) are
 * stream-ordered and never synchronise; the *_host entry points take host buffers, copy H2D / D2H themselves and
 * return after the result is in the host buffer.
 *
 * There is NO CPU fallback: every entry point fails with SB200_E_CUDA when no sm_90 device is usable.
 */
#ifndef SEAL_B200_H
#define SEAL_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* status codes; the mapping mirrors the reference's exception -> HRESULT ladder (c/defines.h:72-96) */
#define SB200_OK 0
#define SB200_E_INVALID_ARG (-1)  /* std::invalid_argument  -> E_INVALIDARG            */
#define SB200_E_LOGIC (-2)        /* std::logic_error       -> COR_E_INVALIDOPERATION  */
#define SB200_E_OUT_OF_RANGE (-3) /* std::out_of_range      -> ERROR_INVALID_INDEX     */
#define SB200_E_CUDA (-4)         /* std::runtime_error     -> COR_E_IO                */
#define SB200_E_NOMEM (-5)        /* std::bad_alloc         -> E_OUTOFMEMORY           */
#define SB200_E_POINTER (-6)      /* null handle / pointer  -> E_POINTER               */

#define SB200_SCHEME_BFV 1  /* seal::scheme_type::bfv  (encryptionparams.h) */
#define SB200_SCHEME_CKKS 2 /* seal::scheme_type::ckks */
#define SB200_SCHEME_BGV 3  /* seal::scheme_type::bgv: NTT-form ciphertexts like CKKS, plain-modulus-aware mod-down (SURVEY 8f rank 2) */

typedef struct sb200_context sb200_context;   /* mirrors SEALContext + Evaluator state (context.h:277-439) */
typedef struct sb200_public_key sb200_public_key;   /* Encryptor state: the public key on the device (publickey.h) */
typedef struct sb200_secret_key sb200_secret_key;   /* Decryptor state: the secret key and its powers on the device (decryptor.h) */
typedef struct sb200_kswitch_key sb200_kswitch_key; /* one KSwitchKeys::data()[index] entry on the device (kswitchkeys.h) */

/* last error message of the calling thread (never NULL) */
const char *sb200_last_error(void);

/* ---- context ------------------------------------------------------------------------------------------------
 * Replaces SEALContext(parms, expand_mod_chain=true, sec_level_type::none) + Evaluator(context) for this path
 * (context.cpp:495-563, evaluator.cpp:121-128).  coeff_modulus = the k key-level primes (last = special prime),
 * each < 2^61, prime, = 1 mod 2n.  plain_modulus is used by BFV and BGV (BGV: coprime to every prime, rns.cpp:778-787).  All NTT / RNS / Galois tables are computed
 * here from these numbers alone and uploaded to CUDA device `device`. */
int sb200_context_create(int scheme, size_t poly_modulus_degree, const uint64_t *coeff_modulus, size_t k,
                         uint64_t plain_modulus, int device, sb200_context **out);
int sb200_context_destroy(sb200_context *ctx);
/* helpers that reproduce CoeffModulus::Create (modulus.cpp:144-184) */
int sb200_coeff_modulus_create(size_t poly_modulus_degree, const int *bit_sizes, size_t k, uint64_t *out);
/* table introspection for parity tests: NTTTables::get_root / get_from_root_powers / get_from_inv_root_powers /
 * inv_degree_modulo (ntt.h:95-123) in the reference's own order; any output pointer may be NULL */
int sb200_get_ntt_tables(const sb200_context *ctx, size_t prime_index, uint64_t *root, uint64_t *root_powers_operand,
                         uint64_t *root_powers_quotient, uint64_t *inv_root_powers_operand, uint64_t *inv_degree_modulo);
/* RNSTool::base_Bsk() at the level with L primes (rns.h:246-309); out gets |Bsk| values */
int sb200_get_base_bsk(const sb200_context *ctx, size_t L, uint64_t *out, size_t capacity, size_t *count);
/* GaloisTool::get_elt_from_step (galois.cpp:53-95); returns 0 on invalid step */
uint32_t sb200_galois_elt_from_step(const sb200_context *ctx, int step);
/* number of CUDA kernels launched through this context so far */
unsigned long long sb200_launch_count(const sb200_context *ctx);
/* device bytes currently held by the context: its tables, including those built on first use (per-level decryption, plaintext
 * and CRT constants, Galois permutations, encoder and BEHZ tables), plus the two scratch arenas */
size_t sb200_device_bytes(const sb200_context *ctx);
/* resource limits of a context (the reference's counterpart is the MemoryPoolHandle a caller passes to Evaluator members,
 * evaluator.h:219-252): how a batch is cut into device chunks.  Results never depend on them; the parity tests use them
 * to force the multi-chunk paths (ragged last chunk) at small batch sizes.
 *   SB200_LIMIT_SCRATCH_BYTES     budget of the per-context scratch arena (default 8 GiB, env SB200_SCRATCH_MB)
 *   SB200_LIMIT_KS_CHUNK          max ciphertexts per key-switching chunk (0 = derived from the scratch budget)
 *   SB200_LIMIT_HOST_STAGE_BYTES  device staging per pipeline slot of the *_host entry points (default 640 MiB)
 *   SB200_LIMIT_KS_ALGORITHM      key switching: 0 = 64-bit digit transforms per output prime; 1 (default, env SB200_KS_ALGO) =
 *                                 automatic: the exact integer convolution on 29-bit auxiliary primes where it is available
 *                                 (n >= 4096) and pays (levels with >= 16 digits, env SB200_KS_MIN_DIGITS); 2 = that path at every
 *                                 level.  In modes 1 and 2, levels with more digits than the path's unreduced 64-bit product sums
 *                                 hold (L (p_max - 1)^2 >= 2^64: above 64 digits at n = 4096) take the 64-bit digit transforms.
 *                                 Results are identical words in every mode. */
#define SB200_LIMIT_SCRATCH_BYTES 0
#define SB200_LIMIT_KS_CHUNK 1
#define SB200_LIMIT_HOST_STAGE_BYTES 2
#define SB200_LIMIT_KS_ALGORITHM 3
int sb200_context_set_limit(sb200_context *ctx, int which, size_t value);

/* ---- device-resident slabs (the storage behind seal_b200::CiphertextBatch, include/seal_b200/batch.hpp) ------------
 * The reference hands out ciphertext storage from a MemoryPoolHandle (memorymanager.h:36-54, ciphertext.h:100-140); a
 * caller that keeps ciphertexts on the device between Evaluator calls allocates their slabs here.  Slabs belong to the
 * context's device; sb200_host_malloc returns page-locked host memory (first-touched by the calling thread, so bind the
 * thread to the device's NUMA node first) for staging that the *_host entry points and the copies below can stream
 * from at full PCIe rate.  Copies are stream-ordered; sb200_stream_synchronize(ctx, stream) waits for them. */
int sb200_device_malloc(sb200_context *ctx, size_t bytes, uint64_t **d_out);
int sb200_device_free(sb200_context *ctx, uint64_t *d_ptr);
int sb200_host_malloc(sb200_context *ctx, size_t bytes, void **h_out);
int sb200_host_free(sb200_context *ctx, void *h_ptr);
int sb200_memcpy_h2d(sb200_context *ctx, uint64_t *d_dst, const void *h_src, size_t bytes, void *stream);
int sb200_memcpy_d2h(sb200_context *ctx, void *h_dst, const uint64_t *d_src, size_t bytes, void *stream);
int sb200_memcpy_d2d(sb200_context *ctx, uint64_t *d_dst, const uint64_t *d_src, size_t bytes, void *stream);
/* strided copies between ciphertext objects and slabs: `rows` runs of row_bytes, source / destination pitch in bytes
 * (drops or keeps RNS components without touching the rest: mod_switch_drop_to_next, evaluator.cpp:1296-1358) */
int sb200_memcpy_d2d_2d(sb200_context *ctx, uint64_t *d_dst, size_t dst_pitch, const uint64_t *d_src, size_t src_pitch, size_t row_bytes,
                        size_t rows, void *stream);
int sb200_stream_synchronize(sb200_context *ctx, void *stream);
/* gather / scatter between `count` separate host objects (e.g. seal::Ciphertext::data() of a std::vector<Ciphertext>, pageable
 * pool memory) and one device slab [count][row_bytes]: staged through page-locked double buffers owned by the context, several
 * host threads copy, H2D / D2H overlap the host copies.  Both return when the data has arrived. */
int sb200_upload_rows(sb200_context *ctx, uint64_t *d_dst, const uint64_t *const *h_rows, size_t row_bytes, size_t count);
int sb200_download_rows(sb200_context *ctx, uint64_t *const *h_rows, const uint64_t *d_src, size_t row_bytes, size_t count);
/* NUMA node of the context's device (-1 when the platform does not say) and the CUDA device index */
int sb200_device_numa_node(const sb200_context *ctx);
int sb200_device_index(const sb200_context *ctx);
/* ciphertexts per key-switching chunk the context would use for `batch` ciphertexts at level L (fused != 0: the
 * multiply_relinearize entry point).  bench.py samples its verification indices on both sides of a chunk boundary. */
size_t sb200_keyswitch_chunk(const sb200_context *ctx, size_t L, size_t batch, int fused);

/* ---- per-kernel timing (CUDA events on the launching stream) -------------------------------------------------
 * enable, run operations, then read entries 0,1,... until SB200_E_OUT_OF_RANGE.  Each entry aggregates one kernel
 * (a transform contributes "<name>:col" and "<name>:local"): total device ms, launches, and the algorithmic bytes
 * those launches had to move (DESIGN.md lists the per-kernel formula).  Used by bench.py for the roofline line. */
int sb200_profile_enable(sb200_context *ctx, int on);
int sb200_profile_reset(sb200_context *ctx);
int sb200_profile_read(sb200_context *ctx, size_t index, char *name, size_t name_capacity, double *total_ms,
                       unsigned long long *launches, double *algorithmic_bytes);
/* the same plus the arithmetic those launches executed: modular butterflies and 64x64-bit key multiply-accumulates (per
 * coefficient, not per warp) -- the work of the second ceiling of SURVEY 8(d), the integer-multiply issue rate */
int sb200_profile_read_work(sb200_context *ctx, size_t index, char *name, size_t name_capacity, double *total_ms,
                            unsigned long long *launches, double *algorithmic_bytes, double *butterflies, double *macs);
/* that ceiling, measured in this process on the context's device: the path's own butterfly / multiply-accumulate code on
 * registers only, at the launch shapes of the dominant kernels.  kind 0: forward butterflies (column-pass shape), 1: forward
 * butterflies (fused kernel's shape), 2: inverse butterflies, 3: key multiply-accumulates.  Result: warp-level operations per
 * second of the whole device (one warp-level operation = 32 coefficient-level ones). */
int sb200_selftest_rate(sb200_context *ctx, int kind, double *warp_ops_per_second);
/* the integer key-switching path (SB200_LIMIT_KS_ALGORITHM 1): its work is counted in 32-bit butterflies and 32x32->64-bit
 * multiply-accumulates (sb200_profile_read_work32 = sb200_profile_read_work + those two counters); sb200_selftest_rate kinds
 * 10, 11, 12 measure their ceilings (forward butterflies, inverse butterflies, multiply-accumulates); 13, 14, 15 repeat the
 * multiply-accumulate loop at the key-tile kernel's launch shape (512 threads, one CTA per SM), with two products per accumulator and
 * round (the product kernel's form: one three-input 64-bit add per pair), and with both.  The transforms modulo the
 * auxiliary primes are exposed for the parity tests: _info returns the primes (capacity 8), _forward maps rows of n 64-bit
 * words to h_out[prime][row][n] (canonical residues, transformed), _inverse transforms h_data[row][prime][n] in place (values
 * in [0, 2p), not scaled by n^-1).  _product runs the product step alone: h_Dh[prime][digit][ciphertext][n] and
 * h_key[prime][digit][component 2][output prime L + 1][n] (canonical residues) -> h_Acc[ciphertext][2][L + 1][prime][n] (values in
 * [0, 2p)); kernel 0 = the integer-pipe kernels, 1 = the INT8 tensor-core kernel where the shape allows it (L <= 32 digits,
 * B >= 16 ciphertexts); *ran (may be NULL) receives the kernel that ran: 0 register tile, 1 key tile, 2 tensor cores. */
int sb200_profile_read_work32(sb200_context *ctx, size_t index, char *name, size_t name_capacity, double *total_ms,
                              unsigned long long *launches, double *algorithmic_bytes, double *butterflies, double *macs,
                              double *butterflies32, double *macs32);
int sb200_selftest_ksint_info(sb200_context *ctx, int *count, uint32_t *primes);
int sb200_selftest_ksint_forward(sb200_context *ctx, const uint64_t *h_rows, size_t rows, uint32_t *h_out);
int sb200_selftest_ksint_inverse(sb200_context *ctx, uint32_t *h_data, size_t rows);
int sb200_selftest_ksint_product(sb200_context *ctx, const uint32_t *h_Dh, const uint32_t *h_key, size_t L, size_t B, uint32_t *h_Acc,
                                 int kernel, int *ran);

/* ---- key-switching keys --------------------------------------------------------------------------------------
 * h_key = the flattened KSwitchKeys::data()[index]: [digit j < digits][component 2][key prime k][coeff n], i.e. for
 * each j the PublicKey's ciphertext data (kswitchkeys.h, keygenerator.cpp:327-360).  digits must be >= L of every
 * ciphertext it is used with (evaluator.cpp:2635).  For n >= 4096 the handle also holds the key modulo the context's 29-bit
 * auxiliary primes in transformed form (2.5x the bytes above, prepared once at creation: INTT of every key row + the small
 * forward transforms), which is what key switching at levels with >= 16 digits multiplies with (SB200_LIMIT_KS_ALGORITHM). */
int sb200_kswitch_key_create(sb200_context *ctx, const uint64_t *h_key, size_t digits, sb200_kswitch_key **out);
int sb200_kswitch_key_destroy(sb200_kswitch_key *key);
/* KSwitchKeys::load of the single entry data()[index] out of a RelinKeys / GaloisKeys stream saved with
 * compr_mode_type::none or zlib (kswitchkeys.cpp:42-160): the key polynomials go from the stream to the device directly.
 * Seed-compressed members (what KeyGenerator::create_relin_keys / create_galois_keys return as Serializable objects: c_0 and
 * the seed of c_1, of either prng_type) upload c_0 only and expand every digit's c_1 on the device at the key level, bit for bit
 * as Ciphertext::expand_seed does (ciphertext.cpp:118-150); the seeded relinearization key of n = 65536, k = 32 is half the bytes.
 * index = RelinKeys::get_index(2) = 0 for relinearization, GaloisKeys::get_index(galois_elt) = (galois_elt - 1) / 2 for a
 * rotation (relinkeys.h:58-65, galoiskeys.h:48-51).  SB200_E_OUT_OF_RANGE: no such slot; SB200_E_INVALID_ARG: empty slot. */
int sb200_kswitch_key_load(sb200_context *ctx, const uint8_t *stream, size_t len, size_t index, sb200_kswitch_key **out);
/* KSwitchKeys::load of several entries in one pass: the object is inflated at most once and its frame parsed once, and every
 * seeded digit expands on the device.  out[i] = the handle sb200_kswitch_key_load(..., indices[i]) makes, i < count.  indices ==
 * NULL: every non-empty slot in slot order, count = the capacity of out and out_indices.  out_indices (may be NULL) receives each
 * handle's slot, *out_count the number of handles.  Errors, all checked before the first handle is made: SB200_E_OUT_OF_RANGE an
 * index at or past the slot count; SB200_E_INVALID_ARG an empty slot, a duplicated index, or too small a capacity for the NULL
 * form; SB200_E_LOGIC keys of another context.  A failure after that (a word >= its modulus: SB200_E_LOGIC) destroys the
 * handles made so far; out is written only on success.  sb200_kswitch_key_load is the count = 1 case. */
int sb200_kswitch_keys_load(sb200_context *ctx, const uint8_t *stream, size_t len, const size_t *indices, size_t count,
                            sb200_kswitch_key **out, size_t *out_indices, size_t *out_count);
/* bytes the handle holds on the device: the key words plus the integer path's copy (0 for NULL) */
size_t sb200_kswitch_key_device_bytes(const sb200_kswitch_key *key);

/* ---- device-resident batch operations (stream = cudaStream_t, may be NULL) ----------------------------------
 * Output slabs must not alias input slabs unless noted: multiply_relinearize may write over d_a or d_b, add/sub/negate/multiply_plain
 * may run in place; relinearize / rescale / mod_switch / apply_galois change the layout and reject aliasing. */
/* Evaluator::transform_to_ntt_inplace / transform_from_ntt_inplace (evaluator.cpp:2289-2382) */
int sb200_ntt_forward(sb200_context *ctx, size_t L, size_t size, size_t batch, uint64_t *d_data, void *stream);
int sb200_ntt_inverse(sb200_context *ctx, size_t L, size_t size, size_t batch, uint64_t *d_data, void *stream);
/* Evaluator::multiply (evaluator.cpp:352-708), size-2 x size-2 -> size-3; CKKS (NTT form) or BFV (BEHZ) per ctx.
 * BFV multiplication (multiply, multiply_sized, square, multiply_relinearize) supports levels of at most 64 primes whose BEHZ
 * base B holds at most 64 primes (63 primes when the plain modulus enlarges B); deeper levels are rejected with
 * SB200_E_INVALID_ARG before any launch, as decryption rejects levels of more than 60 primes. */
int sb200_multiply(sb200_context *ctx, size_t L, size_t batch, const uint64_t *d_a, const uint64_t *d_b,
                   uint64_t *d_out3, void *stream);
/* the general-size branches of the same function (evaluator.cpp:524-560, :664-700, :796-833): size_a x size_b ->
 * size_a + size_b - 1, out[k] = sum_{i+j=k} a_i * b_j; 2 <= size <= 16 (SEAL_CIPHERTEXT_SIZE_MAX).  No aliasing. */
int sb200_multiply_sized(sb200_context *ctx, size_t L, size_t size_a, size_t size_b, size_t batch, const uint64_t *d_a,
                         const uint64_t *d_b, uint64_t *d_out, void *stream);
/* Evaluator::square (evaluator.cpp:843-1142): same residues as multiply(a, a), size 2 -> 3 */
int sb200_square(sb200_context *ctx, size_t L, size_t batch, const uint64_t *d_a, uint64_t *d_out3, void *stream);
/* Evaluator::add / sub / negate on equal-size operands (evaluator.cpp:130-350), element-wise over [batch][size][L][n];
 * these are the "next" row of SURVEY 8(f): the linear ops users interleave with multiply / relinearize / rescale */
int sb200_add(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *d_a, const uint64_t *d_b, uint64_t *d_out, void *stream);
int sb200_sub(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *d_a, const uint64_t *d_b, uint64_t *d_out, void *stream);
int sb200_negate(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *d_a, uint64_t *d_out, void *stream);
/* Evaluator::add_many (evaluator.cpp:236-262) generalised to a left fold of add_inplace / sub_inplace steps (:155-350), in one
 * pass over the operands.  Operand j (0 <= j < count) is d_operands[j], [batch][sizes[j]][L][n], 1 <= sizes[j] <= 16; d_out is
 * [batch][max sizes[j]][L][n].  Step j >= 1 folds operand j into the accumulator with modes[j - 1]: SB200_FOLD_ADD (0) or
 * SB200_FOLD_SUB (1), optionally ORed with SB200_FOLD_SCALED (2): before the step the accumulator's present polynomials are
 * multiplied by h_factors[2 (j - 1)] and operand j by h_factors[2 (j - 1) + 1] (BGV correction-factor balancing,
 * :188-209; the factors are host words, reduced mod each prime here).  modes may be NULL (every step adds); h_factors may be
 * NULL when no step is scaled.  A polynomial no earlier operand has is copied (add) or negated (sub), as the reference copies or
 * negates the longer operand's tail.  The words equal those of the chained add / sub calls for any input words.
 * Errors, all before the first launch: count = 0 or a size outside 1..16 or a mode outside 0..3 (SB200_E_INVALID_ARG); a NULL
 * operand, d_out, sizes or (with a scaled step) h_factors (SB200_E_POINTER); d_out overlapping an operand other than exactly in
 * place on operand 0 (d_out == d_operands[0] with sizes[0] the largest size) (SB200_E_INVALID_ARG).  The _host form stages the
 * batch through the pipeline of every _host entry point, in chunks of SB200_LIMIT_HOST_STAGE_BYTES per pipeline slot. */
#define SB200_FOLD_ADD 0
#define SB200_FOLD_SUB 1
#define SB200_FOLD_SCALED 2
int sb200_add_many(sb200_context *ctx, size_t L, size_t batch, size_t count, const size_t *sizes, const uint64_t *const *d_operands,
                   const int *modes, const uint64_t *h_factors, uint64_t *d_out, void *stream);
/* Sums of plaintext products: a plaintext matrix times a vector of ciphertexts in one pass.  Member b of d_outs[j] (j < outputs = M)
 * has the words of the chain t_i = multiply_plain(member b of d_cts[i], plaintext b (or the shared one) of d_plains[j K + i]) for
 * i < count = K, then sb200_add_many(t_0 .. t_{K-1}, modes, h_factors) (evaluator.cpp:1975-2195, :155-262), for any input words.
 *   d_cts[i]: [batch][sizes[i]][L][n], 1 <= sizes[i] <= 16, all in NTT form (ct_is_ntt = 1) or all in coefficient form (0, BFV);
 *   d_plains[j K + i]: plain_counts[j K + i] plaintexts (1: shared by the batch, or batch), all NTT form [count][L][n] at the
 *     ciphertexts' level (plain_is_ntt = 1) or all coefficient form [count][n], words < t, zero above coeff_count (0, BFV / BGV);
 *   modes [K - 1] / h_factors [K - 1][2]: as for sb200_add_many (NULL: every step adds; BGV correction-factor balancing);
 *   d_outs[j]: [batch][max sizes[i]][L][n], in the ciphertexts' form.
 * The four NTT-form cases of multiply_plain are covered: coefficient-form plaintexts are lifted and transformed (sb200_plain_to_ntt)
 * and coefficient-form ciphertexts transformed into scratch, in chunks of terms, and each output gets one inverse transform.
 * The 128-bit sums are reduced once per window of terms: 256 when every prime of the level is below 2^60, fewer for larger
 * primes (64 at 61 bits); the fold's factors enter as one constant per term.  Errors, all before the first launch, in the
 * chain's order (multiply_plain's, then add_many's): count = 0 or outputs = 0, a plain count neither 1 nor batch, a size outside
 * 1..16, a mode outside 0..3, coefficient-form plaintexts in a CKKS context (SB200_E_INVALID_ARG); a NULL array, operand or
 * output, or (with a scaled step) h_factors (SB200_E_POINTER); an output slab overlapping an operand's slab or another output's
 * (SB200_E_INVALID_ARG).  The _host form stages the batch through the pipeline of every _host entry point, in chunks of
 * SB200_LIMIT_HOST_STAGE_BYTES per pipeline slot, and uploads each shared plaintext once per call. */
int sb200_multiply_plain_sum(sb200_context *ctx, size_t L, size_t batch, size_t count, size_t outputs, const size_t *sizes,
                             const uint64_t *const *d_cts, const size_t *plain_counts, const uint64_t *const *d_plains, int ct_is_ntt,
                             int plain_is_ntt, const int *modes, const uint64_t *h_factors, uint64_t *const *d_outs, void *stream);
int sb200_multiply_plain_sum_host(sb200_context *ctx, size_t L, size_t batch, size_t count, size_t outputs, const size_t *sizes,
                                  const uint64_t *const *h_cts, const size_t *plain_counts, const uint64_t *const *h_plains, int ct_is_ntt,
                                  int plain_is_ntt, const int *modes, const uint64_t *h_factors, uint64_t *const *h_outs);
/* Sums of ciphertext products: sum_i lhs_{j K + i} * rhs_i in one pass, with one size-3 result per sum (the lazy-relinearization
 * idiom: relinearize the sum once).  Member b of d_outs[j] (j < outputs = M) has the words of the chain t_i = sb200_multiply(member b
 * of d_lhs[j K + i], member b of d_rhs[i]) for i < count = K, then sb200_add_many(t_0 .. t_{K-1}, modes, h_factors)
 * (evaluator.cpp:352-841, :155-262), for any input words.
 *   d_lhs[j K + i], d_rhs[i]: [batch][2][L][n], in the scheme's form (NTT form for CKKS and BGV, coefficient form for BFV);
 *     a left operand may be the right one (a square);
 *   modes [K - 1] / h_factors [K - 1][2]: as for sb200_add_many (NULL: every step adds; BGV correction-factor balancing);
 *   d_outs[j]: [batch][3][L][n].
 * CKKS and BGV: one kernel pass reads every right operand once per tile of outputs and every left operand once; the 128-bit sums
 * are reduced once per window of terms (128 when every prime of the level is below 2^60, 32 at 61 bits) and the fold's factors
 * enter as one constant per term.  BFV: the chain's sb200_multiply into scratch, as many terms at a time as
 * SB200_LIMIT_SCRATCH_BYTES holds, each chunk folded into the output (no caller-side intermediates).  Errors, all before the first
 * launch, in the chain's order (multiply's, then add_many's): count = 0 or outputs = 0, a BFV level above sb200_multiply's limit,
 * a mode outside 0..3 (SB200_E_INVALID_ARG); a NULL array, operand or output, or (with a scaled step) h_factors (SB200_E_POINTER);
 * an output slab overlapping an operand's slab or another output's (SB200_E_INVALID_ARG).  The _host form stages the batch
 * through the pipeline of every _host entry point, in chunks of SB200_LIMIT_HOST_STAGE_BYTES per pipeline slot. */
int sb200_multiply_sum(sb200_context *ctx, size_t L, size_t batch, size_t count, size_t outputs, const uint64_t *const *d_lhs,
                       const uint64_t *const *d_rhs, const int *modes, const uint64_t *h_factors, uint64_t *const *d_outs, void *stream);
int sb200_multiply_sum_host(sb200_context *ctx, size_t L, size_t batch, size_t count, size_t outputs, const uint64_t *const *h_lhs,
                            const uint64_t *const *h_rhs, const int *modes, const uint64_t *h_factors, uint64_t *const *h_outs);
/* Evaluator::multiply_plain with ciphertext and plaintext both in NTT form (evaluator.cpp:1975-1994 -> multiply_plain_ntt
 * :2157-2195): every polynomial of the ciphertext times the plaintext, dyadic.  d_plain is [batch][L][n]: one NTT-form
 * plaintext per ciphertext, at the ciphertext's level (Plaintext::data() with parms_id == the ciphertext's).  May run in place. */
int sb200_multiply_plain(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *d_a, const uint64_t *d_plain,
                         uint64_t *d_out, void *stream);
/* ---- coefficient-form plaintexts (BFV / BGV): d_plain is [batch][n] words < plain_modulus, zero above coeff_count ----
 * Evaluator::transform_to_ntt_inplace(Plaintext&, parms_id) (evaluator.cpp:2197-2287): lift to the level with L primes
 * (words >= (t+1)/2 are negative, :2240-2272) and transform; d_out is [batch][L][n] */
int sb200_plain_to_ntt(sb200_context *ctx, size_t L, size_t batch, const uint64_t *d_plain, uint64_t *d_out, void *stream);
/* Evaluator::multiply_plain with such a plaintext: multiply_plain_normal (:2021-2155) for coefficient-form ciphertexts
 * (ct_is_ntt = 0, BFV), transform + multiply_plain_ntt (:1999-2004) for NTT-form ciphertexts (BGV).  May run in place. */
int sb200_multiply_plain_coeff(sb200_context *ctx, size_t L, size_t size, size_t batch, int ct_is_ntt, const uint64_t *d_a,
                               const uint64_t *d_plain, uint64_t *d_out, void *stream);
/* Evaluator::add_plain / sub_plain with such a plaintext: BFV adds round(q m / t) to c_0 (util/scalingvariant.cpp:70-160);
 * BGV adds NTT(lift(m * correction_factor mod t)) (:1838-1849), h_correction_factors = [batch] host words or NULL (= 1).
 * May run in place. */
int sb200_add_plain_coeff(sb200_context *ctx, size_t L, size_t size, size_t batch, int subtract, const uint64_t *d_a,
                          const uint64_t *d_plain, const uint64_t *h_correction_factors, uint64_t *d_out, void *stream);
/* BatchEncoder::encode / decode (batchencoder.cpp:84-330; SURVEY 8f rank 4): d_values [batch][n] matrix slots (< t,
 * row-major 2 x n/2) <-> coefficient-form plaintexts d_plain [batch][n].  Needs an NTT-friendly plain modulus
 * (t prime, t = 1 mod 2n: "encryption parameters are not valid for batching" otherwise).  No aliasing. */
int sb200_batch_encode(sb200_context *ctx, size_t batch, const uint64_t *d_values, uint64_t *d_plain, void *stream);
int sb200_batch_decode(sb200_context *ctx, size_t batch, const uint64_t *d_plain, uint64_t *d_values, void *stream);
/* ---- plaintext operations with plain_count plaintexts: plain_count = batch (one per ciphertext, as the three entry points above)
 * or 1 (one plaintext for the whole batch: a weight, a constant, a mask; it is read, and a coefficient-form one lifted and
 * transformed, once per stream call, and once per staging chunk in the _host forms, which upload it once per call).  Any other plain_count is SB200_E_INVALID_ARG.  The ciphertext may be updated in place
 * (d_out = d_a); a shared plaintext must not alias d_out (SB200_E_INVALID_ARG when d_out == d_plain).
 * sb200_multiply_plain with d_plain [plain_count][L][n] (evaluator.cpp:1975-2019, multiply_plain_ntt :2157-2195). */
int sb200_multiply_plain_n(sb200_context *ctx, size_t L, size_t size, size_t batch, size_t plain_count, const uint64_t *d_a,
                           const uint64_t *d_plain, uint64_t *d_out, void *stream);
/* sb200_multiply_plain_coeff with d_plain [plain_count][n] (multiply_plain_normal :2021-2155; transform_to_ntt_inplace(Plaintext&)
 * :2196-2287 then multiply_plain_ntt for NTT-form ciphertexts) */
int sb200_multiply_plain_coeff_n(sb200_context *ctx, size_t L, size_t size, size_t batch, size_t plain_count, int ct_is_ntt,
                                 const uint64_t *d_a, const uint64_t *d_plain, uint64_t *d_out, void *stream);
/* sb200_add_plain_coeff with d_plain [plain_count][n] (add_plain_inplace :1759-1866, sub_plain_inplace :1867-1974).
 * h_correction_factors: one BGV correction factor per plaintext ([plain_count] host words), or NULL (= 1); with a shared
 * plaintext it is the single correction factor of the batch. */
int sb200_add_plain_coeff_n(sb200_context *ctx, size_t L, size_t size, size_t batch, size_t plain_count, int subtract, const uint64_t *d_a,
                            const uint64_t *d_plain, const uint64_t *h_correction_factors, uint64_t *d_out, void *stream);
/* CKKS Evaluator::add_plain / sub_plain (add_plain_inplace :1759-1866, sub_plain_inplace :1867-1974): c_0 +/- the NTT-form
 * plaintext d_plain [plain_count][L][n] at the ciphertext's level (add_poly_coeffmod / sub_poly_coeffmod); c_1.. are copied
 * (in place: only c_0 is read and written).  The caller checks parms_id and scale as the reference does.  A BFV or BGV
 * context is SB200_E_INVALID_ARG ("BFV plain cannot be in NTT form" / "BGV plain cannot be in NTT form"). */
int sb200_add_plain_ntt(sb200_context *ctx, size_t L, size_t size, size_t batch, size_t plain_count, int subtract, const uint64_t *d_a,
                        const uint64_t *d_plain, uint64_t *d_out, void *stream);
/* Evaluator::relinearize_inplace, size 3 -> 2 (evaluator.cpp:1144-1199 + 2561-2867) */
int sb200_relinearize(sb200_context *ctx, size_t L, size_t batch, const uint64_t *d_in3,
                      const sb200_kswitch_key *relin_key, uint64_t *d_out2, void *stream);
/* multiply followed by relinearize_inplace in one call; the size-3 intermediate never reaches the caller */
int sb200_multiply_relinearize(sb200_context *ctx, size_t L, size_t batch, const uint64_t *d_a, const uint64_t *d_b,
                               const sb200_kswitch_key *relin_key, uint64_t *d_out2, void *stream);
/* Evaluator::rescale_to_next (CKKS; evaluator.cpp:1503-1541, rns.cpp:830-901): [2][L][n] -> [2][L-1][n] */
int sb200_rescale_to_next(sb200_context *ctx, size_t L, size_t batch, const uint64_t *d_in2, uint64_t *d_out2, void *stream);
/* Evaluator::mod_switch_to_next: BFV divide-and-round (rns.cpp:789-828); CKKS drops the last prime */
int sb200_mod_switch_to_next(sb200_context *ctx, size_t L, size_t batch, const uint64_t *d_in2, uint64_t *d_out2, void *stream);
/* the same two functions for ciphertexts of any size (the reference applies the step to every polynomial, evaluator.cpp:1263-1280):
 * d_in [batch][size][L][n] -> d_out [batch][size][L-1][n] */
int sb200_rescale_to_next_sized(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *d_in, uint64_t *d_out, void *stream);
int sb200_mod_switch_to_next_sized(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *d_in, uint64_t *d_out, void *stream);
/* one step of relinearize_internal's loop (evaluator.cpp:1176-1187) on ciphertexts of size >= 3: d_out = d_in with
 * (c_0, c_1) += switch_key(c_{size-1}, key); every other polynomial is copied, the size is unchanged (the caller drops
 * polynomials when the loop is done, as the reference's final resize does).  No aliasing. */
int sb200_relinearize_sized(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *d_in, const sb200_kswitch_key *key,
                            uint64_t *d_out, void *stream);
/* Evaluator::apply_galois (evaluator.cpp:2384-2502): automorphism x -> x^galois_elt on both polys + key switch.
 * rotate_rows / rotate_vector(step) = apply_galois(sb200_galois_elt_from_step(step)) with that element's key. */
int sb200_apply_galois(sb200_context *ctx, size_t L, size_t batch, const uint64_t *d_in2, uint32_t galois_elt,
                       const sb200_kswitch_key *galois_key, uint64_t *d_out2, void *stream);
/* d_out2 = d_addend2 + apply_galois(d_in2): Evaluator::apply_galois_inplace followed by Evaluator::add_inplace (evaluator.cpp:2384-2502,
 * :155-261) on a copy of the input, with the addition in the key switch's last pass (no copy, no add pass; the same words).  All
 * three slabs are [batch][2][L][n] in the scheme's form (BFV coefficient, CKKS / BGV NTT).  d_out2 may be d_addend2 (accumulate
 * rotated terms into one destination) and d_addend2 may be d_in2 (y + rotate(y)); d_out2 == d_in2 is rejected
 * (SB200_E_INVALID_ARG).  Other errors as sb200_apply_galois's, plus a NULL d_addend2 (SB200_E_POINTER); all before the first
 * launch, so the output is unchanged on error.  The _host form: h_a is the input, h_b the addend, h_out2 may be h_b. */
int sb200_apply_galois_add(sb200_context *ctx, size_t L, size_t batch, const uint64_t *d_in2, uint32_t galois_elt,
                           const sb200_kswitch_key *galois_key, const uint64_t *d_addend2, uint64_t *d_out2, void *stream);
int sb200_apply_galois_add_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *h_a, uint32_t galois_elt,
                                const sb200_kswitch_key *galois_key, const uint64_t *h_b, uint64_t *h_out2);
/* Sums of rotations: y_0 = in, y_{j+1} = y_j + apply_galois(y_j, galois_elts[j]) with galois_keys[j] (sb200_apply_galois_add with
 * the addend equal to the input), d_out2 = y_steps.  With the elements of steps s, 2s, 4s, ... this is the slot sum
 * x[i] + x[i + s] + ... of rotate_rows / rotate_vector; it replaces the reference's loop of Evaluator::rotate_rows_inplace /
 * rotate_vector_inplace (evaluator.h:1072-1251, evaluator.cpp:2504-2559) on a copy and add_inplace.  d_out2 may be d_in2; steps = 0 copies.  Each chunk of
 * the key-switching scratch (SB200_LIMIT_SCRATCH_BYTES, SB200_LIMIT_KS_CHUNK) runs every step, through one chunk-sized temporary.
 * Errors, all before the first launch (the output is unchanged): every element and key checked as by sb200_apply_galois; a NULL
 * galois_elts, galois_keys or entry (SB200_E_POINTER).  The _host form stages each chunk of SB200_LIMIT_HOST_STAGE_BYTES once for
 * the whole chain. */
int sb200_rotate_sum(sb200_context *ctx, size_t L, size_t batch, const uint64_t *d_in2, size_t steps, const uint32_t *galois_elts,
                     const sb200_kswitch_key *const *galois_keys, uint64_t *d_out2, void *stream);
int sb200_rotate_sum_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *h_in2, size_t steps, const uint32_t *galois_elts,
                          const sb200_kswitch_key *const *galois_keys, uint64_t *h_out2);
/* d_out2 = d_addend2 + d_plain * apply_galois(d_in2): Evaluator::apply_galois_inplace, Evaluator::multiply_plain_inplace and
 * Evaluator::add_inplace (evaluator.cpp:2384-2502, :1975-2020, :155-261) on a copy of the input.  d_plain holds plain_count (1 for the
 * whole batch, or batch) NTT-form plaintexts [L][n] at the input's level, in any 64-bit words (reduced as sb200_multiply_plain_n
 * reduces them).  CKKS / BGV: one key switch, with the plaintext product and the addition in its last pass (no copy, no product or
 * add pass; the same words).  BFV: the chain itself through one key-switching chunk of temporary (apply_galois, the ciphertext to NTT
 * form, the product, back, the addition), as the reference multiplies a coefficient-form ciphertext by an NTT-form plaintext.
 * Aliasing as sb200_apply_galois_add: d_out2 may be d_addend2, d_addend2 may be d_in2, d_out2 == d_in2 is SB200_E_INVALID_ARG.
 * Errors, all before the first launch in the chain's order (the output is unchanged): sb200_apply_galois's, then a plain_count other
 * than 1 or batch (SB200_E_INVALID_ARG); a NULL slab (SB200_E_POINTER); overlapping slabs (SB200_E_INVALID_ARG).  The _host form takes
 * host buffers of the same layouts; h_out2 may be h_addend2. */
int sb200_apply_galois_multiply_plain_add(sb200_context *ctx, size_t L, size_t batch, const uint64_t *d_in2, uint32_t galois_elt,
                                          const sb200_kswitch_key *galois_key, size_t plain_count, const uint64_t *d_plain,
                                          const uint64_t *d_addend2, uint64_t *d_out2, void *stream);
int sb200_apply_galois_multiply_plain_add_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *h_in2, uint32_t galois_elt,
                                               const sb200_kswitch_key *galois_key, size_t plain_count, const uint64_t *h_plain,
                                               const uint64_t *h_addend2, uint64_t *h_out2);
/* A plaintext matrix times an encrypted vector by diagonals: d_out2 = sum_i d_plains[i] * apply_galois(d_in2, galois_elts[i]), the
 * reference's chain  t = encrypted; rotate_rows / rotate_vector / apply_galois_inplace(t, ...); multiply_plain_inplace(t, plain_i);
 * i == 0 ? destination = t : add_inplace(destination, t)  (evaluator.cpp:2504-2559, :2384-2502, :1975-2020, :155-261) in one call.
 * Element 1 is no rotation (rotate_internal's step 0): no key switch, and its galois_keys entry may be NULL.  d_plains[i] holds
 * plain_counts[i] (1 or batch) plaintexts: NTT form [L][n] (plain_is_ntt != 0) or coefficient form [n] (BFV / BGV; each lifted and
 * transformed as Evaluator::transform_to_ntt_inplace does).  Shared and per-member plaintexts may be mixed in one call.
 * The identity terms go into one sb200_multiply_plain_sum pass that writes d_out2; each rotated term then accumulates into it.  CKKS
 * and BGV: each rotated term is one key switch with the product and the addition in its last pass, with no batch-sized temporary.
 * BFV: each rotated term is the chain itself through one key-switching chunk of temporary.  Each key-switching chunk
 * (SB200_LIMIT_SCRATCH_BYTES, SB200_LIMIT_KS_CHUNK) runs every term, so each key is read once per chunk and term, as by the chain.
 * d_out2 must not alias d_in2 (SB200_E_INVALID_ARG) and may not overlap any input.  Errors, all before the first launch in the chain's
 * order (the output is unchanged): every rotated term's element and key as sb200_apply_galois checks them, then every plain_counts[i]
 * (1 or batch) and coefficient-form plaintexts in CKKS, then count = 0 (all SB200_E_INVALID_ARG); a NULL array, plaintext slab or
 * rotated term's key (SB200_E_POINTER); overlapping slabs (SB200_E_INVALID_ARG).  The _host form stages each chunk of
 * SB200_LIMIT_HOST_STAGE_BYTES once, and each shared plaintext once per call. */
int sb200_diagonal_sum(sb200_context *ctx, size_t L, size_t batch, const uint64_t *d_in2, size_t count, const uint32_t *galois_elts,
                       const sb200_kswitch_key *const *galois_keys, const size_t *plain_counts, const uint64_t *const *d_plains,
                       int plain_is_ntt, uint64_t *d_out2, void *stream);
int sb200_diagonal_sum_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *h_in2, size_t count, const uint32_t *galois_elts,
                            const sb200_kswitch_key *const *galois_keys, const size_t *plain_counts, const uint64_t *const *h_plains,
                            int plain_is_ntt, uint64_t *h_out2);

/* ---- host-buffer variants: H2D copy, operation, D2H copy, synchronise (the plugin-facing end-to-end path) ---- */
int sb200_ntt_forward_host(sb200_context *ctx, size_t L, size_t size, size_t batch, uint64_t *h_data);
int sb200_ntt_inverse_host(sb200_context *ctx, size_t L, size_t size, size_t batch, uint64_t *h_data);
int sb200_multiply_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *h_a, const uint64_t *h_b, uint64_t *h_out3);
int sb200_multiply_sized_host(sb200_context *ctx, size_t L, size_t size_a, size_t size_b, size_t batch, const uint64_t *h_a,
                              const uint64_t *h_b, uint64_t *h_out);
int sb200_square_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *h_a, uint64_t *h_out3);
int sb200_add_host(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *h_a, const uint64_t *h_b, uint64_t *h_out);
int sb200_sub_host(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *h_a, const uint64_t *h_b, uint64_t *h_out);
int sb200_negate_host(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *h_a, uint64_t *h_out);
int sb200_add_many_host(sb200_context *ctx, size_t L, size_t batch, size_t count, const size_t *sizes, const uint64_t *const *h_operands,
                        const int *modes, const uint64_t *h_factors, uint64_t *h_out);
int sb200_multiply_plain_host(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *h_a, const uint64_t *h_plain,
                              uint64_t *h_out);
int sb200_plain_to_ntt_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *h_plain, uint64_t *h_out);
int sb200_multiply_plain_coeff_host(sb200_context *ctx, size_t L, size_t size, size_t batch, int ct_is_ntt, const uint64_t *h_a,
                                    const uint64_t *h_plain, uint64_t *h_out);
int sb200_add_plain_coeff_host(sb200_context *ctx, size_t L, size_t size, size_t batch, int subtract, const uint64_t *h_a,
                               const uint64_t *h_plain, const uint64_t *h_correction_factors, uint64_t *h_out);
int sb200_multiply_plain_n_host(sb200_context *ctx, size_t L, size_t size, size_t batch, size_t plain_count, const uint64_t *h_a,
                                const uint64_t *h_plain, uint64_t *h_out);
int sb200_multiply_plain_coeff_n_host(sb200_context *ctx, size_t L, size_t size, size_t batch, size_t plain_count, int ct_is_ntt,
                                      const uint64_t *h_a, const uint64_t *h_plain, uint64_t *h_out);
int sb200_add_plain_coeff_n_host(sb200_context *ctx, size_t L, size_t size, size_t batch, size_t plain_count, int subtract,
                                 const uint64_t *h_a, const uint64_t *h_plain, const uint64_t *h_correction_factors, uint64_t *h_out);
int sb200_add_plain_ntt_host(sb200_context *ctx, size_t L, size_t size, size_t batch, size_t plain_count, int subtract, const uint64_t *h_a,
                             const uint64_t *h_plain, uint64_t *h_out);
int sb200_batch_encode_host(sb200_context *ctx, size_t batch, const uint64_t *h_values, uint64_t *h_plain);
int sb200_batch_decode_host(sb200_context *ctx, size_t batch, const uint64_t *h_plain, uint64_t *h_values);
int sb200_relinearize_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *h_in3,
                           const sb200_kswitch_key *relin_key, uint64_t *h_out2);
int sb200_multiply_relinearize_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *h_a, const uint64_t *h_b,
                                    const sb200_kswitch_key *relin_key, uint64_t *h_out2);
int sb200_rescale_to_next_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *h_in2, uint64_t *h_out2);
int sb200_mod_switch_to_next_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *h_in2, uint64_t *h_out2);
int sb200_apply_galois_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *h_in2, uint32_t galois_elt,
                            const sb200_kswitch_key *galois_key, uint64_t *h_out2);
int sb200_rescale_to_next_sized_host(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *h_in, uint64_t *h_out);
int sb200_mod_switch_to_next_sized_host(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *h_in, uint64_t *h_out);
int sb200_relinearize_sized_host(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *h_in, const sb200_kswitch_key *key,
                                 uint64_t *h_out);

/* ---- wire format (SURVEY 8f rank 3): Ciphertext::save / load with compr_mode_type::none, straight between a byte
 * stream and a device slab (ciphertext.cpp:190-359, serialization.h:76-91, dynarray.h:662-690).  Seed-compressed ciphertexts
 * (Serializable<Ciphertext> of a symmetric-key encryption: c_1 replaced by the seed of the PRNG that made it) are expanded on
 * the device -- Ciphertext::expand_seed -> sample_poly_uniform on the PRNG the stream names, Blake2xbPRNG or Shake256PRNG
 * (ciphertext.cpp:118-150, util/rlwe.cpp:104-132, randomgen.cpp:163-227), bit for bit -- so a fresh ciphertext crosses PCIe with
 * half its bytes; one batch may mix both types and unseeded members.  zlib-compressed objects (compr_mode_type::zlib,
 * serialization.cpp:236-300, util/ztools.cpp) are inflated on the host with the system's zlib before they are parsed; zstd
 * streams stay with the reference: load rejects them. */
typedef struct sb200_ct_info
{
    uint64_t parms_id[4];         /* Ciphertext::parms_id() */
    uint64_t size;                /* polynomials */
    uint64_t poly_modulus_degree;
    uint64_t coeff_modulus_size;  /* L */
    uint64_t correction_factor;   /* BGV */
    double scale;                 /* CKKS */
    int32_t is_ntt_form;
    int32_t seeded;               /* 0: both polynomials are stored; otherwise only c_0 is, and c_1 is the output of the PRNG of this
                                     prng_type (randomgen.h:29-36: 1 = blake2xb, 2 = shake256) on the 64-byte seed at seed_offset */
    uint64_t data_offset;         /* byte offset of the first coefficient word in the stream */
    uint64_t data_words;          /* 64-bit words stored */
    uint64_t stream_bytes;        /* length of the serialized object (SEALHeader::size) */
    uint64_t seed_offset;         /* seeded streams: byte offset of the prng_seed_type (64 bytes); 0 otherwise */
    uint64_t compr_mode;          /* compr_mode_type of the stream (serialization.h:33-47): 0 none, 1 zlib; for a compressed stream the
                                     offsets above refer to the decompressed object and stream_bytes to the stream as given */
} sb200_ct_info;

/* EncryptionParameters::parms_id() of the level with L primes (L = k: the key level); encryptionparams.cpp:124-158 */
int sb200_get_parms_id(const sb200_context *ctx, size_t L, uint64_t out[4]);
/* Serialization::LoadHeader + the metadata half of Ciphertext::load_members; pure host, needs no context */
int sb200_ciphertext_inspect(const uint8_t *stream, size_t len, sb200_ct_info *info);
/* bytes Ciphertext::save(compr_mode_type::none) produces for size polynomials at the level with L primes */
size_t sb200_ciphertext_save_size(const sb200_context *ctx, size_t L, size_t size);
/* Ciphertext::load (validate != 0; also checks every residue < q_i like is_data_valid_for, valcheck.cpp) or unsafe_load
 * (validate == 0) of `batch` serialized ciphertexts of one shape into d_out [batch][size][L][n]; infos may be NULL.
 * The coefficient words are copied from the streams to the device directly; seeded streams (size 2) upload c_0 and expand
 * c_1 on the device. */
int sb200_ciphertext_load(sb200_context *ctx, size_t batch, const uint8_t *const *streams, const size_t *lens, size_t L, size_t size,
                          int validate, uint64_t *d_out, sb200_ct_info *infos, void *stream);
/* Ciphertext::save(compr_mode_type::none) of d_in [batch][size][L][n] into outs[b] (capacity >= sb200_ciphertext_save_size);
 * meta[b] supplies is_ntt_form / scale / correction_factor (parms_id, sizes and offsets are filled in here).  Returns after
 * the bytes are in place. */
int sb200_ciphertext_save(sb200_context *ctx, size_t batch, size_t L, size_t size, const uint64_t *d_in, const sb200_ct_info *meta,
                          uint8_t *const *outs, size_t capacity, void *stream);
/* Serializable<Ciphertext>::save(compr_mode_type::none) of fresh symmetric encryptions (what Encryptor::encrypt_symmetric /
 * encrypt_zero_symmetric return, ciphertext.cpp:190-247): per ciphertext c_0 and the 64-byte seed c_1 expands from, behind
 * UniformRandomGeneratorInfo's own header (randomgen.cpp:95-118).  d_in [batch][2][L][n]: only c_0 is read.  d_in must come from
 * sb200_encrypt_symmetric / sb200_encrypt_zero_symmetric_prng with save_seed != 0, h_public_seeds [batch][8] = the public seeds those
 * calls returned and prng = their ciphertext_prng (1 blake2xb, 2 shake256): BFV's c_0 differs with and without save_seed, and a
 * stream whose seed does not belong to its c_0 decrypts to garbage.  meta as for sb200_ciphertext_save.  Errors, all checked before
 * any byte is written: NULL d_in / meta / h_public_seeds / outs (SB200_E_POINTER), an invalid level or batch 0, a NULL outs[b],
 * capacity < sb200_ciphertext_save_seeded_size, a PRNG type other than 1 or 2 (SB200_E_INVALID_ARG).  Returns after the bytes are in
 * place. */
size_t sb200_ciphertext_save_seeded_size(const sb200_context *ctx, size_t L);
int sb200_ciphertext_save_seeded(sb200_context *ctx, size_t batch, size_t L, const uint64_t *d_in, const sb200_ct_info *meta,
                                 const uint64_t *h_public_seeds, int prng, uint8_t *const *outs, size_t capacity, void *stream);

/* ---- public-key encryption (SURVEY 8f rank 4): Encryptor(context, public_key) and Encryptor::encrypt_zero(parms_id, destination)
 * (encryptor.cpp:88-174 -> util::encrypt_zero_asymmetric, util/rlwe.cpp:184-276) for a batch.
 * h_public_key = PublicKey::data().data(): [2][k][n] words, NTT form at the key level (range-checked).
 * d_out = [batch][2][L][n] at the level with L primes (L == k: the key level): NTT form for CKKS / BGV, coefficient form for BFV,
 * scale 1, correction factor 1.  As in the reference the sample is drawn one level above (L + 1 primes) and divided down by that
 * level's last prime.  Per ciphertext ONE PRNG (Blake2xb of a 64-byte seed) yields the ternary polynomial u and the two noise
 * polynomials exactly as the reference draws them (u through std::uniform_int_distribution as libstdc++ >= 11 implements it),
 * so the same seed gives the reference's ciphertext bit for bit.  h_seeds = [batch][8] words or NULL = fresh seeds from the OS
 * entropy source.  Synchronises the stream.  sb200_encrypt_asymmetric adds the plaintext: Encryptor::encrypt. */
int sb200_public_key_create(sb200_context *ctx, const uint64_t *h_public_key, sb200_public_key **out);
int sb200_public_key_destroy(sb200_public_key *key);
int sb200_encrypt_zero_asymmetric(sb200_context *ctx, sb200_public_key *key, size_t L, size_t batch, const uint64_t *h_seeds,
                                  uint64_t *d_out, void *stream);
/* the same with the PRNG type of parms.random_generator(), which draws u and both noise polynomials (util/rlwe.cpp:224):
 * prng = SEAL's prng_type, 1 = blake2xb (sb200_encrypt_zero_asymmetric), 2 = shake256 (Shake256PRNG, randomgen.cpp:216-227:
 * buffer b = SHAKE256(seed || b, 4096 bytes)); any other value returns SB200_E_INVALID_ARG. */
int sb200_encrypt_zero_asymmetric_prng(sb200_context *ctx, sb200_public_key *key, size_t L, size_t batch, int prng, const uint64_t *h_seeds,
                                       uint64_t *d_out, void *stream);
/* Encryptor(context, public_key)::encrypt(plain, destination) (encryptor.cpp:176-340) for a batch, one plaintext per ciphertext:
 * sb200_encrypt_zero_asymmetric_prng, then the plaintexts added to c_0 in one pass over the batch (BGV: lift and transform, then
 * the add).  d_plain = CKKS: [batch][L][n] NTT form at the level with L primes; BFV / BGV: [batch][n] words < t (zero above the
 * plaintext's coeff_count), and L must be the first level (k - 1 primes, or 1 when k = 1): anything else is SB200_E_INVALID_ARG.
 * The result is the reference's word for word under the same seeds (its parms_id: the plaintext's for CKKS, first_parms_id for
 * BFV / BGV; scale: the plaintext's for CKKS).  d_plain NULL: SB200_E_POINTER; d_plain == d_out: SB200_E_INVALID_ARG.  Every
 * check runs before the first launch.  Synchronises the stream. */
int sb200_encrypt_asymmetric(sb200_context *ctx, sb200_public_key *key, size_t L, size_t batch, const uint64_t *d_plain, int prng,
                             const uint64_t *h_seeds, uint64_t *d_out, void *stream);

/* ---- CKKSEncoder (SURVEY 8f: the data format either side of the path): CKKSEncoder::encode(values, parms_id, scale, plain) and
 * CKKSEncoder::decode(plain, values) (ckks.h:455-807) for a batch.  values = doubles: [batch][count] complex numbers as (re, im)
 * pairs when is_complex, else [batch][count] reals; count <= n/2, missing slots are zero.  plain = [batch][L][n] NTT form at the
 * level with L primes (Plaintext::data() of each plaintext; its parms_id is sb200_get_parms_id(L), its scale the scale given).
 * Bit-exact with the reference: the double-precision transform performs the reference's operations in the reference's order.
 * Decode can produce non-finite slots (a plaintext whose coefficients exceed the double range after scaling, e.g. one that does not
 * decrypt to a small value): each slot has the reference's class (finite, +inf, -inf or NaN), and every slot the reference does
 * not make NaN has its bits.  A NaN's sign and payload are not specified (IEEE 754 leaves them to the implementation).
 * Errors as the reference throws them (SB200_E_INVALID_ARG): "scale out of bounds", "values must be finite", "encoded values are
 * too large" (the plaintext buffer is left unspecified), "unsupported scheme" for a non-CKKS context.
 * decode writes [batch][n/2] complex numbers as (re, im) pairs; `scale` is Plaintext::scale().  The encode entry points
 * synchronise the stream once (the magnitude check precedes the reduction). */
int sb200_ckks_encode(sb200_context *ctx, size_t L, size_t batch, const double *d_values, size_t count, int is_complex, double scale,
                      uint64_t *d_plain, void *stream);
int sb200_ckks_decode(sb200_context *ctx, size_t L, size_t batch, const uint64_t *d_plain, double scale, double *d_values, void *stream);
int sb200_ckks_encode_host(sb200_context *ctx, size_t L, size_t batch, const double *h_values, size_t count, int is_complex, double scale,
                           uint64_t *h_plain);
int sb200_ckks_decode_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *h_plain, double scale, double *h_values);

/* CKKSEncoder::encode of one scalar per plaintext (ckks.h:272-377) for a batch: values = [batch] doubles (SB200_CKKS_SCALAR_REAL,
 * encode(double value, parms_id, scale, plain), ckks.cpp:75-230), [batch] (re, im) pairs of doubles (SB200_CKKS_SCALAR_COMPLEX,
 * encode(std::complex<double>, ...), ckks.h:794-800: the vector encode of n/2 copies) or [batch] int64_t (SB200_CKKS_SCALAR_INT64,
 * encode(std::int64_t value, parms_id, plain), ckks.cpp:232-287; scale is ignored, the plaintext's scale is 1.0).  plain =
 * [batch][L][n] NTT form at the level with L primes, word for word the reference's.  Real and int64 plaintexts are constant
 * polynomials, written on the device by one fill kernel; a negative int64 v is reduced as the reference reduces it,
 * (uint64_t)v + q_j, which is (2^64 - |v|) mod q_j and not -|v| mod q_j when |v| > q_j.
 * Errors (SB200_E_INVALID_ARG), checked before any launch that writes plain, on the first failing plaintext in batch order:
 * a kind outside 0..2; "unsupported scheme" for a non-CKKS context; "parms_id is not valid for encryption parameters" for L outside
 * 1..k; batch 0.  Real: "scale out of bounds" (!isfinite(scale), scale <= 0 or (int)log2(scale) >= the level's total bit count:
 * unlike the vector encode, a subnormal scale and (int)log2(scale) = total bits - 1 are accepted), "value must be finite",
 * "encoded value is too large" (value * scale not finite, or its bit count + 1 at or above the total bit count).  Int64: "encoded
 * value is too large" (significant bits of |v| + 2 at or above the total bit count, |INT64_MIN| taken as 2^63).  Complex: the
 * vector encode's checks and messages ("scale out of bounds", "values must be finite", "encoded values are too large").  NULL
 * values or plain: SB200_E_POINTER.  Real and int64 copy the values to the host and synchronise the stream once; complex
 * synchronises it as sb200_ckks_encode does. */
#define SB200_CKKS_SCALAR_REAL 0
#define SB200_CKKS_SCALAR_COMPLEX 1
#define SB200_CKKS_SCALAR_INT64 2
int sb200_ckks_encode_scalar(sb200_context *ctx, size_t L, size_t batch, int kind, const void *d_values, double scale, uint64_t *d_plain,
                             void *stream);
int sb200_ckks_encode_scalar_host(sb200_context *ctx, size_t L, size_t batch, int kind, const void *h_values, double scale,
                                  uint64_t *h_plain);

/* ---- decryption (SURVEY 8f rank 4): Decryptor(context, secret_key) and Decryptor::decrypt (decryptor.cpp:62-197) ------
 * h_secret_key = SecretKey::data().data(): [k][n] words, NTT form at the key level.  Powers of the key for ciphertexts
 * of size > 2 are built on the device on first use (compute_secret_key_array, :199-310). */
int sb200_secret_key_create(sb200_context *ctx, const uint64_t *h_secret_key, sb200_secret_key **out);
int sb200_secret_key_destroy(sb200_secret_key *key);
/* Encryptor::encrypt_zero_symmetric(parms_id, destination) for a batch (encryptor.cpp:168-173 -> util/rlwe.cpp:264-408): fresh
 * encryptions of zero under the secret key at the level with L primes, d_out = [batch][2][L][n] (NTT form for CKKS / BGV,
 * coefficient form for BFV; scale 1, correction factor 1).  Per ciphertext ONE bootstrap PRNG (Blake2xb of a 64-byte seed) yields
 * the public seed c_1 is sampled from and the centred binomial noise, exactly as the reference draws them, so that the same
 * bootstrap seed gives the reference's ciphertext bit for bit.  h_bootstrap_seeds = [batch][8] words, or NULL = fresh seeds from
 * the OS entropy source (what the reference's default UniformRandomGeneratorFactory does, randomgen.cpp:34-50).
 * save_seed != 0 selects the Serializable<Ciphertext> variant (differs for BFV only: which domain c_1 is sampled in);
 * h_public_seeds = NULL or [batch][8]: the seed each c_1 expands from (what a seeded stream carries instead of c_1: send
 * (c_0, seed) over the wire and let the receiver expand, sb200_ciphertext_load).  sb200_encrypt_symmetric below adds the plaintext
 * as c_0 is written: Encryptor::encrypt_symmetric. */
int sb200_encrypt_zero_symmetric(sb200_context *ctx, sb200_secret_key *key, size_t L, size_t batch, const uint64_t *h_bootstrap_seeds,
                                 int save_seed, uint64_t *d_out, uint64_t *h_public_seeds, void *stream);
/* the same with both PRNG types given (SEAL's prng_type: 1 = blake2xb, 2 = shake256; any other value returns SB200_E_INVALID_ARG).
 * bootstrap_prng = the type of parms.random_generator(), which draws the public seed and the noise (util/rlwe.cpp:322);
 * ciphertext_prng = the type c_1 is expanded with, UniformRandomGeneratorFactory::DefaultFactory() (util/rlwe.cpp:329), i.e. the
 * SEAL_DEFAULT_PRNG the reference was built with; a seeded stream of the result names this type.
 * sb200_encrypt_zero_symmetric = this with 1, 1. */
int sb200_encrypt_zero_symmetric_prng(sb200_context *ctx, sb200_secret_key *key, size_t L, size_t batch, int bootstrap_prng,
                                      int ciphertext_prng, const uint64_t *h_bootstrap_seeds, int save_seed, uint64_t *d_out,
                                      uint64_t *h_public_seeds, void *stream);
/* Encryptor::encrypt_symmetric(plain, destination) (encryptor.cpp:176-340) for a batch, one plaintext per ciphertext: the
 * plaintext term is added inside the kernels that write c_0 (no extra pass).  Seeds, PRNG types, save_seed and h_public_seeds as
 * for sb200_encrypt_zero_symmetric_prng; d_plain, levels and errors as for sb200_encrypt_asymmetric.  Both encryption paths cut
 * the batch into chunks by SB200_LIMIT_SCRATCH_BYTES; the words do not depend on it. */
int sb200_encrypt_symmetric(sb200_context *ctx, sb200_secret_key *key, size_t L, size_t batch, const uint64_t *d_plain, int bootstrap_prng,
                            int ciphertext_prng, const uint64_t *h_bootstrap_seeds, int save_seed, uint64_t *d_out, uint64_t *h_public_seeds,
                            void *stream);
/* ---- key generation from a given secret key: KeyGenerator(context, secret_key) (keygenerator.cpp:35-52) ----------------------
 * The secret key itself is not sampled here: it comes from seal::KeyGenerator or is loaded.  Every key below is made of key-level
 * encryptions of zero under `key` in NTT form (for every scheme, BFV included; BGV multiplies the noise by t), each drawn from one
 * bootstrap PRNG of type bootstrap_prng (parms.random_generator()) whose c_1 expands with ciphertext_prng, as in
 * sb200_encrypt_zero_symmetric_prng; a bootstrap seed of the reference's factory gives its key bit for bit.  Seeds NULL = fresh
 * seeds from the OS entropy source.  Both calls are synchronous (default stream) and wipe the noise and PRNG streams they used.
 * Errors: a key of another context or a PRNG type other than 1 or 2: SB200_E_INVALID_ARG; both outputs NULL: SB200_E_POINTER. */
/* KeyGenerator::create_relin_keys (galois_elt = 0) / one element of create_galois_keys (keygenerator.cpp:122-226, 327-360)
 * for the secret key `key`: digits = k - 1 key-level encryptions of zero (NTT form, every scheme) with (q_special mod q_j) s'_j
 * added to row j of c_0, s' = s^2 or s under the Galois automorphism.  h_bootstrap_seeds = [k-1][8] (one per digit, in the
 * reference's draw order) or NULL.  Outputs, either may be NULL but not both: h_key = [k-1][2][k][n] (KSwitchKeys::data()[index]
 * words) and *out = a device key handle, as sb200_kswitch_key_create would make from those words, without the host round trip.
 * k < 2: SB200_E_LOGIC "keyswitching is not supported by the context"; an even galois_elt or one >= 2n: SB200_E_INVALID_ARG
 * "Galois element is not valid".  The digits are generated in chunks that fit SB200_LIMIT_SCRATCH_BYTES; the words do not
 * depend on it. */
int sb200_kswitch_key_generate(sb200_context *ctx, sb200_secret_key *key, uint32_t galois_elt, int bootstrap_prng,
                               int ciphertext_prng, const uint64_t *h_bootstrap_seeds, uint64_t *h_key, sb200_kswitch_key **out);
/* KeyGenerator::create_public_key (keygenerator.cpp:96-120): h_public_key = [2][k][n] and / or *out = an Encryptor key handle;
 * h_bootstrap_seed = [8] or NULL */
int sb200_public_key_generate(sb200_context *ctx, sb200_secret_key *key, int bootstrap_prng, int ciphertext_prng,
                              const uint64_t *h_bootstrap_seed, uint64_t *h_public_key, sb200_public_key **out);
/* ---- seed-compressed keys: what KeyGenerator's Serializable<...> overloads save with compr_mode_type::none, byte for byte under the
 * same bootstrap seeds.  Every member is a seeded ciphertext stream (see sb200_ciphertext_save_seeded) at the key level, NTT form,
 * scale 1, correction factor 1, whose seed expands with ciphertext_prng.  c_1 never leaves the device.
 * KeyGenerator::create_public_key() (keygenerator.cpp:96-120): `capacity` >= sb200_ciphertext_save_seeded_size(ctx, k) bytes at out;
 * *handle (may be NULL) receives the Encryptor key handle of the same key. */
int sb200_public_key_generate_seeded(sb200_context *ctx, sb200_secret_key *key, int bootstrap_prng, int ciphertext_prng,
                                     const uint64_t *h_bootstrap_seed, uint8_t *out, size_t capacity, sb200_public_key **handle);
/* KeyGenerator::create_relin_keys() (galois_elts = {0}, count 1: a RelinKeys object of one slot) or create_galois_keys(galois_elts)
 * (a GaloisKeys object of n slots; the elements in the order given, duplicates skipped as has_key does, empty slots a bare dim2 = 0),
 * kswitchkeys.cpp:42-86.  h_bootstrap_seeds = [distinct elements][k-1][8] in draw order, or NULL = fresh seeds from the OS entropy
 * source.  The digits are generated in the chunks of sb200_kswitch_key_generate; each chunk's c_0 rows are copied from the device to
 * their place in `out` through the context's page-locked staging while the next chunk is generated, and the bytes do not depend on
 * SB200_LIMIT_SCRATCH_BYTES.  The _size function returns the stream's length (0 for arguments the generator rejects).  Errors, all
 * checked before anything is generated: k < 2 (SB200_E_LOGIC "keyswitching is not supported by the context"); an even element or one
 * >= 2n, 0 mixed with Galois elements, a key of another context, a PRNG type other than 1 or 2, capacity below the _size
 * (SB200_E_INVALID_ARG); NULL key, galois_elts or out (SB200_E_POINTER).  Synchronous (default stream). */
size_t sb200_kswitch_keys_save_seeded_size(const sb200_context *ctx, const uint32_t *galois_elts, size_t count);
int sb200_kswitch_keys_generate_seeded(sb200_context *ctx, sb200_secret_key *key, const uint32_t *galois_elts, size_t count, int bootstrap_prng,
                                       int ciphertext_prng, const uint64_t *h_bootstrap_seeds, uint8_t *out, size_t capacity);
/* d_ct [batch][size][L][n] in the scheme's own form -> d_plain: CKKS [batch][L][n] (NTT form, same level; the caller keeps
 * scale and parms_id); BFV [batch][n] coefficients mod t (dot product + decrypt_scale_and_round, rns.cpp:1133-1191);
 * BGV [batch][n] (dot product, INTT, exact base conversion rns.cpp:466-539, times the inverse of the ciphertext's
 * correction factor: h_correction_factors = [batch] host words or NULL for 1). */
int sb200_decrypt(sb200_context *ctx, sb200_secret_key *key, size_t L, size_t size, size_t batch, const uint64_t *d_ct,
                  const uint64_t *h_correction_factors, uint64_t *d_plain, void *stream);
int sb200_decrypt_host(sb200_context *ctx, sb200_secret_key *key, size_t L, size_t size, size_t batch, const uint64_t *h_ct,
                       const uint64_t *h_correction_factors, uint64_t *h_plain);
/* Decryptor::invariant_noise_budget (decryptor.cpp:409-486) for a batch: d_ct [batch][size][L][n], BFV in coefficient form, BGV in
 * NTT form -> d_budgets [batch] ints, max(0, bits(Q) - bits(||t c(s) mod Q||) - 1) for BFV, the same without the factor t for BGV,
 * each equal to the reference's.  The phase is composed modulo Q exactly on the device and reduced to one int per ciphertext
 * there; nothing but the budgets leaves the GPU, and the stream entry point does not synchronise with the host.  Sizes 2..16
 * and levels of at most 60 primes, as sb200_decrypt (levels of 61-64 primes are rejected with SB200_E_INVALID_ARG for now, like
 * decryption); a CKKS context gives SB200_E_LOGIC ("unsupported scheme", the reference has no noise budget for CKKS).  The
 * scratch arena (and, for the host entry point, the output staging) is wiped afterwards, as after a decryption. */
int sb200_invariant_noise_budget(sb200_context *ctx, sb200_secret_key *key, size_t L, size_t size, size_t batch, const uint64_t *d_ct,
                                 int *d_budgets, void *stream);
int sb200_invariant_noise_budget_host(sb200_context *ctx, sb200_secret_key *key, size_t L, size_t size, size_t batch, const uint64_t *h_ct,
                                      int *h_budgets);

/* ---- multi-device dispatch (SURVEY 8e): one context per CUDA device of the box, one host thread per device -----------
 * A batch of independent ciphertexts is cut into contiguous slices, slice i goes to device i through that device's own
 * context (tables and keys replicated, no data-path collective); every call returns when all slices are back in the host
 * buffers.  The reference has no counterpart (it is single-threaded per Evaluator call); this is the C++ side of what
 * bench.py does with one process per GPU.  devices == NULL: every visible device. */
typedef struct sb200_group sb200_group;
typedef struct sb200_group_key sb200_group_key; /* one key-switching key replicated on every device of the group */
int sb200_group_create(int scheme, size_t poly_modulus_degree, const uint64_t *coeff_modulus, size_t k, uint64_t plain_modulus,
                       const int *devices, size_t device_count, sb200_group **out);
int sb200_group_destroy(sb200_group *group);
size_t sb200_group_size(const sb200_group *group);
sb200_context *sb200_group_context(sb200_group *group, size_t i); /* the context of device slot i (owned by the group) */
/* first ciphertext and count of slot i's slice of a batch (the same rule for every call; seal_b200/shard.py mirrors it) */
int sb200_group_slice(const sb200_group *group, size_t batch, size_t i, size_t *first, size_t *count);
int sb200_group_kswitch_key_create(sb200_group *group, const uint64_t *h_key, size_t digits, sb200_group_key **out);
int sb200_group_kswitch_key_destroy(sb200_group_key *key);
int sb200_group_multiply_relinearize_host(sb200_group *group, size_t L, size_t batch, const uint64_t *h_a, const uint64_t *h_b,
                                          const sb200_group_key *relin_key, uint64_t *h_out2);
int sb200_group_relinearize_host(sb200_group *group, size_t L, size_t batch, const uint64_t *h_in3, const sb200_group_key *relin_key,
                                 uint64_t *h_out2);
int sb200_group_apply_galois_host(sb200_group *group, size_t L, size_t batch, const uint64_t *h_in2, uint32_t galois_elt,
                                  const sb200_group_key *galois_key, uint64_t *h_out2);
int sb200_group_multiply_host(sb200_group *group, size_t L, size_t batch, const uint64_t *h_a, const uint64_t *h_b, uint64_t *h_out3);
int sb200_group_rescale_to_next_host(sb200_group *group, size_t L, size_t batch, const uint64_t *h_in2, uint64_t *h_out2);
int sb200_group_mod_switch_to_next_host(sb200_group *group, size_t L, size_t batch, const uint64_t *h_in2, uint64_t *h_out2);
int sb200_group_ntt_forward_host(sb200_group *group, size_t L, size_t size, size_t batch, uint64_t *h_data);
int sb200_group_ntt_inverse_host(sb200_group *group, size_t L, size_t size, size_t batch, uint64_t *h_data);

#ifdef __cplusplus
}
#endif
#endif
