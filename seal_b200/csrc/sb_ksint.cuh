// seal_b200/csrc/sb_ksint.cuh -- key switching through an exact integer convolution (declarations; kernels in sb_ksint.cu).
//
// switch_key_inplace (evaluator.cpp:2664-2755) forms, for every output prime q_I, sum_J NTT_I(d_J mod q_I) (.) K_JI mod q_I: L
// 64-bit transforms per output prime.  The same residues are the NTT_I image of the INTEGER polynomial
//     c_I = sum_J d_J * k_JI   (negacyclic; d_J in [0, q_J) the digits, k_JI = INTT_I(K_JI) in [0, q_I))
// reduced mod q_I, and |c_I| < L n q_J q_I (132 bits at n = 2^16, 32 primes of 55 bits).  This path computes c_I exactly:
//   1. digits -> S auxiliary 29-bit NTT primes p_t (S = 5), forward transforms with 32-bit butterflies (shared by all I);
//   2. out[I][c][t] = sum_J dhat[J][t] (.) khat[J][c][I][t]   (32 x 32 -> 64-bit multiply-accumulates, no reduction in the loop);
//   3. inverse 32-bit transforms;
//   4. per coefficient: CRT reconstruction of c_I + P/2 from its S residues, reduction mod q_I, and the mod-down by the special
//      prime (evaluator.cpp:2762-2864) in coefficient form;
//   5. one 64-bit forward transform per output row (CKKS / BGV), fused with the addition into the ciphertext.
// A 32-bit Shoup butterfly is 1 wide + 2 narrow multiplies (8.3 multiply-pipe clocks per warp) against 5 wide + 4 narrow (28.8) for
// the 64-bit one, and the L (L+1) digit transforms become S L forward + 2 S (L+1) inverse small ones.  Results are word-identical
// to the reference (same residues mod q_I), which the parity tests check against the reference itself.
#pragma once
#include "sb_mem.cuh"
#include "sb_src.cuh"
#include <cstddef>
#include <cstdint>

namespace sb
{
    struct Context;
    struct KSwitchKey;

    constexpr int kKsMaxS = 8;

    struct KsIntParams
    {
        int S = 0, r = 0, logn = 0;
        uint32_t p[kKsMaxS] = {}, mu[kKsMaxS] = {}, c2[kKsMaxS] = {}, inv60[kKsMaxS] = {}; // inv60 = floor(2^60 / p)
        uint2 red[kKsMaxS] = {}, c1[kKsMaxS] = {};
    };

    struct KsInt
    {
        bool ready = false;
        bool mac_mma = true;   // product kernel on the INT8 tensor cores (env SB200_KS_MAC_MMA)
        bool mac_tile = true;  // product kernel with the key tile in shared memory (env SB200_KS_MAC_TILE)
        bool fuse_crt = true;  // outer inverse stages inside the reconstruction kernel (env SB200_KS_FUSE_CRT)
        bool fuse_ntt = true;  // entry and exit inside the column passes of the 64-bit transforms (env SB200_KS_FUSE_NTT)
        size_t max_digits = 0; // sbh::KsIntHost::max_digits (64 at n = 4096)
        KsIntParams prm;
        DevBuf<uint2> d_fwd_outer, d_inv_outer; // [S][2^r]
        DevBuf<uint2> d_fwd_local, d_inv_local; // [S][2^r][4096]
        DevBuf<u64> d_punct, d_neg;             // [k][S]
        DevBuf<u64> d_half_mod;                 // [k]: floor(q_special / 2) mod q_i
    };

    // per-ciphertext scratch of the integer path (bytes): digits' transforms, accumulated products, coefficient-form result
    struct KsIntScratch
    {
        uint32_t *Dh = nullptr;  // [S][L][Bpad][n]
        uint32_t *Acc = nullptr; // [B][2][L+1][S][n], output prime index 0 = the special prime, i + 1 = data prime i
        u64 *R = nullptr;        // [B][2][L][n] (aliases Dh: the transformed digits are dead once the products exist)
    };
    size_t ksint_bytes_per_ct(const Context &c, size_t L);
    size_t ksint_bytes_fixed(const Context &c, size_t L); // padding of the digit slab, once per chunk
    KsIntScratch ksint_carve(const Context &c, size_t L, size_t B, void *base);

    void ksint_init(Context &c);
    // khat[t][J][c][ki][n] from the uploaded key [digits][2][k][n]
    void ksint_prepare_key(Context &c, KSwitchKey &key, cudaStream_t st);
    // target (CKKS / BGV: NTT form, BFV: coefficient form) -> out = base + key-switched polynomials (+ the addend of a BaseAddSrc;
    // times the plaintext, then + the addend, of a BasePlainSrc: CKKS / BGV only).  D: [B][L][n] scratch of the target's inverse
    // transforms.  See key_switch_chunk.  Instantiated for BaseSrc, BaseAddSrc, BasePlainSrc<false> and BasePlainSrc<true>
    template <class Base>
    void ksint_core(Context &c, size_t L, size_t B, const KsIntScratch &s, Src target, u64 *D, const KSwitchKey &key, Base base,
                    u64 *out, long long o_bs, cudaStream_t st);
    // arithmetic ceilings of this path measured in process: kind 0 = 32-bit forward butterflies, 1 = inverse, 2 = multiply-accumulates
    double ksint_selftest_rate(Context &c, int kind, cudaStream_t st);
    // parity-test access to the transforms: forward h_rows [rows][n] u64 -> h_io [S][rows][n]; inverse: h_io [rows][S][n] in place
    void ksint_selftest_transform(Context &c, bool inverse, const u64 *h_rows, size_t rows, uint32_t *h_io);
    // parity-test access to the product step alone: h_Dh [S][L][B][n], h_key [S][L][2][L+1][n] (canonical words) ->
    // h_Acc [B][2][L+1][S][n]; mma = 0: the integer-pipe kernels, 1: the tensor-core kernel where it applies (L <= 32, B >= 16).
    // Returns the kernel that ran: 0 register tile, 1 key tile, 2 tensor cores
    int ksint_selftest_product(Context &c, const uint32_t *h_Dh, const uint32_t *h_key, int L, int B, uint32_t *h_Acc, int mma);
} // namespace sb
