// seal_b200/csrc/sb_host.hpp -- host-side precomputation (C++17, no CUDA, no reference code).
//
// Builds, from (scheme, n, coeff_modulus, plain_modulus) alone, every table the kernels need:
//   * per prime: Barrett ratio (reference Modulus::const_ratio, modulus.cpp:86-99), minimal primitive 2n-th root
//     (numth.cpp:386-412), forward / inverse twiddles with Shoup quotients (NTTTables::initialize, ntt.cpp:241-300)
//   * per level: mod-down / rescale constants (RNSTool::initialize, rns.cpp:767-776) and, for BFV, the BEHZ auxiliary
//     base and conversion matrices (rns.cpp:578-787)
//   * Galois permutation tables (GaloisTool::generate_table_ntt, galois.cpp:18-51)
// so the product does not depend on a SEALContext at run time.
#pragma once
#include <cstddef>
#include <cstdint>
#include <stdexcept>
#include <vector>

namespace sbh
{
    using u64 = unsigned long long; // same type the device code uses (64-bit on every supported ABI)
    using u128 = unsigned __int128;

    inline u64 mulmod(u64 a, u64 b, u64 q) { return static_cast<u64>((static_cast<u128>(a) * b) % q); }
    u64 powmod(u64 a, u64 e, u64 q);
    bool invmod(u64 a, u64 m, u64 &out); // any modulus coprime to a
    bool is_prime(u64 v);                // deterministic for 64-bit inputs
    std::vector<u64> get_primes(u64 factor, int bit_size, std::size_t count); // numth.cpp:278-311
    std::vector<u64> coeff_modulus_create(std::size_t n, const std::vector<int> &bits); // modulus.cpp:144-184
    bool minimal_primitive_root(u64 degree, u64 q, u64 &root);
    inline u64 shoup(u64 w, u64 q) { return static_cast<u64>((static_cast<u128>(w) << 64) / q); }
    inline int ilog2(std::size_t n)
    {
        int l = 0;
        while ((std::size_t(1) << l) < n)
            l++;
        return l;
    }
    inline u64 reverse_bits(u64 x, int bits)
    {
        u64 r = 0;
        for (int i = 0; i < bits; i++)
            r |= ((x >> i) & 1) << (bits - 1 - i);
        return r;
    }
    int product_bit_count(const u64 *q, std::size_t count);

    // CKKSEncoder tables (ckks.cpp:33-73 + util/croots.cpp:16-70): the powers of the primitive 2n-th complex root in the order
    // the transforms consume them, as (re, im) pairs; computed exactly as the reference does (std::polar on one eighth of the
    // circle, the rest by symmetry) so that the device transforms reproduce its doubles bit for bit
    struct CkksTables
    {
        std::vector<double> roots, inv_roots; // [n][2]; entry 0 unused
    };
    CkksTables ckks_tables(std::size_t n);
    // what CKKSEncoder::decode needs of a level with L primes: Q = prod q_j, (Q + 1) / 2 (ContextData::upper_half_threshold,
    // context.cpp:406-412), the punctured products Q / q_j and their inverses mod q_j (RNSBase::initialize, rns.cpp:149-193)

    struct TwPair
    {
        u64 w, wq;
    };

    struct CkksLevelHost
    {
        int total_bits = 0;
        std::vector<u64> Q, threshold, punctured; // L, L, L * L words (little endian)
        std::vector<TwPair> inv_punctured;        // L
    };
    CkksLevelHost ckks_level(const u64 *q, std::size_t L);

    struct PrimeTables
    {
        u64 q = 0, root = 0;
        u64 ratio_lo = 0, ratio_hi = 0;
        TwPair inv_n{}, inv_n_w{};
        // reference order (NTTTables::get_from_root_powers / get_from_inv_root_powers)
        std::vector<TwPair> root_powers, inv_root_powers;
        // device order: fwd[m+i] = root_powers[m+i]; inv[m+i] = inv_root_powers[n - 2m + 1 + i]
        std::vector<TwPair> fwd, inv;
        void build(std::size_t n, u64 modulus);
    };

    // BEHZ per-level constants (rns.cpp:578-787); all "pair" arrays are {value, Shoup quotient}
    struct BehzLevel
    {
        std::size_t L = 0, nB = 0, nBsk = 0;
        std::vector<u64> B, Bsk;      // Bsk = B + {m_sk}
        u64 m_sk = 0;
        std::vector<TwPair> inv_punc_q;      // [(q/q_i)^-1]_{q_i}                 [L]
        std::vector<u64> q_to_Bsk;           // (q/q_i) mod Bsk_s                  [nBsk][L]
        std::vector<u64> q_to_mtilde;        // (q/q_i) mod 2^32                   [L]
        std::vector<TwPair> mtilde_mod_q;    // 2^32 mod q_i                       [L]
        u64 neg_inv_q_mod_mtilde = 0;
        std::vector<TwPair> prod_q_mod_Bsk;  // q mod Bsk_s                        [nBsk]
        std::vector<TwPair> inv_mtilde_mod_Bsk; //                                 [nBsk]
        std::vector<TwPair> inv_q_mod_Bsk;   // q^-1 mod Bsk_s                     [nBsk]
        std::vector<TwPair> t_mod_q, t_mod_Bsk; // plain modulus                   [L], [nBsk]
        std::vector<TwPair> inv_punc_B;      // [(B/B_i)^-1]_{B_i}                 [nB]
        std::vector<u64> B_to_q;             // (B/B_i) mod q_j                    [L][nB]
        std::vector<u64> B_to_msk;           // (B/B_i) mod m_sk                   [nB]
        TwPair inv_B_mod_msk{};
        std::vector<TwPair> prod_B_mod_q, neg_prod_B_mod_q; // [L]
    };
    // |B| of the level with the first L primes of q: L, or L + 1 when K n t q^2 < q prod(B) m_sk needs it (rns.cpp:605-612)
    std::size_t behz_base_size(const std::vector<u64> &q, std::size_t L, u64 t);
    BehzLevel build_behz(std::size_t n, const std::vector<u64> &q, std::size_t L, u64 t);


    // ---- key switching through an exact integer convolution (sb_ksint.cu) ------------------------------------------------
    // The sum over digits of switch_key_inplace (evaluator.cpp:2664-2755), sum_J NTT_I(d_J) (.) K_JI mod q_I, is the NTT_I image
    // of the integer polynomial c = sum_J d_J * k_JI (negacyclic, d_J in [0,q_J), k_JI = INTT_I(K_JI) in [0,q_I)) reduced mod
    // q_I.  |c| < L n q_J q_I, so c is computed exactly modulo S auxiliary 29-bit NTT primes (32-bit butterflies, 4x cheaper on
    // 32-bit multipliers than 64-bit ones; the digit transforms are shared by all output primes) and reduced mod q_I afterwards.
    // Tables: {w, floor(w 2^32 / p)} pairs.
    struct KsIntHost
    {
        int S = 0;     // auxiliary primes
        int r = 0;     // stages of the outer pass: logn - 12 (the local pass transforms 4096-element blocks in shared memory)
        // most digits the product kernels sum in 64 bits without a reduction: the largest L with L (max p - 1)^2 < 2^64 (the
        // transformed digits and key words are canonical); levels with more digits take the 64-bit path (Context::ksint_on)
        std::size_t max_digits = 0;
        std::vector<std::uint32_t> p;          // [S]
        std::vector<std::uint32_t> red;        // [S][2]: 2^32 mod p with its quotient (reduction of 64-bit words)
        std::vector<std::uint32_t> mu;         // [S]: floor(2^32 / p)
        // outer-pass twiddles [S][2^r][2]: entry m + i of the stage with m groups (entry 0 unused); forward and inverse
        std::vector<std::uint32_t> fwd_outer, inv_outer;
        // local-pass twiddles [S][2^r blocks][4096][2]: entries 1..255 = stages with 1..128 groups per block in natural order
        // (2^s + i), entries 256.. = the last four stages transposed per thread: [256 + j * 256 + thread], j < 15
        std::vector<std::uint32_t> fwd_local, inv_local;
        // CRT reconstruction (P = prod p_t, H = (P - 1) / 2): y_t = x_t * c1_t + c2_t mod p_t with c1 = n^-1 (P/p_t)^-1,
        // c2 = H (P/p_t)^-1; value = sum y_t (P/p_t) - alpha P - H, alpha = floor(sum y_t / p_t) (the kernels estimate it from
        // sum y_t floor(2^60 / p_t): the true fraction lies in (1/4, 3/4))
        std::vector<std::uint32_t> c1;         // [S][2]
        std::vector<std::uint32_t> c2;         // [S]
        std::vector<u64> punct_mod_q;          // [k][S]: (P/p_t) mod q_i
        std::vector<u64> neg_mod_q;            // [k][S]: (-(alpha P) - H) mod q_i, alpha < S
    };
    KsIntHost build_ksint(std::size_t n, const u64 *q, std::size_t k);

    std::uint32_t galois_elt_from_step(std::size_t n, int step);                 // galois.cpp:53-95
    std::vector<std::uint32_t> galois_table_ntt(std::size_t n, std::uint32_t elt); // galois.cpp:18-51
    // BatchEncoder::populate_matrix_reps_index_map (batchencoder.cpp:54-76): slot i of the 2 x n/2 matrix -> coefficient index
    std::vector<std::uint32_t> batch_index_map(std::size_t n);
} // namespace sbh
