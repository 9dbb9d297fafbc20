// seal_b200/csrc/sb_device.cuh -- device-side modular arithmetic and shared structs (sm_90a).
//
// All residues are uint64 (primes < 2^61: user primes <= 60 bits, BEHZ auxiliary primes 61 bits; reference limits in
// util/defines.h:32-71).  Twiddle multiplications use Shoup/Harvey precomputed quotients (the same mathematical device
// the reference uses in util/uintarithsmallmod.h:255-326), general products use a 128-bit Barrett step.  Outputs that
// leave a kernel are canonical residues in [0, q) so results are word-identical to the reference (SURVEY 0.2).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

typedef unsigned long long u64;

struct __align__(16) Tw
{
    u64 w;  // twiddle value in [0, q)
    u64 wq; // floor(w * 2^64 / q)
};

// Per-prime constants + table pointers, one entry per prime id (q-chain primes first, then BEHZ auxiliary primes).
struct PrimeDev
{
    u64 q;
    u64 q2;         // 2q
    u64 q4;         // 4q
    u64 nq;         // 2^64 - q
    u64 zero;       // always 0, but not a compile-time constant: see ct_bfly
    u64 ratio_lo;   // floor(2^128 / q), low word
    u64 ratio_hi;   //                   high word (= floor(2^64 / q))
    Tw inv_n;       // n^-1 mod q
    Tw inv_n_w;     // n^-1 * (last inverse-stage twiddle) mod q
    const Tw *fwd;  // fwd[m + i]: forward stage with m groups, group i  (psi powers, bit-reversed order)
    const Tw *inv;  // inv[m + i]: inverse stage with m groups, group i  (psi^-1 powers)
    u64 mu;         // floor(2^(b+62) / q), b = bit length of q: one-word Barrett constant of barrett_wide
    int sh;         // b - 2
    int pad_;
};

__device__ __forceinline__ u64 csub(u64 x, u64 q)
{
    return x >= q ? x - q : x;
}

// x - y mod q on words a caller handed in, in the reference's borrow form (sub_uint_mod, util/uintarithsmallmod.h:156-158, and
// sub_poly_coeffmod, polyarithsmallmod.cpp:126-128, in a release build): the 64-bit difference, plus q when it borrowed, and no
// further reduction.  For x, y < q this equals csub(x + q - y, q); for other words it is the reference's word, which x + q - y
// is not (that sum wraps when x - y > 2^64 - q, and stays at or above q when y - x > q).
__device__ __forceinline__ u64 sub_borrow(u64 x, u64 y, u64 q)
{
    return x - y + (x < y ? q : 0);
}

// ---- Shoup / Harvey multiplication tuned for the integer pipes (32-bit multipliers) -------------------------------------------
// Integer multiplies issue on the FMA-heavy pipe only (ncu: the binding pipe of every transform kernel) and a
// 32x32->64 multiply-add costs twice a 32-bit one, so the quotient estimate uses three wide products instead of the
// four (+ carry chain) of an exact 64x64 high half:
//     T = y1*wq1 + hi32(y1*wq0) + hi32(y0*wq1)      with  t-2 <= T <= t,  t = floor(y*wq / 2^64)
// and the remainder y*w - T*q is formed as lo64(y*w + T*(2^64-q)) with two wide and four 32-bit multiply-adds.
// Result: x*w mod q in [0, 4q) for ANY 64-bit x (w < q, wq = floor(w 2^64 / q), q < 2^61).
__device__ __forceinline__ u64 pack64(unsigned lo, unsigned hi)
{
    u64 r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "r"(lo), "r"(hi));
    return r;
}
__device__ __forceinline__ void unpack64(u64 v, unsigned &lo, unsigned &hi)
{
    asm("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(v));
}
// written so that the two 32-bit high halves are added to the low word of y1*wq1 in ONE three-input add with two carry outputs and
// the carries enter the high word in one IADD3.X: no zero-extended register pair, no carry materialised with SEL, nothing on
// the multiply pipe besides the three wide products (tools/bfly2.cu, tools/sass_cost.py)
__device__ __forceinline__ u64 approx_mulhi(u64 y, u64 wq)
{
    unsigned y0, y1, wq0, wq1, alo, ahi, blo, bhi, tl, th;
    unpack64(y, y0, y1);
    unpack64(wq, wq0, wq1);
    u64 a, b, T;
    // the two cross products have equal weight 2^32: keep their high halves, drop their low halves and y0*wq0
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(a) : "r"(y1), "r"(wq0));
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(b) : "r"(y0), "r"(wq1));
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(T) : "r"(y1), "r"(wq1));
    unpack64(a, alo, ahi);
    unpack64(b, blo, bhi);
    unpack64(T, tl, th);
    const u64 s = static_cast<u64>(tl) + ahi + bhi; // < 3 * 2^32
    return pack64(static_cast<unsigned>(s), th + static_cast<unsigned>(s >> 32));
}
// lo64(y*w + T*nq)
__device__ __forceinline__ u64 mullo_combine(u64 y, u64 w, u64 T, u64 nq)
{
    unsigned y0, y1, w0, w1, T0, T1, n0, n1, lo, hi;
    unpack64(y, y0, y1);
    unpack64(w, w0, w1);
    unpack64(T, T0, T1);
    unpack64(nq, n0, n1);
    u64 acc;
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(acc) : "r"(y0), "r"(w0));
    asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc) : "r"(T0), "r"(n0));
    unpack64(acc, lo, hi);
    asm("mad.lo.u32 %0, %1, %2, %0;" : "+r"(hi) : "r"(y0), "r"(w1));
    asm("mad.lo.u32 %0, %1, %2, %0;" : "+r"(hi) : "r"(y1), "r"(w0));
    asm("mad.lo.u32 %0, %1, %2, %0;" : "+r"(hi) : "r"(T0), "r"(n1));
    asm("mad.lo.u32 %0, %1, %2, %0;" : "+r"(hi) : "r"(T1), "r"(n0));
    return pack64(lo, hi);
}
__device__ __forceinline__ u64 mul_shoup_lazy4(u64 x, Tw t, u64 nq)
{
    return mullo_combine(x, t.w, approx_mulhi(x, t.wq), nq);
}
// exact variants (result in [0,2q) / canonical) for the element-wise epilogues
__device__ __forceinline__ u64 mul_shoup_lazy(u64 x, Tw t, u64 q)
{
    u64 h = __umul64hi(x, t.wq);
    return x * t.w - h * q;
}
__device__ __forceinline__ u64 mul_shoup(u64 x, Tw t, u64 q)
{
    return csub(mul_shoup_lazy(x, t, q), q);
}
// x mod q, lazily in [0, 4q), for any 64-bit x (three wide products + one wide + two 32-bit multiply-adds)
__device__ __forceinline__ u64 barrett_lazy4(u64 x, u64 ratio_hi, u64 nq)
{
    u64 T = approx_mulhi(x, ratio_hi);
    const unsigned T0 = static_cast<unsigned>(T), T1 = static_cast<unsigned>(T >> 32);
    const unsigned n0 = static_cast<unsigned>(nq), n1 = static_cast<unsigned>(nq >> 32);
    u64 acc = static_cast<u64>(T0) * n0 + x;
    unsigned hi = static_cast<unsigned>(acc >> 32) + T0 * n1 + T1 * n0;
    return (static_cast<u64>(hi) << 32) | static_cast<unsigned>(acc);
}

// x mod q for any 64-bit x (ratio_hi = floor(2^64 / q)); result canonical.
__device__ __forceinline__ u64 barrett64(u64 x, u64 q, u64 ratio_hi)
{
    u64 t = __umul64hi(x, ratio_hi);
    return csub(x - t * q, q);
}

// (hi:lo) mod q for a 128-bit value; ratio = floor(2^128 / q).  Exact floor of the 256-bit product's top limb is
// approximated from below by at most 1, so one conditional subtraction canonicalises.
__device__ __forceinline__ u64 barrett128(u64 lo, u64 hi, u64 q, u64 ratio_lo, u64 ratio_hi)
{
    u64 c0 = __umul64hi(lo, ratio_lo);
    u64 a_lo = lo * ratio_hi, a_hi = __umul64hi(lo, ratio_hi);
    u64 b_lo = hi * ratio_lo, b_hi = __umul64hi(hi, ratio_lo);
    u64 s = a_lo + c0;
    u64 carry = (s < a_lo);
    u64 s2 = s + b_lo;
    carry += (s2 < s);
    u64 t = hi * ratio_hi + a_hi + b_hi + carry;
    return csub(lo - t * q, q);
}

// (hi:lo) mod q for values below 2^(b+62), b = bit length of q (a product of two residues, a sum of two such products, the CRT sums
// of sb_ksint.cu): the quotient is estimated from the top 64 bits of the value with ONE high multiply -- floor(z / 2^(b-2)) * mu
// / 2^64 is at most 2 below floor(z / q) -- instead of the three high + three low multiplies of the full 128-bit Barrett step.
__device__ __forceinline__ u64 barrett_wide(u64 lo, u64 hi, const PrimeDev &P)
{
    unsigned w0, w1, w2, w3;
    unpack64(lo, w0, w1);
    unpack64(hi, w2, w3);
    const bool up = P.sh >= 32;
    const unsigned a0 = up ? w1 : w0, a1 = up ? w2 : w1, a2 = up ? w3 : w2;
    const u64 zh = pack64(__funnelshift_r(a0, a1, P.sh), __funnelshift_r(a1, a2, P.sh)); // z >> sh, fits 64 bits
    const u64 t = __umul64hi(zh, P.mu);
    const u64 r = lo - t * P.q; // in [0, 3q)
    return csub(csub(r, P.q2), P.q);
}
// a word of a ciphertext / plaintext the caller handed in: below q for valid objects; anything else is reduced first, so that the
// dyadic kernels give the reference's result (its Barrett step accepts any 64-bit operands) instead of relying on the range
__device__ __forceinline__ u64 canon_in(u64 x, const PrimeDev &P)
{
    return x < P.q ? x : barrett64(x, P.q, P.ratio_hi);
}
// a * b mod q, canonical, for a * b < 2^(b+62) (e.g. both operands below q)
__device__ __forceinline__ u64 mulmod_wide(u64 a, u64 b, const PrimeDev &P)
{
    return barrett_wide(a * b, __umul64hi(a, b), P);
}

// a * b mod q, canonical, a and b arbitrary 64-bit with a*b < 2^128 trivially.
__device__ __forceinline__ u64 mulmod_barrett(u64 a, u64 b, const PrimeDev &P)
{
    return barrett128(a * b, __umul64hi(a, b), P.q, P.ratio_lo, P.ratio_hi);
}

// ---- coefficient-form plaintext words (BFV / BGV), shared by the plaintext operations and encryption ----
// lift of one coefficient-form plaintext word v < t to the prime q: the representative in (-t/2, t/2] modulo q
// (plain_upper_half_threshold / plain_upper_half_increment, evaluator.cpp:2240-2272, :2101-2127)
__device__ __forceinline__ u64 plain_lift(u64 v, u64 t, u64 t_mod_q, const PrimeDev &P)
{
    u64 r = t > P.q ? barrett64(v, P.q, P.ratio_hi) : v;
    if (v >= ((t + 1) >> 1))
        r = csub(r + P.q - t_mod_q, P.q);
    return r;
}

// BFV: round(q m / t) of a plaintext word m < t, in two parts (multiply_add_plain_with_scaling_variant, util/scalingvariant.cpp:70-160).
// bfv_plain_fix = floor((m (q mod t) + (t + 1) / 2) / t), the same for every prime: quotient estimate from the Barrett ratio
// floor((2^128 - 1) / t), corrected by the remainder.
__device__ __forceinline__ u64 bfv_plain_fix(u64 m, u64 t, u64 t_ratio_lo, u64 t_ratio_hi, u64 q_mod_t)
{
    u64 lo = m * q_mod_t, hi = __umul64hi(m, q_mod_t);
    const u64 half = (t + 1) >> 1;
    lo += half, hi += (lo < half);
    const u64 c0 = __umul64hi(lo, t_ratio_lo);
    const u64 a_lo = lo * t_ratio_hi, a_hi = __umul64hi(lo, t_ratio_hi), b_lo = hi * t_ratio_lo, b_hi = __umul64hi(hi, t_ratio_lo);
    u64 s1 = a_lo + c0, carry = (s1 < a_lo);
    const u64 s2 = s1 + b_lo;
    carry += (s2 < s1);
    u64 fix = hi * t_ratio_hi + a_hi + b_hi + carry;
    u64 rem = lo - fix * t;
#pragma unroll
    for (int r = 0; r < 2; r++)
        if (rem >= t)
            rem -= t, fix++;
    return fix;
}
// ... and modulo one prime: m floor(q / t) + fix mod q_i, canonical (delta = floor(q / t) mod q_i with its Shoup quotient)
__device__ __forceinline__ u64 bfv_plain_scaled(u64 m, u64 fix, u64 t, Tw delta, const PrimeDev &P)
{
    const u64 mm = t > P.q ? barrett64(m, P.q, P.ratio_hi) : m;
    return csub(mul_shoup(mm, delta, P.q) + barrett64(fix, P.q, P.ratio_hi), P.q);
}

// 128-bit accumulate: (hi:lo) += a*b
__device__ __forceinline__ void mac128(u64 &lo, u64 &hi, u64 a, u64 b)
{
    // one carry chain instead of a compare + select per accumulate
    asm("mad.lo.cc.u64 %0, %2, %3, %0;\n\tmadc.hi.u64 %1, %2, %3, %1;" : "+l"(lo), "+l"(hi) : "l"(a), "l"(b));
}

// RNSBase::compose (rns.cpp:321-352) of one coefficient into val = L little-endian words in [0, Q): val = sum_j punct_j * (x_j *
// (Q/q_j)^-1 mod q_j) with one conditional subtraction of Q per prime, x_j = residue(j) modulo prime j (the caller loads it).
// Q = [L] words, punct = [L][L] words of Q / q_j, invp = (Q/q_j)^-1 mod q_j (sb_engine.cuh: Context::CrtLevel).  Used by CKKS
// decode (sb_ckks.cu) and the invariant noise budget (sb_engine.cu); the integers live in local memory, one thread per coefficient.
constexpr int kCrtMaxWords = 64; // SEAL_COEFF_MOD_COUNT_MAX (util/defines.h)
template <class Residue>
__device__ __forceinline__ void crt_compose(const Residue &residue, const u64 *__restrict__ Q, const u64 *__restrict__ punct,
                                            const Tw *__restrict__ invp, const PrimeDev *__restrict__ primes, int L, u64 (&val)[kCrtMaxWords])
{
    for (int w = 0; w < L; w++)
        val[w] = 0;
    if (L == 1)
        val[0] = residue(0);
    else
        for (int j = 0; j < L; j++)
        {
            const u64 t = mul_shoup(residue(j), invp[j], primes[j].q);
            // val += punct_j * t  (punct_j * t < Q), then one conditional subtraction of Q
            u64 carry = 0, cy = 0;
            for (int w = 0; w < L; w++)
            {
                const u64 p = punct[j * L + w];
                const u64 lo = p * t, hi = __umul64hi(p, t);
                u64 term = lo + carry;
                carry = hi + (term < lo);
                u64 sum = val[w] + term;
                const u64 c1 = sum < term;
                sum += cy;
                cy = c1 | (sum < cy);
                val[w] = sum;
            }
            bool ge = cy != 0;
            if (!ge)
            {
                ge = true;
                for (int w = L - 1; w >= 0; w--)
                    if (val[w] != Q[w])
                    {
                        ge = val[w] > Q[w];
                        break;
                    }
            }
            if (ge)
            {
                u64 bw = 0;
                for (int w = 0; w < L; w++)
                {
                    const u64 a = val[w], s1 = a - Q[w], s2 = s1 - bw;
                    bw = (a < Q[w]) | (s1 < bw);
                    val[w] = s2;
                }
            }
        }
}

// (hi:lo) += a*b for bounded operands (a < 2^63.25, b < 2^62: lazily grown transform outputs times canonical key words): four
// wide multiplies -- p0 = a0*b0, mid = a0*b1 + a1*b0 (fits 64 bits under the bounds), p3 = a1*b1 -- and two carry chains over the
// four 32-bit words of the sum.  ptxas expands the generic mac128 into 5-7 wide multiplies and ~10 adds per product.
__device__ __forceinline__ void mac128_4(u64 &lo, u64 &hi, u64 a, u64 b)
{
    unsigned a0, a1, b0, b1, w0, w1, w2, w3, p00, p01, m0, m1, p30, p31;
    unpack64(a, a0, a1);
    unpack64(b, b0, b1);
    unpack64(lo, w0, w1);
    unpack64(hi, w2, w3);
    u64 p0, mid, p3;
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(p0) : "r"(a0), "r"(b0));
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(mid) : "r"(a0), "r"(b1));
    asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(mid) : "r"(a1), "r"(b0));
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(p3) : "r"(a1), "r"(b1));
    unpack64(p0, p00, p01);
    unpack64(mid, m0, m1);
    unpack64(p3, p30, p31);
    asm("add.cc.u32 %0, %0, %4;\n\t"
        "addc.cc.u32 %1, %1, %5;\n\t"
        "addc.cc.u32 %2, %2, %6;\n\t"
        "addc.u32 %3, %3, %7;\n\t"
        "add.cc.u32 %1, %1, %8;\n\t"
        "addc.cc.u32 %2, %2, %9;\n\t"
        "addc.u32 %3, %3, 0;"
        : "+r"(w0), "+r"(w1), "+r"(w2), "+r"(w3)
        : "r"(p00), "r"(p01), "r"(p30), "r"(p31), "r"(m0), "r"(m1));
    lo = pack64(w0, w1), hi = pack64(w2, w3);
}

// Harvey-style butterflies on lazily reduced values.
// forward (Cooley-Tukey).  FAST (all primes of the launch < 2^57): no conditional subtraction at all -- values grow
//   by at most 4q per stage ((4 + 4*17) q < 2^64), the kernel reduces once before the store.
//   guarded (any prime < 2^61): inputs in [0,8q) -> outputs in [0,8q).
template <bool FAST>
__device__ __forceinline__ void ct_bfly(u64 &x, u64 &y, Tw w, const PrimeDev &P)
{
    u64 v = mul_shoup_lazy4(y, w, P.nq);
    u64 u = FAST ? x : csub(x, P.q4);
    // three-operand form: keeps the 64-bit adds on the integer ALU (IADD3/IADD3.X); the two-operand form is scheduled by
    // ptxas onto the multiply pipe (IMAD.X), which is the pipe that limits these kernels
    x = u + v + P.zero;
    y = u - v + P.q4;
}
// inverse (Gentleman-Sande): inputs in [0,4q) -> outputs in [0,4q)
__device__ __forceinline__ void gs_bfly(u64 &x, u64 &y, Tw w, const PrimeDev &P)
{
    u64 u = x, v = y;
    x = csub(u + v, P.q4);
    y = mul_shoup_lazy4(u - v + P.q4, w, P.nq);
}
// forward values before the store: -> [0, 4q)
template <bool FAST>
__device__ __forceinline__ u64 fwd_finish(u64 v, const PrimeDev &P)
{
    return FAST ? barrett_lazy4(v, P.ratio_hi, P.nq) : csub(v, P.q4);
}

__device__ __forceinline__ Tw ldg_tw(const Tw *p)
{
    ulonglong2 v = __ldg(reinterpret_cast<const ulonglong2 *>(p));
    Tw t;
    t.w = v.x;
    t.wq = v.y;
    return t;
}

// ---- TMA (1-D bulk async copy global -> shared) + mbarrier helpers --------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p)
{
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(u64 *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(u64 *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void *dst_smem, const void *src_gmem, uint32_t bytes, u64 *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// 1-D bulk async copy shared -> global, one bulk group per copy.  The threads that wrote the source run fence_proxy_async() before
// the barrier that precedes the copy; the source may be rewritten after bulk_wait_read, the CTA may exit after bulk_wait
__device__ __forceinline__ void tma_store_1d(void *dst_gmem, const void *src_smem, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)), "r"(bytes)
                 : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// all but the newest N bulk groups of this thread have read their sources / have completed
template <int N>
__device__ __forceinline__ void bulk_wait_read()
{
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait()
{
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void mbar_wait(u64 *bar, uint32_t phase)
{
    asm volatile("{\n"
                 ".reg .pred p;\n"
                 "WAIT_%=:\n"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
                 "@p bra DONE_%=;\n"
                 "bra WAIT_%=;\n"
                 "DONE_%=:\n"
                 "}" ::"r"(smem_u32(bar)),
                 "r"(phase)
                 : "memory");
}
