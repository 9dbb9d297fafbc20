// seal_b200/csrc/sb_src.cuh -- how the key-switching kernels see their operands (shared by sb_engine.cu and sb_ksint.cu).
#pragma once
#include "sb_device.cuh"

namespace sb
{
    // --------------------------------------------------------------------------------- source accessors ----
    // A batch of [L][n] polynomials, optionally seen through a Galois automorphism (galois.cpp:148-218).
    struct Src
    {
        const u64 *p = nullptr;
        long long bstride = 0; // words between consecutive batch items
        const uint32_t *perm = nullptr; // NTT-form: out[i] = in[perm[i]]
        uint32_t ginv = 0;              // coefficient form: inverse Galois element mod 2n (0 = identity)
        int logn = 0;

        __device__ __forceinline__ bool plain() const { return perm == nullptr && ginv == 0; }
        __device__ __forceinline__ const u64 *row(int b, int J) const { return p + b * bstride + (static_cast<long long>(J) << logn); }
        __device__ __forceinline__ u64 get(int b, int J, int idx, u64 qJ) const
        {
            const u64 *r = p + b * bstride + (static_cast<long long>(J) << logn);
            if (perm)
                return r[perm[idx]];
            if (ginv)
            {
                uint32_t ip = (static_cast<uint32_t>(idx) * ginv) & ((2u << logn) - 1u);
                u64 v = r[ip & ((1u << logn) - 1u)];
                if (ip >> logn)
                    v = v ? qJ - v : 0;
                return v;
            }
            return r[idx];
        }
    };


    // what the mod-down result is added to (the ciphertext being updated)
    struct BaseSrc
    {
        Src s;            // polys 0,1 of the base ciphertext: poly c of item b at s.p + b*s.bstride + c*pstride
        long long pstride = 0;
        int c1_zero = 0;  // apply_galois: component 1 starts from zero (evaluator.cpp:2487)
        int present = 0;
        __device__ __forceinline__ u64 get(int b, int c, int i, int idx, u64 q) const
        {
            if (!present || (c == 1 && c1_zero))
                return 0;
            Src t = s;
            t.p += c * pstride;
            return t.get(b, i, idx, q);
        }
        static constexpr bool kAddend = false;
        static constexpr bool kPlain = false;
    };

    // BaseSrc plus an addend: a plain [B][2][L][n] source added to both output components after the base term (apply_galois_add:
    // out = addend + apply_galois(in)).  A type of its own, so that the kernels without an addend compile exactly as before.
    struct BaseAddSrc : BaseSrc
    {
        const u64 *a = nullptr; // component c of item b, prime i at a + b*a_bs + c*a_ps + i*n
        long long a_bs = 0, a_ps = 0;
        static constexpr bool kAddend = true;
        __device__ __forceinline__ const u64 *arow(int b, int c, int i, int logn) const
        {
            return a + b * a_bs + c * a_ps + (static_cast<long long>(i) << logn);
        }
    };

    // BaseSrc times an NTT-form plaintext, plus an addend when ADD (apply_galois_multiply_plain_add: out = addend + plain *
    // apply_galois(in)).  Both output components are multiplied by the same plaintext word, after the base term; the plaintext is
    // [P][L][n] with P = 1 (p_bs = 0, one plaintext for the batch) or one per item.  CKKS / BGV only: the key switch's result is
    // in NTT form there, so the plaintext product is element-wise.
    template <bool ADD>
    struct BasePlainSrc : BaseAddSrc
    {
        const u64 *pl = nullptr; // prime i of item b's plaintext at pl + b*p_bs + i*n
        long long p_bs = 0;
        static constexpr bool kAddend = ADD;
        static constexpr bool kPlain = true;
        __device__ __forceinline__ const u64 *prow(int b, int i, int logn) const { return pl + b * p_bs + (static_cast<long long>(i) << logn); }
    };

    // the last step of every key-switching exit, on r (canonical, the base term added): r * plaintext word (reduced on the way in, as
    // plain_mul_kernel reduces it: any 64-bit word is accepted), then + the addend word with a second csub, so words of q - 1
    // everywhere stay below q.  No-op for BaseSrc.
    template <class Base>
    __device__ __forceinline__ u64 finish(const Base &base, int b, int c, int i, int logn, int idx, u64 r, const PrimeDev &P)
    {
        if constexpr (Base::kPlain)
            r = mulmod_wide(r, canon_in(base.prow(b, i, logn)[idx], P), P);
        if constexpr (Base::kAddend)
            r = csub(r + base.arow(b, c, i, logn)[idx], P.q);
        return r;
    }
    // the same on the coefficient pair 2h, 2h + 1 past idx0, with 16-byte loads (the store8 exits)
    template <class Base>
    __device__ __forceinline__ void finish2(const Base &base, int b, int c, int i, int logn, int idx0, int h, u64 &r0, u64 &r1, const PrimeDev &P)
    {
        if constexpr (Base::kPlain)
        {
            const ulonglong2 pv = reinterpret_cast<const ulonglong2 *>(base.prow(b, i, logn) + idx0)[h];
            r0 = mulmod_wide(r0, canon_in(pv.x, P), P), r1 = mulmod_wide(r1, canon_in(pv.y, P), P);
        }
        if constexpr (Base::kAddend)
        {
            const ulonglong2 av = reinterpret_cast<const ulonglong2 *>(base.arow(b, c, i, logn) + idx0)[h];
            r0 = csub(r0 + av.x, P.q), r1 = csub(r1 + av.y, P.q);
        }
    }

    // (1) target -> coefficient form (CKKS / BGV): rows (b, J); evaluator.cpp:2651-2658
    struct OpKsIntt
    {
        Src tgt;
        u64 *D; // [B][L][n]
        int logn, L;
        __device__ __forceinline__ bool skip(int) const { return false; }
        __device__ __forceinline__ int pid(int row) const { return row % L; }
        __device__ __forceinline__ const u64 *direct(int row, const PrimeDev &) const { return tgt.plain() ? tgt.row(row / L, row % L) : nullptr; }
        __device__ __forceinline__ u64 load1(int row, int idx, const PrimeDev &P) const
        {
            return tgt.get(row / L, row % L, idx, P.q);
        }
        __device__ __forceinline__ void load8(int row, int idx0, u64 (&a)[8], const PrimeDev &P) const
        {
            if (tgt.plain())
            {
                const ulonglong2 *p = reinterpret_cast<const ulonglong2 *>(tgt.row(row / L, row % L) + idx0);
#pragma unroll
                for (int j = 0; j < 4; j++)
                {
                    ulonglong2 v = p[j];
                    a[2 * j] = v.x, a[2 * j + 1] = v.y;
                }
                return;
            }
#pragma unroll
            for (int j = 0; j < 8; j++)
                a[j] = load1(row, idx0 + j, P);
        }
        __device__ __forceinline__ u64 *mid(int row) const { return D + (static_cast<long long>(row) << logn); }
        __device__ __forceinline__ void store1(int row, int idx, u64 v, const PrimeDev &P) const { mid(row)[idx] = csub(v, P.q); }
        __device__ __forceinline__ void store8(int row, int idx0, u64 (&a)[8], const PrimeDev &P) const
        {
#pragma unroll
            for (int j = 0; j < 8; j++)
                store1(row, idx0 + j, a[j], P);
        }
    };
} // namespace sb
