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

    // r (canonical) + the addend word, canonical: a second csub, so words of q - 1 everywhere stay below q.  No-op without an addend.
    template <class Base>
    __device__ __forceinline__ u64 plus_addend(const Base &base, int b, int c, int i, int logn, int idx, u64 r, u64 q)
    {
        if constexpr (Base::kAddend)
            return csub(r + base.arow(b, c, i, logn)[idx], q);
        else
            return r;
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
