// seal_b200/csrc/sb_ntt.cuh -- batched negacyclic NTT / inverse NTT kernels for sm_90a.
//
// Replaces the reference's DWTHandler::transform_to_rev / transform_from_rev (util/dwthandler.h:94-356) driven by
// ntt_negacyclic_harvey(_lazy) / inverse_ntt_negacyclic_harvey(_lazy) (util/ntt.cpp:394-475).  Same mathematical
// transform (psi = minimal primitive 2n-th root, output of the forward transform in bit-reversed order), different
// schedule:
//
//   n = NA * 256.  The log2(NA) stages whose butterflies span more than 256 coefficients run in a "column pass":
//   a CTA owns NA rows x C columns (4096 coefficients, C = 4096/NA) in shared memory, every thread keeps 8
//   coefficients in registers and does radix-8 (3 stages) per register pass; the NA-1 twiddles of those stages are the
//   same for every column and are staged to shared memory with one TMA bulk copy.  The 8 stages that stay inside a
//   256-coefficient block run in a "local pass": one warp owns one block, 8 coefficients per lane, exchanges through a
//   warp-private, XOR-swizzled (bank-conflict-free) 2 KiB shared-memory slice with __syncwarp only.
//   The two passes meet in an intermediate row that is sized to stay L2-resident (see DESIGN.md).
//
// Every kernel is parameterised by an Op functor that supplies the row->prime map, the load (prologue) and the store
// (epilogue), so digit reduction, rounding corrections, canonicalisation and the key-switch combine are fused into the
// transforms instead of being separate passes over HBM.
//
// Op interface (all __device__):
//   bool skip(int row)                       row needs no transform (CTA exits)
//   int  pid(int row)                        prime id of the row
//   u64  load1(int row, int idx, P)          value of coefficient idx  (forward: < 4q, inverse: < 4q)
//   const u64 *direct(int row, P)            non-null when load1(row, idx) == direct(row)[idx] (plain row, no prologue)
//   void load8(int row, int idx0, u64(&)[8], P)   8 consecutive coefficients
//   u64 *mid(int row)                        n-word intermediate row between the two passes
//   void store1(int row, int idx, u64 v, P)  v lazily reduced (forward: < 4q, inverse: < 2q)
//   void store8(int row, int idx0, u64(&)[8], P)
#pragma once
#include "sb_device.cuh"
#include <vector>

#ifndef SB_COL_MIN_BLOCKS
#define SB_COL_MIN_BLOCKS 3 // 512-thread column-pass CTAs per SM the register allocation is tuned for
#endif

namespace sb
{
    constexpr int kLocalLog = 8;       // 256-coefficient local blocks
    constexpr int kTile = 4096;        // coefficients per column-pass CTA
    constexpr int kColThreads = kTile / 8;

    // ------------------------------------------------------------------------------- register radix-8 helpers ----
    // forward, pair levels in order: (j,j+4), (j,j+2), (j,j+1)
    template <int NST, bool FAST, class TwF>
    __device__ __forceinline__ void fwd_regs(u64 (&a)[8], TwF tw, const PrimeDev &P)
    {
        {
            Tw w = tw(0, 0);
#pragma unroll
            for (int j = 0; j < 4; j++)
                ct_bfly<FAST>(a[j], a[j + 4], w, P);
        }
        if (NST >= 2)
        {
            Tw w0 = tw(1, 0), w1 = tw(1, 1);
            ct_bfly<FAST>(a[0], a[2], w0, P);
            ct_bfly<FAST>(a[1], a[3], w0, P);
            ct_bfly<FAST>(a[4], a[6], w1, P);
            ct_bfly<FAST>(a[5], a[7], w1, P);
        }
        if (NST >= 3)
        {
#pragma unroll
            for (int p = 0; p < 4; p++)
                ct_bfly<FAST>(a[2 * p], a[2 * p + 1], tw(2, p), P);
        }
    }

    // inverse, pair levels in order: (j,j+1) [level 0], (j,j+2) [level 1], (j,j+4) [level 2]; FIRST = first level run
    // FINAL: the (j,j+4) level is the last stage of the whole transform -> fold n^-1 (dwthandler.h:273-313)
    template <int FIRST, bool FINAL, class TwF>
    __device__ __forceinline__ void inv_regs(u64 (&a)[8], TwF tw, const PrimeDev &P)
    {
        if (FIRST <= 0)
        {
#pragma unroll
            for (int p = 0; p < 4; p++)
                gs_bfly(a[2 * p], a[2 * p + 1], tw(0, p), P);
        }
        if (FIRST <= 1)
        {
            Tw w0 = tw(1, 0), w1 = tw(1, 1);
            gs_bfly(a[0], a[2], w0, P);
            gs_bfly(a[1], a[3], w0, P);
            gs_bfly(a[4], a[6], w1, P);
            gs_bfly(a[5], a[7], w1, P);
        }
        if (!FINAL)
        {
            Tw w = tw(2, 0);
#pragma unroll
            for (int j = 0; j < 4; j++)
                gs_bfly(a[j], a[j + 4], w, P);
        }
        else
        {
            // last stage: outputs reduced to [0, 2q) for the store
#pragma unroll
            for (int j = 0; j < 4; j++)
            {
                u64 u = a[j], v = a[j + 4];
                a[j] = csub(mul_shoup_lazy4(u + v, P.inv_n, P.nq), P.q2);
                a[j + 4] = csub(mul_shoup_lazy4(u - v + P.q4, P.inv_n_w, P.nq), P.q2);
            }
        }
    }

    // warp-private swizzle of a 256-word slice: every access pattern used below hits 16 distinct 8-byte banks per
    // half-warp (checked exhaustively in tests/test_host_logic.py::test_swizzle_conflict_free)
    __device__ __forceinline__ int swz(int e)
    {
        int b4 = (e >> 4) & 1, b5 = (e >> 5) & 1, b6 = (e >> 6) & 1;
        return e ^ (b4 | (b5 << 1) | (b6 << 2) | ((b5 ^ b6) << 3));
    }

    // ---------------------------------------------------------------------------------- forward: column pass ----
    // The log2(NA) column stages on one thread's 8 coefficients: in = layout r = ridx + j*(NA/8), out = layout r = 8*ridx + j.
    // Layout changes go through the CTA's shared tile (two barriers each); tw_s = the NA-1 twiddles of these stages.
    template <int LOGNA, bool FAST>
    __device__ __forceinline__ void fwd_col_passes(u64 (&a)[8], u64 *tile, const Tw *tw_s, int ridx, int c, const PrimeDev &P)
    {
        constexpr int NA = 1 << LOGNA;
        constexpr int C = kTile / NA;
        constexpr int NST0 = LOGNA % 3;
        int prev_g = NA >> 3; // layout of the loaded registers: r = rhi*8g + rlo + j*g with g = NA/8 (rhi = 0)
        if (NST0 != 0)
        {
            // partial first pass: stages 0..NST0-1 in the initial layout
            auto twf = [&](int lvl, int k) { return tw_s[(1 << lvl) + k]; };
            fwd_regs<NST0, FAST>(a, twf, P);
        }
        // full 3-stage passes; the layout changes between passes through the shared tile
#pragma unroll
        for (int S = NST0; S < LOGNA; S += 3)
        {
            const int g = NA >> (S + 3);
            const int rhi = ridx / g, rlo = ridx % g;
            if (g != prev_g)
            {
                const int prhi = ridx / prev_g, prlo = ridx % prev_g;
#pragma unroll
                for (int j = 0; j < 8; j++)
                    tile[(prhi * 8 * prev_g + prlo + j * prev_g) * C + c] = a[j];
                __syncthreads();
#pragma unroll
                for (int j = 0; j < 8; j++)
                    a[j] = tile[(rhi * 8 * g + rlo + j * g) * C + c];
                __syncthreads();
            }
            const int m = 1 << S;
            auto twf = [&](int lvl, int k) { return tw_s[(m << lvl) + (rhi << lvl) + k]; };
            fwd_regs<3, FAST>(a, twf, P);
            prev_g = g;
        }
    }

    template <int LOGNA, bool FAST, class Op>
    __global__ void __launch_bounds__(kColThreads, SB_COL_MIN_BLOCKS) ntt_fwd_col(Op op, const PrimeDev *__restrict__ primes)
    {
        constexpr int NA = 1 << LOGNA;
        constexpr int C = kTile / NA;
        constexpr int NST0 = LOGNA % 3;
        __shared__ __align__(16) u64 tile[kTile];
        __shared__ __align__(16) Tw tw_s[NA];
        __shared__ __align__(8) u64 bar;

        const int row = blockIdx.x, col0 = blockIdx.y * C;
        if (op.skip(row))
            return;
        const int tid = threadIdx.x, c = tid % C, ridx = tid / C;
        const PrimeDev P = primes[op.pid(row)];

        if (tid == 0)
            mbar_init(&bar, 1);
        __syncthreads();
        if (tid == 0)
        {
            mbar_expect_tx(&bar, NA * sizeof(Tw));
            tma_load_1d(tw_s, P.fwd, NA * sizeof(Tw), &bar); // entries [1, NA) are the twiddles of stages 0..LOGNA-1
        }

        u64 a[8];
        {
            constexpr int g = NA >> 3; // first layout: r = ridx + j*g
            const u64 *dp = op.direct(row, P); // non-null: the row is a plain array in range, no prologue needed
            if (dp)
            {
                dp += (ridx << kLocalLog) + col0 + c;
#pragma unroll
                for (int j = 0; j < 8; j++)
                    a[j] = dp[(j * g) << kLocalLog];
            }
            else
            {
#pragma unroll
                for (int j = 0; j < 8; j++)
                    a[j] = op.load1(row, ((ridx + j * g) << kLocalLog) + col0 + c, P);
            }
        }
        mbar_wait(&bar, 0);

        fwd_col_passes<LOGNA, FAST>(a, tile, tw_s, ridx, c, P);
        // last layout has g = 1: r = 8*ridx + j
        u64 *mid = op.mid(row);
#pragma unroll
        for (int j = 0; j < 8; j++)
            mid[((8 * ridx + j) << kLocalLog) + col0 + c] = a[j];
    }

    // ----------------------------------------------------------------------------------- forward: local pass ----
    // The 8 stages inside one 256-coefficient block, executed by one warp.  In: a[j] = coefficient l + 32 j of the
    // block (lane l).  Out: a[j] = coefficient 8 l + j, lazily reduced (FAST: unreduced growth, guarded: < 8q).
    // x = the warp's private 256-word shared slice; t0 = NA + block index (twiddle base of the block).
    // twf(s, i): twiddle of in-block stage s (0..7), group i of this block (0 <= i < 2^s)
    template <bool FAST, class TwF>
    __device__ __forceinline__ void fwd_local_block_tw(u64 (&a)[8], u64 *x, TwF twf, int l, const PrimeDev &P)
    {
        {
            auto t = [&](int lvl, int k) { return twf(lvl, k); };
            fwd_regs<3, FAST>(a, t, P);
        }
#pragma unroll
        for (int j = 0; j < 8; j++)
            x[swz(l + 32 * j)] = a[j];
        __syncwarp();
        {
            const int hi = l >> 2, lo = l & 3;
#pragma unroll
            for (int j = 0; j < 8; j++)
                a[j] = x[swz(32 * hi + lo + 4 * j)];
            auto t = [&](int lvl, int k) { return twf(3 + lvl, (hi << lvl) + k); };
            fwd_regs<3, FAST>(a, t, P);
            __syncwarp();
#pragma unroll
            for (int j = 0; j < 8; j++)
                x[swz(32 * hi + lo + 4 * j)] = a[j];
        }
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 8; j++)
            a[j] = x[swz(8 * l + j)];
        __syncwarp();
        {
            // strides 2 and 1: pairs (j,j+2) then (j,j+1)
            Tw wa = twf(6, 2 * l), wb = twf(6, 2 * l + 1);
            ct_bfly<FAST>(a[0], a[2], wa, P);
            ct_bfly<FAST>(a[1], a[3], wa, P);
            ct_bfly<FAST>(a[4], a[6], wb, P);
            ct_bfly<FAST>(a[5], a[7], wb, P);
#pragma unroll
            for (int p = 0; p < 4; p++)
                ct_bfly<FAST>(a[2 * p], a[2 * p + 1], twf(7, 4 * l + p), P);
        }
    }
    template <bool FAST>
    __device__ __forceinline__ void fwd_local_block(u64 (&a)[8], u64 *x, const Tw *__restrict__ tw, int t0, int l, const PrimeDev &P)
    {
        auto twf = [&](int s, int i) { return ldg_tw(tw + (t0 << s) + i); };
        fwd_local_block_tw<FAST>(a, x, twf, l, P);
    }

    // dynamic shared memory of the local passes: [xs 8 x 256 u64 | twiddles of the CTA's 8 adjacent blocks 8 * 255 x 16 B | mbarrier].
    // Stage s of 8 adjacent blocks is one contiguous run of 8 * 2^s table entries: 8 TMA bulk copies stage all 2040 twiddles while
    // the data loads are in flight (fetching them with one dependent global load per stage left the warps waiting on memory 8 times
    // per block: ncu long-scoreboard 6.5 per issue in round 2's capture of the result transform).
    constexpr int kLocalSmem = 8 * 256 * 8 + 8 * 255 * 16 + 16;
    __device__ __forceinline__ void stage_local_twiddles(Tw *tws, u64 *bar, const Tw *table, int na)
    {
        if (threadIdx.x == 0)
            mbar_init(bar, 1);
        __syncthreads();
        if (threadIdx.x == 0)
        {
            mbar_expect_tx(bar, 8 * 255 * sizeof(Tw));
#pragma unroll
            for (int st = 0; st < 8; st++)
                tma_load_1d(tws + 8 * ((1 << st) - 1), table + ((na + blockIdx.y * 8) << st), (8u << st) * sizeof(Tw), bar);
        }
    }
    template <bool FAST, class Op>
    __global__ void __launch_bounds__(256) ntt_fwd_local(Op op, const PrimeDev *__restrict__ primes, int na)
    {
        extern __shared__ __align__(16) unsigned char nl_smem[];
        u64(*xs)[256] = reinterpret_cast<u64(*)[256]>(nl_smem);
        Tw *tws = reinterpret_cast<Tw *>(nl_smem + 8 * 256 * 8);
        u64 *bar = reinterpret_cast<u64 *>(tws + 8 * 255);
        const int row = blockIdx.x, warp = threadIdx.x >> 5, l = threadIdx.x & 31;
        if (op.skip(row))
            return;
        const int b = blockIdx.y * 8 + warp;
        const PrimeDev P = primes[op.pid(row)];
        stage_local_twiddles(tws, bar, P.fwd, na);
        const u64 *src = op.mid(row) + (b << kLocalLog);
        u64 a[8];
#pragma unroll
        for (int j = 0; j < 8; j++)
            a[j] = src[l + 32 * j];
        mbar_wait(bar, 0);
        fwd_local_block_tw<FAST>(a, xs[warp], [&](int s_, int i) { return tws[8 * ((1 << s_) - 1) + (warp << s_) + i]; }, l, P);
#pragma unroll
        for (int j = 0; j < 8; j++)
            a[j] = fwd_finish<FAST>(a[j], P);
        op.store8(row, (b << kLocalLog) + 8 * l, a, P);
    }

    // ----------------------------------------------------------------------------------- inverse: local pass ----
    template <class Op>
    __global__ void __launch_bounds__(256) ntt_inv_local(Op op, const PrimeDev *__restrict__ primes, int na)
    {
        extern __shared__ __align__(16) unsigned char nl_smem[];
        u64(*xs)[256] = reinterpret_cast<u64(*)[256]>(nl_smem);
        Tw *tws = reinterpret_cast<Tw *>(nl_smem + 8 * 256 * 8);
        u64 *bar = reinterpret_cast<u64 *>(tws + 8 * 255);
        const int row = blockIdx.x, warp = threadIdx.x >> 5, l = threadIdx.x & 31;
        if (op.skip(row))
            return;
        const int b = blockIdx.y * 8 + warp;
        const PrimeDev P = primes[op.pid(row)];
        u64 *x = xs[warp];
        stage_local_twiddles(tws, bar, P.inv, na);
        // in-block stage s (2^s groups per block), group i of this warp's block
        auto tws_at = [&](int s_, int i) { return tws[8 * ((1 << s_) - 1) + (warp << s_) + i]; };

        u64 a[8];
        op.load8(row, (b << kLocalLog) + 8 * l, a, P);
        mbar_wait(bar, 0);
        {
            // strides 1,2,4
            auto twf = [&](int lvl, int k) { return tws_at(7 - lvl, (l << (2 - lvl)) + k); };
            inv_regs<0, false>(a, twf, P);
        }
#pragma unroll
        for (int j = 0; j < 8; j++)
            x[swz(8 * l + j)] = a[j];
        __syncwarp();
        {
            const int hi = l >> 3, lo = l & 7;
#pragma unroll
            for (int j = 0; j < 8; j++)
                a[j] = x[swz(64 * hi + lo + 8 * j)];
            // strides 8,16,32
            auto twf = [&](int lvl, int k) { return tws_at(4 - lvl, (hi << (2 - lvl)) + k); };
            inv_regs<0, false>(a, twf, P);
            __syncwarp();
#pragma unroll
            for (int j = 0; j < 8; j++)
                x[swz(64 * hi + lo + 8 * j)] = a[j];
        }
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 8; j++)
            a[j] = x[swz(l + 32 * j)];
        {
            // strides 64 (pairs j,j+2) and 128 (pairs j,j+4)
            auto twf = [&](int lvl, int k) { return tws_at(2 - lvl, k); };
            inv_regs<1, false>(a, twf, P);
        }
        u64 *mid = op.mid(row) + (b << kLocalLog);
#pragma unroll
        for (int j = 0; j < 8; j++)
            mid[l + 32 * j] = a[j];
    }

    // ---------------------------------------------------------------------------------- inverse: column pass ----
    // The log2(NA) column stages on one thread's 8 coefficients: in = layout r = 8*ridx + j, out = layout r = ridx + j*(NA/8),
    // reduced to [0, 2q).  The last read of the shared tile is not followed by a barrier.
    template <int LOGNA>
    __device__ __forceinline__ void inv_col_passes(u64 (&a)[8], u64 *tile, const Tw *tw_s, int ridx, int c, const PrimeDev &P)
    {
        constexpr int NA = 1 << LOGNA;
        constexpr int C = kTile / NA;
        constexpr int NSTL = LOGNA % 3; // stages in the (partial) last pass
        constexpr int NFULL = LOGNA / 3;
        int prev_g = 1;
#pragma unroll
        for (int p = 0; p < NFULL; p++)
        {
            const int U = 3 * p, g = 1 << U;
            const int rhi = ridx / g, rlo = ridx % g;
            if (p > 0)
            {
                const int prhi = ridx / prev_g, prlo = ridx % prev_g;
#pragma unroll
                for (int j = 0; j < 8; j++)
                    tile[(prhi * 8 * prev_g + prlo + j * prev_g) * C + c] = a[j];
                __syncthreads();
#pragma unroll
                for (int j = 0; j < 8; j++)
                    a[j] = tile[(rhi * 8 * g + rlo + j * g) * C + c];
                __syncthreads();
            }
            // level lvl has r-stride g<<lvl: m_r = NA >> (U+lvl+1), group = (rhi << (2-lvl)) + k
            auto twf = [&](int lvl, int k) { return tw_s[(NA >> (U + lvl + 1)) + (rhi << (2 - lvl)) + k]; };
            if (NSTL == 0 && p == NFULL - 1)
                inv_regs<0, true>(a, twf, P);
            else
                inv_regs<0, false>(a, twf, P);
            prev_g = g;
        }
        if (NSTL != 0)
        {
            constexpr int g = NA >> 3; // layout covering r-strides NA/8, NA/4, NA/2; run only the last NSTL of them
            {
                const int prhi = ridx / prev_g, prlo = ridx % prev_g;
#pragma unroll
                for (int j = 0; j < 8; j++)
                    tile[(prhi * 8 * prev_g + prlo + j * prev_g) * C + c] = a[j];
                __syncthreads();
#pragma unroll
                for (int j = 0; j < 8; j++)
                    a[j] = tile[(ridx + j * g) * C + c];
            }
            // level 1: r-stride NA/4 -> m_r = 2 ; level 2: r-stride NA/2 -> m_r = 1 (final)
            auto twf = [&](int lvl, int k) { return tw_s[(lvl == 1 ? 2 : 1) + k]; };
            inv_regs<3 - NSTL, true>(a, twf, P);
        }
        // (without a partial last pass the last layout is r = rhi*8g + rlo + j*g with g = NA/8, i.e. rhi = 0, rlo = ridx)
    }

    template <int LOGNA, class Op>
    __global__ void __launch_bounds__(kColThreads) ntt_inv_col(Op op, const PrimeDev *__restrict__ primes)
    {
        constexpr int NA = 1 << LOGNA;
        constexpr int C = kTile / NA;
        __shared__ __align__(16) u64 tile[kTile];
        __shared__ __align__(16) Tw tw_s[NA];
        __shared__ __align__(8) u64 bar;

        const int row = blockIdx.x, col0 = blockIdx.y * C;
        if (op.skip(row))
            return;
        const int tid = threadIdx.x, c = tid % C, ridx = tid / C;
        const PrimeDev P = primes[op.pid(row)];

        if (tid == 0)
            mbar_init(&bar, 1);
        __syncthreads();
        if (tid == 0)
        {
            mbar_expect_tx(&bar, NA * sizeof(Tw));
            tma_load_1d(tw_s, P.inv, NA * sizeof(Tw), &bar);
        }
        u64 a[8];
        const u64 *mid = op.mid(row);
#pragma unroll
        for (int j = 0; j < 8; j++)
            a[j] = mid[((8 * ridx + j) << kLocalLog) + col0 + c];
        mbar_wait(&bar, 0);

        inv_col_passes<LOGNA>(a, tile, tw_s, ridx, c, P);
#pragma unroll
        for (int j = 0; j < 8; j++)
            op.store1(row, ((ridx + j * (NA >> 3)) << kLocalLog) + col0 + c, a[j], P);
    }

    // ------------------------------------------------------------------- small transforms (n < 4096): one CTA/row ----
    template <class Op>
    __global__ void __launch_bounds__(256) ntt_fwd_small(Op op, const PrimeDev *__restrict__ primes, int logn)
    {
        extern __shared__ __align__(16) u64 s[];
        const int n = 1 << logn, row = blockIdx.x;
        if (op.skip(row))
            return;
        const PrimeDev P = primes[op.pid(row)];
        for (int i = threadIdx.x; i < n; i += blockDim.x)
            s[i] = op.load1(row, i, P);
        __syncthreads();
        for (int m = 1, gap = n >> 1; m < n; m <<= 1, gap >>= 1)
        {
            for (int k = threadIdx.x; k < (n >> 1); k += blockDim.x)
            {
                int i = k / gap, j = k % gap, pos = 2 * i * gap + j;
                ct_bfly<false>(s[pos], s[pos + gap], ldg_tw(P.fwd + m + i), P);
            }
            __syncthreads();
        }
        for (int i = threadIdx.x; i < n; i += blockDim.x)
            op.store1(row, i, csub(s[i], P.q4), P);
    }

    template <class Op>
    __global__ void __launch_bounds__(256) ntt_inv_small(Op op, const PrimeDev *__restrict__ primes, int logn)
    {
        extern __shared__ __align__(16) u64 s[];
        const int n = 1 << logn, row = blockIdx.x;
        if (op.skip(row))
            return;
        const PrimeDev P = primes[op.pid(row)];
        for (int i = threadIdx.x; i < n; i += blockDim.x)
            s[i] = op.load1(row, i, P);
        __syncthreads();
        for (int m = n >> 1, gap = 1; m >= 1; m >>= 1, gap <<= 1)
        {
            for (int k = threadIdx.x; k < (n >> 1); k += blockDim.x)
            {
                int i = k / gap, j = k % gap, pos = 2 * i * gap + j;
                if (m > 1)
                    gs_bfly(s[pos], s[pos + gap], ldg_tw(P.inv + m + i), P);
                else
                {
                    u64 u = s[pos], v = s[pos + gap];
                    s[pos] = csub(mul_shoup_lazy4(u + v, P.inv_n, P.nq), P.q2);
                    s[pos + gap] = csub(mul_shoup_lazy4(u - v + P.q4, P.inv_n_w, P.nq), P.q2);
                }
            }
            __syncthreads();
        }
        for (int i = threadIdx.x; i < n; i += blockDim.x)
            op.store1(row, i, s[i], P);
    }

    // ------------------------------------------------------------------------------------------- launchers ----
    // Launch bookkeeping + optional per-kernel CUDA-event timing (sb200_profile_* in the C-ABI).  Timing is recorded on
    // the launching stream; algorithmic bytes are what the kernel must move once (rows x 2 x n x 8 for a transform pass).
    struct LaunchStats
    {
        unsigned long long launches = 0;
        bool profiling = false;
        struct Rec
        {
            const char *name;
            int pass; // 0 = whole kernel, 1 = column pass of a transform, 2 = local pass
            double bytes;
            double bflys, macs; // modular butterflies / 64x64-bit multiply-accumulates the launch executes (second ceiling, SURVEY 8d)
            cudaEvent_t e0, e1;
            double bflys32 = 0, macs32 = 0; // 32-bit butterflies / 32x32->64 multiply-accumulates (integer key-switching path)
        };
        std::vector<Rec> recs;
        std::vector<cudaEvent_t> pool;
        cudaEvent_t get_event()
        {
            cudaEvent_t e;
            if (!pool.empty())
            {
                e = pool.back();
                pool.pop_back();
                return e;
            }
            cudaEventCreate(&e);
            return e;
        }
        void begin(const char *name, int pass, double bytes, cudaStream_t st, double bflys = 0, double macs = 0)
        {
            launches++;
            if (!profiling)
                return;
            Rec r{ name, pass, bytes, bflys, macs, get_event(), get_event() };
            cudaEventRecord(r.e0, st);
            recs.push_back(r);
        }
        void work32(double bflys32, double macs32)
        {
            if (profiling)
                recs.back().bflys32 = bflys32, recs.back().macs32 = macs32;
        }
        void end(cudaStream_t st)
        {
            if (profiling)
                cudaEventRecord(recs.back().e1, st);
        }
        void clear()
        {
            for (auto &r : recs)
            {
                pool.push_back(r.e0);
                pool.push_back(r.e1);
            }
            recs.clear();
        }
        ~LaunchStats()
        {
            clear();
            for (auto e : pool)
                cudaEventDestroy(e);
        }
    };

    template <class Op>
    inline cudaError_t launch_ntt_fwd(const Op &op, int nrows, int logn, const PrimeDev *primes, cudaStream_t st, LaunchStats &ls,
                                      const char *name = "ntt_fwd", int active_rows = -1, bool fast = false, bool local_only = false)
    {
        if (nrows <= 0)
            return cudaSuccess;
        const double arows = active_rows < 0 ? nrows : active_rows, bytes = 16.0 * arows * (1 << logn);
        const double bf_stage = arows * (1 << logn) / 2.0; // butterflies per stage
        if (logn < 12)
        {
            int n = 1 << logn, threads = n / 2 < 32 ? 32 : (n / 2 > 256 ? 256 : n / 2);
            ls.begin(name, 0, bytes, st, bf_stage * logn);
            ntt_fwd_small<Op><<<nrows, threads, n * sizeof(u64), st>>>(op, primes, logn);
            ls.end(st);
            return cudaGetLastError();
        }
        const int logna = logn - kLocalLog, na = 1 << logna;
        dim3 gc(nrows, (1 << kLocalLog) / (kTile / na));
        if (!local_only) // otherwise the caller's own column pass has written op.mid()
        {
            ls.begin(name, 1, bytes, st, bf_stage * logna); // column pass
            switch (logna)
            {
            case 4: fast ? ntt_fwd_col<4, true, Op><<<gc, kColThreads, 0, st>>>(op, primes) : ntt_fwd_col<4, false, Op><<<gc, kColThreads, 0, st>>>(op, primes); break;
            case 5: fast ? ntt_fwd_col<5, true, Op><<<gc, kColThreads, 0, st>>>(op, primes) : ntt_fwd_col<5, false, Op><<<gc, kColThreads, 0, st>>>(op, primes); break;
            case 6: fast ? ntt_fwd_col<6, true, Op><<<gc, kColThreads, 0, st>>>(op, primes) : ntt_fwd_col<6, false, Op><<<gc, kColThreads, 0, st>>>(op, primes); break;
            case 7: fast ? ntt_fwd_col<7, true, Op><<<gc, kColThreads, 0, st>>>(op, primes) : ntt_fwd_col<7, false, Op><<<gc, kColThreads, 0, st>>>(op, primes); break;
            case 8: fast ? ntt_fwd_col<8, true, Op><<<gc, kColThreads, 0, st>>>(op, primes) : ntt_fwd_col<8, false, Op><<<gc, kColThreads, 0, st>>>(op, primes); break;
            case 9: fast ? ntt_fwd_col<9, true, Op><<<gc, kColThreads, 0, st>>>(op, primes) : ntt_fwd_col<9, false, Op><<<gc, kColThreads, 0, st>>>(op, primes); break;
            default: return cudaErrorInvalidValue;
            }
            ls.end(st);
        }
        ls.begin(name, 2, bytes, st, bf_stage * kLocalLog); // local pass
        if (fast)
        {
            cudaFuncSetAttribute(ntt_fwd_local<true, Op>, cudaFuncAttributeMaxDynamicSharedMemorySize, kLocalSmem);
            ntt_fwd_local<true, Op><<<dim3(nrows, na / 8), 256, kLocalSmem, st>>>(op, primes, na);
        }
        else
        {
            cudaFuncSetAttribute(ntt_fwd_local<false, Op>, cudaFuncAttributeMaxDynamicSharedMemorySize, kLocalSmem);
            ntt_fwd_local<false, Op><<<dim3(nrows, na / 8), 256, kLocalSmem, st>>>(op, primes, na);
        }
        ls.end(st);
        return cudaGetLastError();
    }

    template <class Op>
    inline cudaError_t launch_ntt_inv(const Op &op, int nrows, int logn, const PrimeDev *primes, cudaStream_t st, LaunchStats &ls,
                                      const char *name = "ntt_inv", int active_rows = -1, bool local_only = false)
    {
        if (nrows <= 0)
            return cudaSuccess;
        const double arows = active_rows < 0 ? nrows : active_rows, bytes = 16.0 * arows * (1 << logn);
        const double bf_stage = arows * (1 << logn) / 2.0;
        if (logn < 12)
        {
            int n = 1 << logn, threads = n / 2 < 32 ? 32 : (n / 2 > 256 ? 256 : n / 2);
            ls.begin(name, 0, bytes, st, bf_stage * logn);
            ntt_inv_small<Op><<<nrows, threads, n * sizeof(u64), st>>>(op, primes, logn);
            ls.end(st);
            return cudaGetLastError();
        }
        const int logna = logn - kLocalLog, na = 1 << logna;
        ls.begin(name, 2, bytes, st, bf_stage * kLocalLog); // local pass
        cudaFuncSetAttribute(ntt_inv_local<Op>, cudaFuncAttributeMaxDynamicSharedMemorySize, kLocalSmem);
        ntt_inv_local<Op><<<dim3(nrows, na / 8), 256, kLocalSmem, st>>>(op, primes, na);
        ls.end(st);
        if (local_only)
            return cudaGetLastError(); // the caller runs its own column pass on op.mid()
        dim3 gc(nrows, (1 << kLocalLog) / (kTile / na));
        ls.begin(name, 1, bytes, st, bf_stage * logna); // column pass
        switch (logna)
        {
        case 4: ntt_inv_col<4, Op><<<gc, kColThreads, 0, st>>>(op, primes); break;
        case 5: ntt_inv_col<5, Op><<<gc, kColThreads, 0, st>>>(op, primes); break;
        case 6: ntt_inv_col<6, Op><<<gc, kColThreads, 0, st>>>(op, primes); break;
        case 7: ntt_inv_col<7, Op><<<gc, kColThreads, 0, st>>>(op, primes); break;
        case 8: ntt_inv_col<8, Op><<<gc, kColThreads, 0, st>>>(op, primes); break;
        case 9: ntt_inv_col<9, Op><<<gc, kColThreads, 0, st>>>(op, primes); break;
        default: return cudaErrorInvalidValue;
        }
        ls.end(st);
        return cudaGetLastError();
    }
} // namespace sb
