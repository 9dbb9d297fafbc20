// seal_b200/csrc/sb_ksint.cu -- key switching through an exact integer convolution on 29-bit auxiliary primes (sm_90a).
// Design and the reference lines it replaces: sb_ksint.cuh.  All kernels are integer-only; every word that leaves the path is
// a canonical residue mod q_i, identical to the reference's.
#include "sb_engine.cuh"
#include "sb_ksint.cuh"
#include <algorithm>
#include <cstdlib>

namespace sb
{
    // ---------------------------------------------------------------------------------- 32-bit lazy arithmetic ----
    struct P32
    {
        uint32_t p, p2, np; // p, 2p, 2^32 - p
    };
    __device__ __forceinline__ P32 make_p32(uint32_t p) { return P32{ p, 2 * p, 0u - p }; }
    // x in [0, 2m) -> [0, m)
    __device__ __forceinline__ uint32_t minsub(uint32_t x, uint32_t m) { return min(x, x - m); }
    // y * w mod p in [0, 2p) for ANY 32-bit y  (w < p, w.y = floor(w 2^32 / p)): one high + two low multiplies
    __device__ __forceinline__ uint32_t mul32_lazy(uint32_t y, uint2 w, uint32_t np) { return y * w.x + __umulhi(y, w.y) * np; }
    // forward (Cooley-Tukey), values in [0, 4p)
    __device__ __forceinline__ void ct32(uint32_t &x, uint32_t &y, uint2 w, const P32 &P)
    {
        const uint32_t u = minsub(x, P.p2), t = mul32_lazy(y, w, P.np);
        x = u + t;
        y = u - t + P.p2;
    }
    // inverse (Gentleman-Sande), values in [0, 2p)
    __device__ __forceinline__ void gs32(uint32_t &x, uint32_t &y, uint2 w, const P32 &P)
    {
        const uint32_t u = x + y, v = x - y + P.p2;
        x = minsub(u, P.p2);
        y = mul32_lazy(v, w, P.np);
    }
    // any 64-bit word -> [0, 4p)
    __device__ __forceinline__ uint32_t reduce64(u64 v, uint2 red, uint32_t mu, const P32 &P)
    {
        const uint32_t hi = static_cast<uint32_t>(v >> 32), lo = static_cast<uint32_t>(v);
        return mul32_lazy(hi, red, P.np) + (lo + __umulhi(lo, mu) * P.np);
    }

    // LOG stages on 2^LOG registers; tw(lvl, g): twiddle of group g (< 2^lvl) of level lvl.  One level per instantiation: the gap
    // is a compile-time constant, so every register index is one even inside a loop the compiler keeps rolled
    template <int LOG, int LVL = 0, class TwF>
    __device__ __forceinline__ void radix_fwd(uint32_t *a, TwF tw, const P32 &P)
    {
        if constexpr (LVL < LOG)
        {
            constexpr int gap = (1 << (LOG - 1)) >> LVL;
#pragma unroll
            for (int g = 0; g < (1 << LVL); g++)
            {
                const uint2 w = tw(LVL, g);
#pragma unroll
                for (int e = 0; e < gap; e++)
                    ct32(a[2 * g * gap + e], a[2 * g * gap + e + gap], w, P);
            }
            radix_fwd<LOG, LVL + 1>(a, tw, P);
        }
    }
    template <int LOG, int LVL = LOG - 1, class TwF>
    __device__ __forceinline__ void radix_inv(uint32_t *a, TwF tw, const P32 &P)
    {
        if constexpr (LVL >= 0)
        {
            constexpr int gap = (1 << (LOG - 1)) >> LVL;
#pragma unroll
            for (int g = 0; g < (1 << LVL); g++)
            {
                const uint2 w = tw(LVL, g);
#pragma unroll
                for (int e = 0; e < gap; e++)
                    gs32(a[2 * g * gap + e], a[2 * g * gap + e + gap], w, P);
            }
            radix_inv<LOG, LVL - 1>(a, tw, P);
        }
    }

    // ------------------------------------------------------------------------------ (1a) forward, outer pass ----
    // thread = coefficients j + 4096 e (e < 2^R) of one digit row: reduce the 64-bit words modulo every auxiliary prime and run the
    // R stages whose butterflies span more than a 4096-block.  grid.x = rows * 16.  Dh[t][out row][n], out rows per RowMap.
    struct RowMap
    {
        int mode, a, rows_out;
        // 0: identity; 1: digit rows (b, J) -> J * a + b (a = padded ciphertext count: the product kernel reads the ciphertexts of one
        // digit at constant strides); 2: key rows (J, c, ki) -> (J, c, (ki + 1) mod k), a = k: the special prime first, so that the
        // output primes of every level are consecutive rows
        __device__ __forceinline__ int out(int row, int b, int J) const
        {
            if (mode == 1)
                return J * a + b;
            if (mode == 2)
            {
                const int hi = row / a, ki = row - hi * a;
                return hi * a + (ki + 1 == a ? 0 : ki + 1);
            }
            return row;
        }
    };
    template <int R, bool PLAIN>
    __global__ void __launch_bounds__(256) ks32_fwd_outer(Src dsrc, int L, const PrimeDev *__restrict__ primes, KsIntParams prm,
                                                           const uint2 *__restrict__ tw_outer, uint32_t *__restrict__ Dh, RowMap map)
    {
        constexpr int E = 1 << R;
        const int row = blockIdx.x >> 4, j = ((blockIdx.x & 15) << 8) + threadIdx.x;
        const int b = row / L, J = row - b * L;
        u64 v[E];
        if (PLAIN)
        {
            const u64 *p = dsrc.row(b, J) + j;
#pragma unroll
            for (int e = 0; e < E; e++)
                v[e] = p[e << 12];
        }
        else
        {
            const u64 qJ = primes[J].q;
#pragma unroll
            for (int e = 0; e < E; e++)
                v[e] = dsrc.get(b, J, j + (e << 12), qJ);
        }
        const int orow = map.out(row, b, J);
        for (int t = 0; t < prm.S; t++)
        {
            const P32 P = make_p32(prm.p[t]);
            const uint2 red = prm.red[t];
            const uint32_t mu = prm.mu[t];
            uint32_t a[E];
#pragma unroll
            for (int e = 0; e < E; e++)
                a[e] = reduce64(v[e], red, mu, P);
            const uint2 *tw = tw_outer + (t << R);
            radix_fwd<R>(a, [&](int lvl, int g) { return __ldg(tw + (1 << lvl) + g); }, P);
            uint32_t *o = Dh + ((static_cast<size_t>(t) * map.rows_out + orow) << prm.logn) + j;
#pragma unroll
            for (int e = 0; e < E; e++)
                o[e << 12] = a[e];
        }
    }

    // ------------------------------------------- (1a') forward, outer pass, as the epilogue of the target's inverse column pass ----
    // The column pass of the 64-bit inverse transform of target row (b, J) owns the coefficients r 256 + col0 + c (r < NA, c < C);
    // with n = 4096 2^R the groups j + 4096 e (e < 2^R) of ks32_fwd_outer are among them.  The finished words go to the shared tile
    // and every (group, auxiliary prime) pair leaves it as the words ks32_fwd_outer forms from them: the digits D are never written.
    template <int LOGNA>
    __global__ void __launch_bounds__(kColThreads) ks32_intt_fwd_outer(OpKsIntt op, const PrimeDev *__restrict__ primes, KsIntParams prm,
                                                                        const uint2 *__restrict__ tw_outer, uint32_t *__restrict__ Dh, RowMap map)
    {
        constexpr int NA = 1 << LOGNA, C = kTile / NA, R = LOGNA - 4, E = 1 << R, G = kTile / E;
        __shared__ __align__(16) u64 tile[kTile];
        __shared__ __align__(16) Tw tw_s[NA];
        __shared__ __align__(8) u64 bar;
        const int row = blockIdx.x, col0 = blockIdx.y * C, tid = threadIdx.x, c = tid % C, ridx = tid / C;
        const int b = row / op.L, J = row - b * op.L;
        const PrimeDev P = primes[J];
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
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 8; j++)
            tile[(ridx + j * (NA >> 3)) * C + c] = csub(a[j], P.q);
        __syncthreads();
        const int orow = map.out(row, b, J);
#pragma unroll 1
        for (int w = tid; w < G * prm.S; w += kColThreads)
        {
            const int t = w / G, grp = w - t * G, rl = grp / C, cc = grp - rl * C;
            const P32 Pt = make_p32(prm.p[t]);
            const uint2 red = prm.red[t];
            const uint32_t mu = prm.mu[t];
            uint32_t x[E];
#pragma unroll
            for (int e = 0; e < E; e++)
                x[e] = reduce64(tile[(rl + 16 * e) * C + cc], red, mu, Pt);
            const uint2 *tw = tw_outer + (t << R);
            radix_fwd<R>(x, [&](int lvl, int g) { return __ldg(tw + (1 << lvl) + g); }, Pt);
            uint32_t *o = Dh + ((static_cast<size_t>(t) * map.rows_out + orow) << prm.logn) + (rl << kLocalLog) + col0 + cc;
#pragma unroll
            for (int e = 0; e < E; e++)
                o[e << 12] = x[e];
        }
    }

    // -------------------------------------------------------------------------------- local passes (12 stages) ----
    // One CTA (256 threads) transforms up to kRowsPerCta 4096-word blocks (one per row, 16 KB, contiguous) with three radix-16
    // register passes each.  The blocks stream through a ring of kRing linear buffers: one thread loads each block with a bulk
    // asynchronous copy (mbarrier completion) kRing - 1 blocks ahead and stores the result from the same buffer with a bulk copy, so
    // the global traffic is whole lines and the next block is in flight while the current one is transformed.  The block's 4095
    // twiddles are the same for every row: staged once per CTA with one bulk copy (32 KB).  The exchanges between passes go through
    // a tile in the layout idx ^ (bit 8 -> bit 4) ^ (bits 5,6 -> bits 2,3).  Every shared-memory access is conflict-free, on the
    // tile and on the linear buffers: lanes consecutive (tid + 256 e), half-warps 256 apart (pass 2), and 16 consecutive words per
    // lane as 4 x 16 B, visited in the order h ^ hx.
    constexpr int kRowsPerCta = 16, kRing = 3;
    constexpr int kKsLocalSmem = 4096 * 8 + 4096 * 4 + kRing * 4096 * 4 + (kRing + 1) * 8;
    __device__ __forceinline__ int swz32(int idx) { return idx ^ (((idx >> 8) & 1) << 4) ^ (((idx >> 5) & 3) << 2); }

    // a[4 h + i] <-> a[4 (h ^ x) + i]: the 16-byte groups of a lane's words in the order its accesses of a linear buffer visit them
    // (x varies across the lanes: selects, not a register index that only the run time knows)
    __device__ __forceinline__ void xor_groups(uint32_t (&a)[16], int x)
    {
        const bool s1 = x & 1, s2 = x & 2;
#pragma unroll
        for (int i = 0; i < 4; i++)
        {
#pragma unroll
            for (int h = 0; h < 4; h += 2)
            {
                const uint32_t u = a[4 * h + i], v = a[4 * h + 4 + i];
                a[4 * h + i] = s1 ? v : u, a[4 * h + 4 + i] = s1 ? u : v;
            }
#pragma unroll
            for (int h = 0; h < 2; h++)
            {
                const uint32_t u = a[4 * h + i], v = a[4 * h + 8 + i];
                a[4 * h + i] = s2 ? v : u, a[4 * h + 8 + i] = s2 ? u : v;
            }
        }
    }

    // rows: row rr of this launch lives at data + ((rr * rstride + t) << logn).  In place.  One-dimensional grid, the block index of
    // the row (auxiliary prime t, 4096-word block g; S * 2^r of them) fastest: the CTAs in flight together cover a few groups of
    // consecutive rows completely instead of one block of many rows that lie tstride or rstride rows apart
    // Forward: outputs canonical.  Inverse: inputs in [0, 2p), outputs in [0, 2p) (the scaling by n^-1 is folded into the CRT
    // constants)
    template <bool INV>
    __device__ __forceinline__ void ks32_local(uint32_t *__restrict__ data, int rows, long long rstride, long long tstride,
                                               const KsIntParams &prm, const uint2 *__restrict__ tw_local)
    {
        extern __shared__ __align__(16) unsigned char ks32_smem[];
        uint2 *tws = reinterpret_cast<uint2 *>(ks32_smem);
        uint32_t *xs = reinterpret_cast<uint32_t *>(ks32_smem + 4096 * 8);
        uint32_t *ring = xs + 4096;
        u64 *bar = reinterpret_cast<u64 *>(ring + kRing * 4096); // [0]: twiddles, [1 + s]: ring buffer s
        const int ntg = prm.S << prm.r, tg = blockIdx.x % ntg, t = tg >> prm.r, g = tg - (t << prm.r), tid = threadIdx.x;
        const int row0 = blockIdx.x / ntg * kRowsPerCta, nrows = min(rows - row0, kRowsPerCta);
        auto block = [&](int i) { return data + (((row0 + i) * rstride + t * tstride) << prm.logn) + (g << 12); };
        auto fetch = [&](int i) {
            u64 *b = bar + 1 + i % kRing;
            mbar_expect_tx(b, 4096 * 4);
            tma_load_1d(ring + (i % kRing) * 4096, block(i), 4096 * 4, b);
        };
        if (tid == 0)
            for (int s = 0; s <= kRing; s++)
                mbar_init(bar + s, 1);
        __syncthreads();
        if (tid == 0)
        {
            mbar_expect_tx(bar, 4096 * 8);
            tma_load_1d(tws, tw_local + (static_cast<size_t>(tg) << 12), 4096 * 8, bar);
            for (int i = 0; i < min(nrows, kRing - 1); i++)
                fetch(i);
        }
        const P32 P = make_p32(prm.p[t]);
        const int blk = tid >> 4, l16 = tid & 15;
        const int p3 = ((16 * tid) ^ (((tid >> 4) & 1) << 4)), hx = (tid >> 1) & 3;
        mbar_wait(bar, 0);
        for (int i = 0; i < nrows; i++)
        {
            uint32_t *buf = ring + (i % kRing) * 4096;
            mbar_wait(bar + 1 + i % kRing, (i / kRing) & 1);
            uint32_t a[16];
            if constexpr (!INV)
            {
#pragma unroll
                for (int e = 0; e < 16; e++)
                    a[e] = buf[tid + 256 * e];
                radix_fwd<4>(a, [&](int lvl, int gg) { return tws[(1 << lvl) + gg]; }, P);
#pragma unroll
                for (int e = 0; e < 16; e++)
                    xs[swz32(tid + 256 * e)] = a[e];
                __syncthreads();
#pragma unroll
                for (int e = 0; e < 16; e++)
                    a[e] = xs[swz32((blk << 8) + l16 + 16 * e)];
                radix_fwd<4>(a, [&](int lvl, int gg) { return tws[(16 << lvl) + (blk << lvl) + gg]; }, P);
#pragma unroll
                for (int e = 0; e < 16; e++)
                    xs[swz32((blk << 8) + l16 + 16 * e)] = a[e];
                __syncthreads();
#pragma unroll
                for (int h = 0; h < 4; h++)
                {
                    const uint4 q = *reinterpret_cast<const uint4 *>(xs + p3 + 4 * (h ^ hx));
                    a[4 * h] = q.x, a[4 * h + 1] = q.y, a[4 * h + 2] = q.z, a[4 * h + 3] = q.w;
                }
                radix_fwd<4>(a, [&](int lvl, int gg) { return tws[256 + (((1 << lvl) - 1 + gg) << 8) + tid]; }, P);
#pragma unroll
                for (int e = 0; e < 16; e++)
                    a[e] = minsub(minsub(a[e], P.p2), P.p); // canonical: the multiply-accumulate sums L products in 64 bits
                xor_groups(a, hx);
#pragma unroll
                for (int h = 0; h < 4; h++)
                    *reinterpret_cast<uint4 *>(buf + 16 * tid + 4 * (h ^ hx)) = make_uint4(a[4 * h], a[4 * h + 1], a[4 * h + 2], a[4 * h + 3]);
            }
            else
            {
#pragma unroll
                for (int h = 0; h < 4; h++)
                {
                    const uint4 q = *reinterpret_cast<const uint4 *>(buf + 16 * tid + 4 * (h ^ hx));
                    a[4 * h] = q.x, a[4 * h + 1] = q.y, a[4 * h + 2] = q.z, a[4 * h + 3] = q.w;
                }
                xor_groups(a, hx);
                radix_inv<4>(a, [&](int lvl, int gg) { return tws[256 + (((1 << lvl) - 1 + gg) << 8) + tid]; }, P);
#pragma unroll
                for (int h = 0; h < 4; h++)
                    *reinterpret_cast<uint4 *>(xs + p3 + 4 * (h ^ hx)) = make_uint4(a[4 * h], a[4 * h + 1], a[4 * h + 2], a[4 * h + 3]);
                __syncthreads();
#pragma unroll
                for (int e = 0; e < 16; e++)
                    a[e] = xs[swz32((blk << 8) + l16 + 16 * e)];
                radix_inv<4>(a, [&](int lvl, int gg) { return tws[(16 << lvl) + (blk << lvl) + gg]; }, P);
#pragma unroll
                for (int e = 0; e < 16; e++)
                    xs[swz32((blk << 8) + l16 + 16 * e)] = a[e];
                __syncthreads();
#pragma unroll
                for (int e = 0; e < 16; e++)
                    a[e] = xs[swz32(tid + 256 * e)];
                radix_inv<4>(a, [&](int lvl, int gg) { return tws[(1 << lvl) + gg]; }, P);
#pragma unroll
                for (int e = 0; e < 16; e++)
                    buf[tid + 256 * e] = a[e];
            }
            // the buffer goes out once every thread's words are in it; the tile is free for the next row
            fence_proxy_async();
            __syncthreads();
            if (tid == 0)
            {
                tma_store_1d(block(i), buf, 4096 * 4);
                if (i + kRing - 1 < nrows)
                {
                    bulk_wait_read<1>(); // the buffer of row i + kRing - 1 last held row i - 1: its store has read it
                    fetch(i + kRing - 1);
                }
            }
        }
        if (tid == 0)
            bulk_wait<0>(); // no store may still read shared memory when the CTA exits
    }
    __global__ void __launch_bounds__(256, 2) ks32_fwd_local(uint32_t *__restrict__ data, int rows, long long rstride, long long tstride,
                                                              KsIntParams prm, const uint2 *__restrict__ tw_local)
    {
        ks32_local<false>(data, rows, rstride, tstride, prm, tw_local);
    }
    __global__ void __launch_bounds__(256, 2) ks32_inv_local(uint32_t *__restrict__ data, int rows, long long rstride, long long tstride,
                                                              KsIntParams prm, const uint2 *__restrict__ tw_local)
    {
        ks32_local<true>(data, rows, rstride, tstride, prm, tw_local);
    }

    // ------------------------------------------------------------------------------ (3b) inverse, outer pass ----
    // rows (b, c, I, t): row % S = auxiliary prime.  In place.  grid.x = rows * 16
    template <int R>
    __global__ void __launch_bounds__(256) ks32_inv_outer(uint32_t *__restrict__ data, KsIntParams prm, const uint2 *__restrict__ tw_outer)
    {
        constexpr int E = 1 << R;
        const int row = blockIdx.x >> 4, j = ((blockIdx.x & 15) << 8) + threadIdx.x;
        const int t = row % prm.S;
        const P32 P = make_p32(prm.p[t]);
        uint32_t *o = data + (static_cast<size_t>(row) << prm.logn) + j;
        uint32_t a[E];
#pragma unroll
        for (int e = 0; e < E; e++)
            a[e] = o[e << 12];
        const uint2 *tw = tw_outer + (t << R);
        radix_inv<R>(a, [&](int lvl, int g) { return __ldg(tw + (1 << lvl) + g); }, P);
#pragma unroll
        for (int e = 0; e < E; e++)
            o[e << 12] = a[e];
    }

    // ----------------------------------------------------------------------------- (2) multiply-accumulate ----
    // Acc[b][c][I'][t][x] = sum_J Dh[t][J][b][x] * key32[t][J][c][I'][x]  mod p_t  (-> [0, 2p));  I' = 0: the special prime,
    // I' = i + 1: data prime i (so the L + 1 outputs of every level are consecutive key rows).
    // lane = coefficient; a warp owns a register tile of TB ciphertexts x TC outputs (one component c); the 4 warps of a CTA take 4
    // output tiles over the same 32 coefficients and ciphertexts, and consecutive CTAs (other ciphertexts, same key tile) share the
    // key through L2.  Every operand word is a 128-byte line of its own row (rows are 4 n bytes apart): the loads are latency-bound
    // (ncu: long-scoreboard stalls), so the operands of the next kStages - 1 digits are kept in flight with cp.async into a
    // per-thread ring in shared memory -- each lane copies and later reads only its own words, no barrier is involved -- and the
    // products read them from there.  LOGN is a template parameter: every copy has an immediate offset from one of two pointers that
    // advance once per digit.  No reduction inside the loop: L p^2 < 2^64.
    constexpr int kMacTB = 4, kMacTC = 8, kMacStages = 8;
    constexpr int kMacSmem = kMacStages * (kMacTB + kMacTC) * 128 * 4;
    __device__ __forceinline__ void cp_async4(uint32_t *dst_smem, const uint32_t *src)
    {
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
    }
    template <int LOGN>
    __global__ void __launch_bounds__(128, 3) ks32_mac(const uint32_t *__restrict__ Dh, const uint32_t *__restrict__ key32, uint32_t *__restrict__ Acc,
                                                        KsIntParams prm, int L, int k, int digits, int B, int nbt)
    {
        constexpr int TB = kMacTB, TC = kMacTC, D = kMacStages, W = TB + TC;
        extern __shared__ __align__(16) uint32_t ks_ring[]; // [stage][word W][thread 128]
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        // CTA order: ciphertext tile fastest (same key tile: L2), then the output-tile group (same digit words: L2), then coefficients
        const int ntile = (L + TC) / TC; // tiles per component: ceil((L + 1) / TC)
        const int ny = (2 * ntile + 3) / 4;
        const int bt = blockIdx.x % nbt, yg = (blockIdx.x / nbt) % ny, xt = blockIdx.x / (nbt * ny), t = blockIdx.z;
        const int task = yg * 4 + warp;
        if (task >= 2 * ntile)
            return;
        const int c = task / ntile, i0 = (task - c * ntile) * TC, b0 = bt * TB, Bpad = nbt * TB;
        const int x = (xt << 5) + lane;
        const uint32_t *dp = Dh + ((static_cast<size_t>(t) * L * Bpad + b0) << LOGN) + x;
        const uint32_t *kp = key32 + (((static_cast<size_t>(t) * digits * 2 + c) * k + i0) << LOGN) + x;
        const size_t dstep = static_cast<size_t>(Bpad) << LOGN, kstep = static_cast<size_t>(2 * k) << LOGN;
        uint32_t *ring = ks_ring + threadIdx.x;
        u64 acc[TB][TC];
#pragma unroll
        for (int i = 0; i < TB; i++)
#pragma unroll
            for (int r = 0; r < TC; r++)
                acc[i][r] = 0;
        int Jissue = 0;
        auto issue = [&]() { // operands of digit Jissue -> stage Jissue % D (an empty group once the digits are exhausted)
            if (Jissue < L)
            {
                uint32_t *dst = ring + (Jissue & (D - 1)) * (W * 128);
#pragma unroll
                for (int i = 0; i < TB; i++)
                    cp_async4(dst + i * 128, dp + (i << LOGN));
#pragma unroll
                for (int r = 0; r < TC; r++)
                    cp_async4(dst + (TB + r) * 128, kp + (r << LOGN));
                dp += dstep, kp += kstep;
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
            Jissue++;
        };
        uint32_t dA[TB], kA[TC], dB[TB], kB[TC];
        auto fetch = [&](uint32_t(&d_)[TB], uint32_t(&k_)[TC], int J) {
            const uint32_t *src = ring + (J & (D - 1)) * (W * 128);
#pragma unroll
            for (int i = 0; i < TB; i++)
                d_[i] = src[i * 128];
#pragma unroll
            for (int r = 0; r < TC; r++)
                k_[r] = src[(TB + r) * 128];
        };
        auto macs = [&](const uint32_t(&d_)[TB], const uint32_t(&k_)[TC]) {
#pragma unroll
            for (int i = 0; i < TB; i++)
#pragma unroll
                for (int r = 0; r < TC; r++)
                    asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[i][r]) : "r"(d_[i]), "r"(k_[r]));
        };
#pragma unroll
        for (int j = 0; j < D - 1; j++)
            issue();
        // invariant at the top of an iteration: groups 0 .. J + D - 2 committed; "wait_group D - 2" leaves digit J complete
        asm volatile("cp.async.wait_group %0;" ::"n"(D - 2) : "memory");
        fetch(dA, kA, 0);
        int J = 0;
#pragma unroll 1
        for (; J + 2 <= L; J += 2)
        {
            issue();
            asm volatile("cp.async.wait_group %0;" ::"n"(D - 2) : "memory");
            fetch(dB, kB, J + 1);
            macs(dA, kA);
            issue();
            asm volatile("cp.async.wait_group %0;" ::"n"(D - 2) : "memory");
            fetch(dA, kA, J + 2); // digit L (one past the end) reads a stale stage; its products are never formed
            macs(dB, kB);
        }
        if (J < L)
            macs(dA, kA);
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        const P32 P = make_p32(prm.p[t]);
        const uint2 red = prm.red[t];
        const uint32_t mu = prm.mu[t];
#pragma unroll
        for (int i = 0; i < TB; i++)
        {
            if (b0 + i < B)
            {
                uint32_t *o = Acc + ((((static_cast<size_t>(b0 + i) * 2 + c) * (L + 1) + i0) * prm.S + t) << LOGN) + x;
#pragma unroll
                for (int r = 0; r < TC; r++)
                    if (i0 + r <= L)
                        o[(static_cast<size_t>(r) * prm.S) << LOGN] = minsub(reduce64(acc[i][r], red, mu, P), P.p2);
            }
        }
    }
    // The same product with the key tile in shared memory: a CTA (16 warps = 4 ciphertext tiles x 4 output tiles) owns 32
    // coefficients x 32 outputs of one auxiliary prime, copies the L x 32 key rows of that tile (L x 4 KB) into shared memory once and
    // then walks over ALL ciphertexts of the chunk, 16 per iteration.  Key words come from shared memory (conflict-free: lanes =
    // consecutive words); only the digit words (4 per digit and thread) travel through the cp.async ring, so the number of global
    // requests in flight per multiply-accumulate is a third of the register-tile kernel's -- that kernel is bound by request
    // latency x requests in flight (ncu: the first product after each operand fetch holds half of the stall samples).
    // grid = (output groups * n/32, 1, S); dynamic shared memory L * 4096 + ring bytes.
    constexpr int kMacRingBytes = kMacStages * kMacTB * 512 * 4;
    template <int LOGN>
    __global__ void __launch_bounds__(512, 1) ks32_mac_tile(const uint32_t *__restrict__ Dh, const uint32_t *__restrict__ key32, uint32_t *__restrict__ Acc,
                                                             KsIntParams prm, int L, int k, int digits, int B, int Bpad)
    {
        constexpr int TB = kMacTB, TC = kMacTC, D = kMacStages;
        extern __shared__ __align__(16) uint32_t ks_tile[]; // [J][32 rows][32 lanes] | ring [stage][TB][512 threads]
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        const int ntile = (L + TC) / TC, ny = (2 * ntile + 3) / 4;
        const int yg = blockIdx.x % ny, xt = blockIdx.x / ny, t = blockIdx.z;
        const int x = (xt << 5) + lane;
        const uint32_t *kbase = key32 + ((static_cast<size_t>(t) * digits * 2 * k) << LOGN) + x;
        const size_t kstep = static_cast<size_t>(2 * k) << LOGN;
        // tile rows: row tr (< 32) = output r = tr % 8 of task yg * 4 + tr / 8; unused tasks of a ragged last group re-read valid rows
        // (asynchronous copies: all of a warp's rows are in flight together instead of one load-store round trip per row)
        for (int rho = warp; rho < L * 32; rho += 16)
        {
            const int J = rho >> 5, tr = rho & 31;
            const int task = min(yg * 4 + (tr >> 3), 2 * ntile - 1), c = task / ntile, i0 = (task - c * ntile) * TC;
            // tile layout [J][output tile][half][lane][4 words]: a lane's 8 key words of a digit are two 16-byte reads
            cp_async4(ks_tile + ((((J << 3) + (tr >> 2)) << 5) + lane) * 4 + (tr & 3),
                      kbase + J * kstep + (static_cast<size_t>(c * k + i0 + (tr & 7)) << LOGN));
        }
        asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
        __syncthreads();
        const int bsub = warp & 3, icsub = warp >> 2;
        const int task = yg * 4 + icsub;
        if (task >= 2 * ntile)
            return;
        const int c = task / ntile, i0 = (task - c * ntile) * TC;
        const uint32_t *ktile = ks_tile + (((icsub * 2) << 5) + lane) * 4; // + J * 1024 words per digit, + 128 words for the second half
        uint32_t *ring = ks_tile + L * 1024 + threadIdx.x * 4;           // [stage][thread][TB words]
        const P32 P = make_p32(prm.p[t]);
        const uint2 red = prm.red[t];
        const uint32_t mu = prm.mu[t];
        const size_t dstep = static_cast<size_t>(Bpad) << LOGN;
        for (int b0 = bsub * TB; b0 < B; b0 += 4 * TB)
        {
            const uint32_t *dp = Dh + ((static_cast<size_t>(t) * L * Bpad + b0) << LOGN) + x;
            u64 acc[TB][TC];
#pragma unroll
            for (int i = 0; i < TB; i++)
#pragma unroll
                for (int r = 0; r < TC; r++)
                    acc[i][r] = 0;
            // The digits are consumed in pairs: the two products that go to one accumulator sit next to each other, so ptxas forms them
            // with zero addends and adds both with ONE three-input 64-bit add (2.0 instructions per multiply-accumulate; one digit at a
            // time costs 3.0, and this kernel is bound by instruction issue: ncu).  The loop is unrolled by the ring depth, so stage
            // offsets are compile-time constants.  One cp.async group = four digits (two pairs); the next group is in flight.
            auto issue_quad = [&](int stage, int J) { // digits J .. J + 3 -> stages `stage` .. `stage + 3`: one cp.async group
#pragma unroll
                for (int h = 0; h < 4; h++)
                    if (J + h < L)
                    {
                        uint32_t *dst = ring + (stage + h) * (TB * 512);
#pragma unroll
                        for (int i = 0; i < TB; i++)
                            cp_async4(dst + i, dp + (i << LOGN));
                        dp += dstep;
                    }
                asm volatile("cp.async.commit_group;" ::: "memory");
            };
            static_assert(TB == 4 && TC == 8 && D == 8, "operand fetches are 16-byte reads; the ring holds two groups of four digits");
            auto pair_step = [&](int stage, const uint32_t *kt, bool both) {
                uint32_t d0[TB], k0[TC], d1[TB], k1[TC];
                const uint32_t *src = ring + stage * (TB * 512);
                const uint4 da = *reinterpret_cast<const uint4 *>(src), db = *reinterpret_cast<const uint4 *>(src + TB * 512);
                const uint4 ka = *reinterpret_cast<const uint4 *>(kt), kb = *reinterpret_cast<const uint4 *>(kt + 128);
                const uint4 kc = *reinterpret_cast<const uint4 *>(kt + 1024), kd = *reinterpret_cast<const uint4 *>(kt + 1024 + 128);
                d0[0] = da.x, d0[1] = da.y, d0[2] = da.z, d0[3] = da.w, d1[0] = db.x, d1[1] = db.y, d1[2] = db.z, d1[3] = db.w;
                k0[0] = ka.x, k0[1] = ka.y, k0[2] = ka.z, k0[3] = ka.w, k0[4] = kb.x, k0[5] = kb.y, k0[6] = kb.z, k0[7] = kb.w;
                k1[0] = kc.x, k1[1] = kc.y, k1[2] = kc.z, k1[3] = kc.w, k1[4] = kd.x, k1[5] = kd.y, k1[6] = kd.z, k1[7] = kd.w;
                if (both)
                {
#pragma unroll
                    for (int i = 0; i < TB; i++)
#pragma unroll
                        for (int r = 0; r < TC; r++)
                        {
                            asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[i][r]) : "r"(d0[i]), "r"(k0[r]));
                            asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[i][r]) : "r"(d1[i]), "r"(k1[r]));
                        }
                }
                else
                {
#pragma unroll
                    for (int i = 0; i < TB; i++)
#pragma unroll
                        for (int r = 0; r < TC; r++)
                            asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[i][r]) : "r"(d0[i]), "r"(k0[r]));
                }
            };
            issue_quad(0, 0);
            const uint32_t *kt = ktile;
#pragma unroll 1
            for (int J0 = 0; J0 < L; J0 += D)
            {
#pragma unroll
                for (int u = 0; u < D; u += 4)
                {
                    const int J = J0 + u;
                    if (J >= L)
                        break;
                    issue_quad((u + 4) & (D - 1), J + 4);
                    asm volatile("cp.async.wait_group 1;" ::: "memory"); // the four digits of this step have landed
                    pair_step(u, kt, J + 1 < L);
                    if (J + 2 < L)
                        pair_step(u + 2, kt + 2048, J + 3 < L);
                    kt += 4096;
                }
            }
            asm volatile("cp.async.wait_group 0;" ::: "memory");
#pragma unroll
            for (int i = 0; i < TB; i++)
            {
                if (b0 + i < B)
                {
                    uint32_t *o = Acc + ((((static_cast<size_t>(b0 + i) * 2 + c) * (L + 1) + i0) * prm.S + t) << LOGN) + x;
#pragma unroll
                    for (int r = 0; r < TC; r++)
                        if (i0 + r <= L)
                            o[(static_cast<size_t>(r) * prm.S) << LOGN] = minsub(reduce64(acc[i][r], red, mu, P), P.p2);
                }
            }
        }
    }
    // The same product on the INT8 tensor cores.  For one auxiliary prime t and coefficient x the sum is a small integer GEMM,
    // [B x L] . [L x 2(L+1)] (ciphertexts x digits, digits x outputs).  Every canonical 29-bit word splits into four u8 limbs; the 16
    // limb-pair products of one m16n8k32 step go to 7 s32 class accumulators C_s = sum_{l+m=s} sum_J d_l k_m, each below
    // 4 * 32 * 255^2 < 2^31 (no wrap whatever the words), and sum_s C_s 2^(8s) is the exact 64-bit sum ks32_mac_tile forms: the same
    // Acc words.  A CTA (8 warps) owns 8 coefficients of one auxiliary prime -- 32-byte runs of every Acc row -- and all outputs.  It
    // stages the key of its coefficients once, split into limb planes in B-fragment order, and walks the chunk 16 ciphertexts at a
    // time: the digit tile of the next 16 arrives by cp.async while the current one is byte-transposed into A fragments (one pass,
    // shared by all output tiles) and multiplied.  Warp w takes output tiles w, w + 8 for all 8 coefficients, so a thread ends with
    // the 8 consecutive x of each of its Acc rows (one 32-byte sector; stored by two lanes).  One K step: L <= 32 digits, and digits
    // J >= L meet zero key limbs.  Shared memory 112 KB at L = 31: two CTAs per SM.
    constexpr int kMmaX = 8, kMmaMaxDigits = 32;
    constexpr int kMmaAfStride = 4 * 128 + 4; // words of one coefficient's A fragments; +4: the transposition's writes are conflict-free
    constexpr size_t mac_mma_smem(int nt) { return static_cast<size_t>(nt) * 8192 + 2 * 16384 + kMmaX * kMmaAfStride * 4; }
    __device__ __forceinline__ void cp_async16(uint32_t *dst_smem, const uint32_t *src)
    {
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
    }
    // 4 x 4 byte transpose: byte j of l[m] = byte m of w[j] (limb m of four consecutive digits: one fragment register)
    __device__ __forceinline__ void limbs4(const uint32_t (&w)[4], uint32_t (&l)[4])
    {
        const uint32_t t0 = __byte_perm(w[0], w[1], 0x5140), t1 = __byte_perm(w[0], w[1], 0x7362);
        const uint32_t t2 = __byte_perm(w[2], w[3], 0x5140), t3 = __byte_perm(w[2], w[3], 0x7362);
        l[0] = __byte_perm(t0, t2, 0x5410), l[1] = __byte_perm(t0, t2, 0x7632);
        l[2] = __byte_perm(t1, t3, 0x5410), l[3] = __byte_perm(t1, t3, 0x7632);
    }
    __device__ __forceinline__ void mma_u8(uint32_t (&c)[4], const uint4 &a, const uint2 &b)
    {
        asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
            : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
            : "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w), "r"(b.x), "r"(b.y));
    }
    __device__ __forceinline__ u64 madw(uint32_t a, uint32_t b, u64 c)
    {
        asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(c) : "r"(a), "r"(b));
        return c;
    }
    // grid = (n / 8, S); dynamic shared memory mac_mma_smem(ceil(2 (L + 1) / 8))
    template <int LOGN>
    __global__ void __launch_bounds__(256, 2) ks32_mac_mma(const uint32_t *__restrict__ Dh, const uint32_t *__restrict__ key32, uint32_t *__restrict__ Acc,
                                                            KsIntParams prm, int L, int k, int digits, int B, int Bpad)
    {
        extern __shared__ __align__(16) unsigned char ks_mma_smem[];
        const int NO = 2 * (L + 1), NT = (NO + 7) / 8;
        uint2 *kf = reinterpret_cast<uint2 *>(ks_mma_smem);                  // [x][output tile][limb][lane]
        uint32_t *ds = reinterpret_cast<uint32_t *>(ks_mma_smem + NT * 8192); // [stage][J][b][x]: 16-byte chunks, swizzled
        uint32_t *af = ds + 2 * 4096;                                          // [x][limb][lane][4], kMmaAfStride words per x
        const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
        const int x0 = blockIdx.x * kMmaX, t = blockIdx.y;
        // digit rows (J, b0 + b) -> stage; chunk h of row (J, b) goes to chunk q ^ (b bit 3 -> bit 2) ^ (J bit 4 -> bit 0) so that the
        // transposition's reads are conflict-free.  Rows past Bpad and digits past L are not copied: their stale words meet only
        // products that are never stored, or zero key limbs
        const uint32_t *dbase = Dh + ((static_cast<size_t>(t) * L * Bpad) << LOGN) + x0;
        auto load_tile = [&](int b0, int stage) {
            uint32_t *dst = ds + stage * 4096;
            for (int it = tid; it < L * 32; it += 256)
            {
                const int J = it >> 5, b = (it >> 1) & 15, h = it & 1;
                if (b0 + b < Bpad)
                {
                    const int q = ((J * 16 + b) * 2 + h) ^ (((b >> 3) & 1) << 2) ^ ((J >> 4) & 1);
                    cp_async16(dst + q * 4, dbase + ((static_cast<size_t>(J) * Bpad + b0 + b) << LOGN) + 4 * h);
                }
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
        };
        load_tile(0, 0);
        // the key of the 8 coefficients: lane (g, i) of output tile nt holds limb m of digits 4i .. 4i + 3 and 16 + 4i .. 16 + 4i + 3
        // of output 8 nt + g (output o = c (L + 1) + I' is key row c k + I'); four items' loads are in flight together
        {
            const uint32_t *kbase = key32 + ((static_cast<size_t>(t) * digits * 2 * k) << LOGN) + x0;
            for (int it0 = tid; it0 < NT * 256; it0 += 4 * 256)
            {
                uint32_t w[4][2][4];
#pragma unroll
                for (int u = 0; u < 4; u++)
                {
                    const int it = it0 + u * 256, x = it & 7, ln = (it >> 3) & 31, o = 8 * (it >> 8) + (ln >> 2);
                    const int c = o > L ? 1 : 0, row = c * k + o - c * (L + 1);
#pragma unroll
                    for (int hh = 0; hh < 2; hh++)
#pragma unroll
                        for (int j = 0; j < 4; j++)
                        {
                            const int J = 16 * hh + 4 * (ln & 3) + j;
                            w[u][hh][j] = (it < NT * 256 && J < L && o < NO) ? __ldg(kbase + (static_cast<size_t>(J * 2 * k + row) << LOGN) + x) : 0;
                        }
                }
#pragma unroll
                for (int u = 0; u < 4; u++)
                {
                    const int it = it0 + u * 256;
                    if (it < NT * 256)
                    {
                        uint32_t l0[4], l1[4];
                        limbs4(w[u][0], l0), limbs4(w[u][1], l1);
#pragma unroll
                        for (int m = 0; m < 4; m++)
                            kf[(((it & 7) * NT + (it >> 8)) * 4 + m) * 32 + ((it >> 3) & 31)] = make_uint2(l0[m], l1[m]);
                    }
                }
            }
        }
        const P32 P = make_p32(prm.p[t]);
        const uint2 red = prm.red[t];
        const uint32_t mu = prm.mu[t];
        const int g = lane >> 2, tig = lane & 3;
        int stage = 0;
        for (int b0 = 0; b0 < B; b0 += 16, stage ^= 1)
        {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            __syncthreads(); // this tile has landed; the other stage and the fragments are free
            if (b0 + 16 < B)
                load_tile(b0 + 16, stage ^ 1);
            // transposition: an item (x, b, digit quad Jq) -> limb registers of the A fragment of x.  Lane bits: x & 3, b & 1, b >> 3,
            // Jq >> 2; warp and round bits: x >> 2, (b >> 1) & 3, Jq & 3 (digit reads and fragment writes both conflict-free)
            const uint32_t *src = ds + stage * 4096;
#pragma unroll
            for (int rr = 0; rr < 4; rr++)
            {
                const int r = warp * 4 + rr;
                const int x = (r & 1) * 4 + (lane & 3), b = ((lane >> 3) & 1) * 8 + ((r >> 1) & 3) * 2 + ((lane >> 2) & 1);
                const int Jq = (lane >> 4) * 4 + (r >> 3);
                uint32_t w[4], l[4];
#pragma unroll
                for (int j = 0; j < 4; j++)
                {
                    const int J = 4 * Jq + j;
                    const int q = ((J * 16 + b) * 2 + (x >> 2)) ^ (((b >> 3) & 1) << 2) ^ ((J >> 4) & 1);
                    w[j] = src[q * 4 + (x & 3)];
                }
                limbs4(w, l);
                // A fragment of m16n8k32: register 0 = row g, digits 4i ..; 1 = row g + 8; 2 = row g, digits 16 + 4i ..; 3 = row g + 8
                const int fl = (b & 7) * 4 + (Jq & 3), reg = (b >> 3) + 2 * (Jq >> 2);
#pragma unroll
                for (int m = 0; m < 4; m++)
                    af[x * kMmaAfStride + m * 128 + fl * 4 + reg] = l[m];
            }
            __syncthreads();
            // output tile nt, all 8 coefficients; the A fragment of one limb is read just before its four products
            for (int nt = warp; nt < NT; nt += 8)
            {
                uint32_t res[kMmaX][4];
#pragma unroll
                for (int x = 0; x < kMmaX; x++)
                {
                    uint2 bf[4];
#pragma unroll
                    for (int m = 0; m < 4; m++)
                        bf[m] = kf[((x * NT + nt) * 4 + m) * 32 + lane];
                    uint32_t cs[7][4];
#pragma unroll
                    for (int s = 0; s < 7; s++)
#pragma unroll
                        for (int e = 0; e < 4; e++)
                            cs[s][e] = 0;
#pragma unroll
                    for (int l = 0; l < 4; l++)
                    {
                        const uint4 a = *reinterpret_cast<const uint4 *>(af + x * kMmaAfStride + l * 128 + lane * 4);
#pragma unroll
                        for (int m = 0; m < 4; m++)
                            mma_u8(cs[l + m], a, bf[m]);
                    }
#pragma unroll
                    for (int e = 0; e < 4; e++)
                    {
                        const u64 lo = madw(cs[3][e], 1u << 24, madw(cs[2][e], 1u << 16, madw(cs[1][e], 1u << 8, cs[0][e])));
                        const u64 hi = madw(cs[6][e], 1u << 16, madw(cs[5][e], 1u << 8, cs[4][e]));
                        res[x][e] = minsub(reduce64(lo + (hi << 32), red, mu, P), P.p2);
                    }
                }
                // C fragment: e = 0, 1: row g, outputs 2i, 2i + 1; e = 2, 3: row g + 8.  Lanes i and i ^ 1 swap half of their words so
                // that every store writes whole 32-byte sectors: the first store is row (2 (i & ~1) + e & 1) -- x 0..3 from the even
                // lane, x 4..7 from the odd one -- the second row (2 (i | 1) + e & 1).  (Half-sector stores made the kernel 2.4x slower.)
                const int half = tig & 1;
#pragma unroll
                for (int e = 0; e < 4; e++)
                {
                    uint32_t keep[4], recv[4];
#pragma unroll
                    for (int j = 0; j < 4; j++)
                    {
                        keep[j] = half ? res[4 + j][e] : res[j][e];
                        recv[j] = __shfl_xor_sync(0xffffffffu, half ? res[j][e] : res[4 + j][e], 1);
                    }
                    const int b = b0 + g + 8 * (e >> 1), oA = 8 * nt + 2 * (tig & 2) + (e & 1), oB = oA + 2;
                    const uint4 vA = half ? make_uint4(recv[0], recv[1], recv[2], recv[3]) : make_uint4(keep[0], keep[1], keep[2], keep[3]);
                    const uint4 vB = half ? make_uint4(keep[0], keep[1], keep[2], keep[3]) : make_uint4(recv[0], recv[1], recv[2], recv[3]);
                    if (b < B && oA < NO)
                        *reinterpret_cast<uint4 *>(Acc + ((static_cast<size_t>(b * NO + oA) * prm.S + t) << LOGN) + x0 + 4 * half) = vA;
                    if (b < B && oB < NO)
                        *reinterpret_cast<uint4 *>(Acc + ((static_cast<size_t>(b * NO + oB) * prm.S + t) << LOGN) + x0 + 4 * half) = vB;
                }
            }
        }
    }
    // returns the kernel that ran: 0 register tile, 1 key tile, 2 tensor cores
    template <int LOGN>
    static int launch_mac(const KsIntScratch &s, const uint32_t *key32, const KsInt &d, bool mma, int L, int k, int digits, int B, int nbt, int n,
                          cudaStream_t st)
    {
        // below 16 ciphertexts the key tile every CTA stages outweighs the products: the integer kernels take those chunks (H100,
        // n = 65536, 31 digits, ms per multiply + relinearize call with / without the tensor cores: 3.1 / 1.6 at B = 1, 8.1 / 8.2 at
        // B = 15, 8.4 / 9.0 at B = 16)
        if (mma && L <= kMmaMaxDigits && B >= 16)
        {
            const size_t smem = mac_mma_smem((2 * (L + 1) + 7) / 8);
            cuda_check(cudaFuncSetAttribute(ks32_mac_mma<LOGN>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)), "smem attr");
            const dim3 grid(static_cast<unsigned>(n / kMmaX), static_cast<unsigned>(d.prm.S));
            ks32_mac_mma<LOGN><<<grid, 256, smem, st>>>(s.Dh, key32, s.Acc, d.prm, L, k, digits, B, nbt * kMacTB);
            return 2;
        }
        const int ntile = (L + kMacTC) / kMacTC, ny = (2 * ntile + 3) / 4;
        const size_t tile_smem = static_cast<size_t>(L) * 4096 + kMacRingBytes;
        // the tile kernel walks over all ciphertexts with one CTA per (coefficient tile, output group): worth it from a few tiles on
        if (d.mac_tile && tile_smem <= 227 * 1024 && B >= 16)
        {
            cuda_check(cudaFuncSetAttribute(ks32_mac_tile<LOGN>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(tile_smem)), "smem attr");
            dim3 grid(static_cast<unsigned>(ny) * static_cast<unsigned>(n / 32), 1, static_cast<unsigned>(d.prm.S));
            ks32_mac_tile<LOGN><<<grid, 512, tile_smem, st>>>(s.Dh, key32, s.Acc, d.prm, L, k, digits, B, nbt * kMacTB);
            return 1;
        }
        cuda_check(cudaFuncSetAttribute(ks32_mac<LOGN>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMacSmem), "smem attr");
        dim3 grid(static_cast<unsigned>(nbt) * static_cast<unsigned>(ny) * static_cast<unsigned>(n / 32), 1, static_cast<unsigned>(d.prm.S));
        ks32_mac<LOGN><<<grid, 128, kMacSmem, st>>>(s.Dh, key32, s.Acc, d.prm, L, k, digits, B, nbt);
        return 0;
    }
    static int launch_mac_logn(const KsIntScratch &s, const uint32_t *key32, const KsInt &d, bool mma, int L, int k, int digits, int B, int nbt,
                               int logn, cudaStream_t st)
    {
        const int n = 1 << logn;
        switch (logn)
        {
        case 12: return launch_mac<12>(s, key32, d, mma, L, k, digits, B, nbt, n, st);
        case 13: return launch_mac<13>(s, key32, d, mma, L, k, digits, B, nbt, n, st);
        case 14: return launch_mac<14>(s, key32, d, mma, L, k, digits, B, nbt, n, st);
        case 15: return launch_mac<15>(s, key32, d, mma, L, k, digits, B, nbt, n, st);
        case 16: return launch_mac<16>(s, key32, d, mma, L, k, digits, B, nbt, n, st);
        case 17: return launch_mac<17>(s, key32, d, mma, L, k, digits, B, nbt, n, st);
        default: throw std::logic_error("unsupported transform size");
        }
    }

    // -------------------------------------------------------------- (4) reconstruction + mod-down, per coefficient ----
    template <class Base = BaseSrc>
    struct CrtArgs
    {
        uint32_t *Acc;           // ks32_crt_kernel<..., TOP = true> leaves U in place of the special prime's first two residue rows
        const u64 *punct, *neg; // [k][S]
        const PrimeDev *primes;
        const Tw *inv_top;       // q_sp^-1 mod q_i
        const u64 *half_mod;     // floor(q_sp / 2) mod q_i
        const Tw *qtop_mod;      // BGV: q_sp mod q_i
        u64 t = 0, t_ratio = 0;  // BGV plain modulus
        Tw inv_top_mod_t = { 0, 0 };
        u64 *R;                  // MODE 0 / 3: [B][2][L][n]
        u64 *out;                // MODE 1: out + b*o_bs + c*o_ps + i*n
        long long o_bs, o_ps;
        Base base;               // MODE 1 only
        int L, k;
        long long total;         // B * 2 * n
    };
    // Per output prime and coefficient: y_t = x_t c1_t + c2_t mod p_t (canonical), three 64-bit sums sum y_t C_t.lo, sum y_t C_t.hi,
    // sum y_t floor(2^60 / p_t) (the last one's top bits are alpha: the true fraction lies in (1/4, 3/4), the estimate is 2^-28 below
    // it), one barrett_wide of sum y_t (P/p_t) + (-(alpha P) - H) mod q, then the mod-down (evaluator.cpp:2762-2864) with lazy operands:
    // (a_i - ((u mod q_i) - half)) q_sp^-1 is formed from a_i + (2 q_i + half mod q_i) - u without reducing u when q_sp < 2 q_i.
    // The instruction count per reconstruction (it is what bounds this step: ncu, issue slots 75 % busy in the first version) is
    // ~2.5x lower than with a 96-bit carry chain, a 128-bit Barrett step and canonical intermediates.
    // x in [0, 2p) -> y_t: (x n^-1 + H) (P/p_t)^-1 mod p_t, canonical: the three sums then stay inside 64 bits (S 2^29 2^32 < 2^64)
    __device__ __forceinline__ uint32_t crt_y(uint32_t x, uint2 c1, uint32_t c2, const P32 &P)
    {
        return minsub(minsub(x * c1.x + c2 + __umulhi(x, c1.y) * P.np, P.p2), P.p);
    }
    __device__ __forceinline__ void crt_acc(uint32_t y, u64 C, uint32_t ip, u64 &a0, u64 &a1, u64 &f)
    {
        asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(a0) : "r"(y), "r"(static_cast<uint32_t>(C)));
        asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(a1) : "r"(y), "r"(static_cast<uint32_t>(C >> 32)));
        asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(f) : "r"(y), "r"(ip));
    }
    // the three sums -> the exact integer mod Q, < S 2^29 q + q;  neg = A.neg + ki * S
    __device__ __forceinline__ u64 crt_finish(u64 a0, u64 a1, u64 f, const u64 *neg, const PrimeDev &Q)
    {
        const u64 ng = __ldg(neg + static_cast<int>(f >> 60));
        u64 lo = a0 + (a1 << 32), hi = (a1 >> 32) + (lo < a0);
        lo += ng;
        hi += (lo < ng);
        return barrett_wide(lo, hi, Q);
    }
    // the special prime's value: CKKS shifts it by half (evaluator.cpp:2809-2817); BGV keeps it and derives k = -u q_top^-1 mod t
    // (evaluator.cpp:2770-2779, rns.cpp:1202-1213)
    template <int MODE>
    __device__ __forceinline__ u64 crt_top(u64 U, const PrimeDev &T)
    {
        return MODE == 3 ? U : csub(U + (T.q >> 1), T.q);
    }
    template <class Args>
    __device__ __forceinline__ u64 crt_top_k(u64 U, const Args &A)
    {
        const u64 r = barrett64(U, A.t, A.t_ratio);
        return mul_shoup(r ? A.t - r : 0, A.inv_top_mod_t, A.t);
    }
    // residue a of output prime i, U = crt_top<MODE>(special prime's value), K = crt_top_k(U) (BGV) -> the mod-down result, canonical
    template <int MODE, class Args>
    __device__ __forceinline__ u64 crt_moddown(u64 a, u64 U, u64 K, int i, const PrimeDev &Q, const PrimeDev &T, const Args &A)
    {
        u64 x; // a_i - delta_i + (multiple of q_i), in (0, 4 q_i)
        const u64 u = T.q < Q.q2 ? U : barrett64(U, Q.q, Q.ratio_hi); // u < q_top < 2 q_i: no reduction of u needed
        if (MODE == 3)
        {
            const u64 kk = (A.t > Q.q) ? barrett64(K, Q.q, Q.ratio_hi) : K;
            x = a + (Q.q2 + Q.q) - u - mul_shoup(kk, A.qtop_mod[i], Q.q); // rns.cpp:1216-1235
        }
        else
            x = a + (Q.q2 + __ldg(A.half_mod + i)) - u; // evaluator.cpp:2819-2864
        return mul_shoup(x, A.inv_top[i], Q.q);
    }
    // One kernel, two shapes.  FUSE = false: a thread reconstructs one coefficient of one (ciphertext, component) for every output
    // prime.  FUSE = true: a thread owns the 2^(LOGN-12) coefficients j + 4096 e and first runs the outer inverse stages on them (they
    // are exactly the words those butterflies couple), so the outer pass of the inverse transforms never goes through memory.
    // TOP (with FUSE): only the special prime's value, crt_top<MODE>(U), stored as two 32-bit halves over the words of the special
    // prime's residue rows t = 0, 1 that the same thread has just read; ks32_inv_crt_ntt does the rest.
    // MODE 0: CKKS (coefficient-form result to R), 1: BFV (result + base to out), 3: BGV (R)
    template <int MODE, int LOGN, bool FUSE, bool TOP = false, class Base = BaseSrc>
    __global__ void __launch_bounds__(FUSE ? 128 : 256) ks32_crt_kernel(CrtArgs<Base> A, KsIntParams prm, const uint2 *__restrict__ tw_outer)
    {
        constexpr int R = LOGN - 12, E = FUSE ? (1 << R) : 1;
        const int S = prm.S, L = A.L, k = A.k;
        int bc, j;
        if (FUSE)
            bc = blockIdx.x >> 5, j = ((blockIdx.x & 31) << 7) + threadIdx.x;
        else
        {
            const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
            if (e >= A.total)
                return;
            bc = static_cast<int>(e >> LOGN), j = static_cast<int>(e & ((1 << LOGN) - 1));
        }
        const int b = bc >> 1, c = bc & 1;
        const uint32_t *src = A.Acc + ((static_cast<size_t>(bc) * (L + 1) * S) << LOGN) + j; // output prime I' = 0; += S << LOGN per prime
        // the residues of the NEXT output prime are requested before the arithmetic of the current one (ncu of the first version: the
        // first multiply after each load held the stall samples); the fused shape has 2^R words per residue and loads them in place
        constexpr int PF = FUSE ? 1 : kKsMaxS;
        uint32_t nxt[PF];
        auto prefetch = [&]() {
            if (!FUSE)
            {
#pragma unroll
                for (int t = 0; t < kKsMaxS; t++)
                    if (t < S)
                        nxt[t] = src[static_cast<size_t>(t) << LOGN];
            }
        };
        prefetch();
        // fused shape: the rows (output prime, auxiliary prime) are consecutive in memory; the 2^R words of the NEXT row are requested
        // before the butterflies of the current one (two warps per scheduler cannot hide a DRAM round trip per row otherwise)
        uint32_t nrow[FUSE ? E : 1];
        int rows_left = FUSE ? (TOP ? S : (L + 1) * S) : 0;
        auto fetch_row = [&]() {
            if (FUSE)
            {
                if (rows_left > 0)
                {
#pragma unroll
                    for (int e = 0; e < E; e++)
                        nrow[e] = src[e << 12];
                }
                src += size_t(1) << LOGN;
                rows_left--;
            }
        };
        fetch_row();
        auto reconstruct = [&](int ki, const PrimeDev &Q, u64(&val)[E], bool more) {
            u64 a0[E], a1[E], f[E];
#pragma unroll
            for (int e = 0; e < E; e++)
                a0[e] = a1[e] = f[e] = 0;
            const u64 *punct = A.punct + ki * S;
            uint32_t cur[PF];
            if (!FUSE)
            {
#pragma unroll
                for (int t = 0; t < kKsMaxS; t++)
                    cur[t] = nxt[t];
                src += static_cast<size_t>(S) << LOGN;
                if (more)
                    prefetch();
            }
            // fully unrolled with an early exit: the per-prime constants become constant-bank operands of the instructions
#pragma unroll
            for (int t = 0; t < kKsMaxS; t++)
            {
                if (t >= S)
                    break;
                const P32 P = make_p32(prm.p[t]);
                uint32_t a[E];
                if (FUSE)
                {
#pragma unroll
                    for (int e = 0; e < E; e++)
                        a[e] = nrow[e];
                    fetch_row();
                    const uint2 *tw = tw_outer + (t << R);
                    radix_inv<R>(a, [&](int lvl, int g) { return __ldg(tw + (1 << lvl) + g); }, P);
                }
                else
                    a[0] = cur[t];
                const uint2 c1 = prm.c1[t];
                const uint32_t c2 = prm.c2[t], ip = prm.inv60[t];
                const u64 C = __ldg(punct + t);
#pragma unroll
                for (int e = 0; e < E; e++)
                    crt_acc(crt_y(a[e], c1, c2, P), C, ip, a0[e], a1[e], f[e]);
            }
#pragma unroll
            for (int e = 0; e < E; e++)
                val[e] = crt_finish(a0[e], a1[e], f[e], A.neg + ki * S, Q);
        };
        const PrimeDev T = A.primes[k - 1];
        u64 U[E], K[MODE == 3 ? E : 1];
        reconstruct(k - 1, T, U, L > 0);
#pragma unroll
        for (int e = 0; e < E; e++)
            U[e] = crt_top<MODE>(U[e], T);
        if (TOP)
        {
            uint32_t *o = A.Acc + ((static_cast<size_t>(bc) * (L + 1) * S) << LOGN) + j;
#pragma unroll
            for (int e = 0; e < E; e++)
            {
                o[e << 12] = static_cast<uint32_t>(U[e]);
                o[(size_t(1) << LOGN) + (e << 12)] = static_cast<uint32_t>(U[e] >> 32);
            }
            return;
        }
        if (MODE == 3)
        {
#pragma unroll
            for (int e = 0; e < E; e++)
                K[e] = crt_top_k(U[e], A);
        }
        for (int i = 0; i < L; i++)
        {
            const PrimeDev Q = A.primes[i];
            u64 a[E];
            reconstruct(i, Q, a, i + 1 < L);
#pragma unroll
            for (int e = 0; e < E; e++)
            {
                const u64 r = crt_moddown<MODE>(a[e], U[e], K[MODE == 3 ? e : 0], i, Q, T, A);
                const int xi = j + (e << 12);
                if (MODE == 1)
                    A.out[b * A.o_bs + c * A.o_ps + (static_cast<long long>(i) << LOGN) + xi] =
                        finish(A.base, b, c, i, LOGN, xi, csub(r + A.base.get(b, c, i, xi, Q.q), Q.q), Q);
                else
                    A.R[((static_cast<size_t>(bc) * L + i) << LOGN) + xi] = r;
            }
        }
    }
    template <int MODE, int LOGN, class Base>
    static void launch_crt_logn(const CrtArgs<Base> &A, const KsInt &d, bool fuse, size_t B, cudaStream_t st)
    {
        if (fuse)
            ks32_crt_kernel<MODE, LOGN, true, false, Base><<<static_cast<unsigned>(B * 2 * 32), 128, 0, st>>>(A, d.prm, d.d_inv_outer.get());
        else
            ks32_crt_kernel<MODE, LOGN, false, false, Base><<<static_cast<unsigned>((A.total + 255) / 256), 256, 0, st>>>(A, d.prm, d.d_inv_outer.get());
    }
    template <int MODE, class Base>
    static void launch_crt(const CrtArgs<Base> &A, const KsInt &d, bool fuse, size_t B, int logn, cudaStream_t st)
    {
        switch (logn)
        {
        case 12: launch_crt_logn<MODE, 12>(A, d, false, B, st); break; // no outer stages at n = 4096
        case 13: launch_crt_logn<MODE, 13>(A, d, fuse, B, st); break;
        case 14: launch_crt_logn<MODE, 14>(A, d, fuse, B, st); break;
        case 15: launch_crt_logn<MODE, 15>(A, d, fuse, B, st); break;
        case 16: launch_crt_logn<MODE, 16>(A, d, fuse, B, st); break;
        case 17: launch_crt_logn<MODE, 17>(A, d, false, B, st); break; // 32 coefficients per thread do not fit the register file
        default: throw std::logic_error("unsupported transform size");
        }
    }

    // ---------------------------------- (4 + 5a) reconstruction and mod-down as the load of the result's forward column pass ----
    // One CTA = the column pass of result row (b, c, i) over the coefficients r 256 + col0 + c (r < NA, c < C); with n = 4096 2^R the
    // groups j + 4096 e (e < 2^R) that the outer inverse stages couple are among them.  (1) every (group, auxiliary prime t) pair runs
    // the outer stages on the accumulated products of output prime i and leaves y_t in shared memory; (2) every thread reconstructs its
    // 8 coefficients from their S values y_t and mods them down with U (ks32_crt_kernel<..., TOP = true>); (3) the column stages of the
    // 64-bit forward transform, whose tile reuses the shared memory of (1).  The coefficient-form result never goes through memory.
    // 2 CTAs per SM (64 registers): the launch bound of the plain column pass (SB_COL_MIN_BLOCKS) leaves too few for (2).
    template <int LOGNA>
    constexpr size_t crt_ntt_smem(int S) { return static_cast<size_t>(S > 2 ? S : 2) * kTile * 4 + (size_t(1) << LOGNA) * sizeof(Tw) + 8; }
    template <int MODE, int LOGNA, bool FAST>
    __global__ void __launch_bounds__(kColThreads, 2) ks32_inv_crt_ntt(CrtArgs<> A, KsIntParams prm, const uint2 *__restrict__ tw_outer, u64 *__restrict__ mid)
    {
        constexpr int NA = 1 << LOGNA, C = kTile / NA, R = LOGNA - 4, E = 1 << R, G = kTile / E, LOGN = LOGNA + kLocalLog;
        extern __shared__ __align__(16) unsigned char ks_crt_smem[];
        const int S = prm.S, L = A.L;
        uint32_t *ys = reinterpret_cast<uint32_t *>(ks_crt_smem); // [t][r C + c]
        u64 *tile = reinterpret_cast<u64 *>(ks_crt_smem);
        Tw *tw_s = reinterpret_cast<Tw *>(ks_crt_smem + static_cast<size_t>(S > 2 ? S : 2) * kTile * 4);
        u64 *bar = reinterpret_cast<u64 *>(tw_s + NA);
        const int row = blockIdx.x, col0 = blockIdx.y * C, tid = threadIdx.x, c = tid % C, ridx = tid / C;
        const int bc = row / L, i = row - bc * L;
        const PrimeDev Q = A.primes[i];
        if (tid == 0)
            mbar_init(bar, 1);
        __syncthreads();
        if (tid == 0)
        {
            mbar_expect_tx(bar, NA * sizeof(Tw));
            tma_load_1d(tw_s, Q.fwd, NA * sizeof(Tw), bar);
        }
        // (1) rows (bc, I' = i + 1, t) of the accumulated products
        const uint32_t *acc = A.Acc + ((static_cast<size_t>(bc) * (L + 1) + i + 1) * S << LOGN) + col0;
#pragma unroll 1
        for (int w = tid; w < G * S; w += kColThreads)
        {
            const int t = w / G, grp = w - t * G, rl = grp / C, cc = grp - rl * C;
            const P32 P = make_p32(prm.p[t]);
            const uint32_t *p = acc + (static_cast<size_t>(t) << LOGN) + (rl << kLocalLog) + cc;
            uint32_t x[E];
#pragma unroll
            for (int e = 0; e < E; e++)
                x[e] = p[e << 12];
            const uint2 *tw = tw_outer + (t << R);
            radix_inv<R>(x, [&](int lvl, int g) { return __ldg(tw + (1 << lvl) + g); }, P);
            const uint2 c1 = prm.c1[t];
            const uint32_t c2 = prm.c2[t];
#pragma unroll
            for (int e = 0; e < E; e++)
                ys[t * kTile + (rl + 16 * e) * C + cc] = crt_y(x[e], c1, c2, P);
        }
        __syncthreads();
        // (2) coefficients r = ridx + j NA/8: the first layout of the column stages
        const uint32_t *ulo = A.Acc + ((static_cast<size_t>(bc) * (L + 1) * S) << LOGN) + col0 + c, *uhi = ulo + (size_t(1) << LOGN);
        const PrimeDev T = A.primes[A.k - 1];
        const u64 *punct = A.punct + i * S;
        u64 a[8];
#pragma unroll
        for (int j = 0; j < 8; j++)
        {
            const int r = ridx + j * (NA >> 3);
            u64 a0 = 0, a1 = 0, f = 0;
#pragma unroll
            for (int t = 0; t < kKsMaxS; t++)
            {
                if (t >= S)
                    break;
                crt_acc(ys[t * kTile + r * C + c], __ldg(punct + t), prm.inv60[t], a0, a1, f);
            }
            const u64 U = pack64(ulo[r << kLocalLog], uhi[r << kLocalLog]);
            a[j] = crt_moddown<MODE>(crt_finish(a0, a1, f, A.neg + i * S, Q), U, MODE == 3 ? crt_top_k(U, A) : 0, i, Q, T, A);
        }
        __syncthreads(); // the values y_t are consumed: the shared memory becomes the tile
        mbar_wait(bar, 0);
        // (3)
        fwd_col_passes<LOGNA, FAST>(a, tile, tw_s, ridx, c, Q);
        u64 *m = mid + (static_cast<size_t>(row) << LOGN);
#pragma unroll
        for (int j = 0; j < 8; j++)
            m[((8 * ridx + j) << kLocalLog) + col0 + c] = a[j];
    }
    template <int MODE, int LOGNA>
    static void launch_crt_ntt_logna(const CrtArgs<> &A, const KsInt &d, u64 *mid, size_t B, bool fast, bool top, cudaStream_t st)
    {
        if (top)
        {
            ks32_crt_kernel<MODE, LOGNA + kLocalLog, true, true><<<static_cast<unsigned>(B * 2 * 32), 128, 0, st>>>(A, d.prm, d.d_inv_outer.get());
            return;
        }
        auto kern = fast ? ks32_inv_crt_ntt<MODE, LOGNA, true> : ks32_inv_crt_ntt<MODE, LOGNA, false>;
        const size_t smem = crt_ntt_smem<LOGNA>(d.prm.S);
        cuda_check(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)), "smem attr");
        const dim3 grid(static_cast<unsigned>(B * 2 * A.L), static_cast<unsigned>((1 << kLocalLog) / (kTile >> LOGNA)));
        kern<<<grid, kColThreads, smem, st>>>(A, d.prm, d.d_inv_outer.get(), mid);
    }
    // top: the special prime's value (ks32_crt_kernel<..., TOP = true>); otherwise ks32_inv_crt_ntt into mid.  n = 8192 .. 65536
    template <int MODE>
    static void launch_crt_ntt(const CrtArgs<> &A, const KsInt &d, u64 *mid, size_t B, bool fast, bool top, int logn, cudaStream_t st)
    {
        switch (logn)
        {
        case 13: launch_crt_ntt_logna<MODE, 5>(A, d, mid, B, fast, top, st); break;
        case 14: launch_crt_ntt_logna<MODE, 6>(A, d, mid, B, fast, top, st); break;
        case 15: launch_crt_ntt_logna<MODE, 7>(A, d, mid, B, fast, top, st); break;
        case 16: launch_crt_ntt_logna<MODE, 8>(A, d, mid, B, fast, top, st); break;
        default: throw std::logic_error("unsupported transform size");
        }
    }

    // ------------------------------------------------- (5) the result back to NTT form, added into the ciphertext ----
    template <class Base = BaseSrc>
    struct OpAddBaseFwd
    {
        u64 *R;   // [B][2][L][n], transformed in place
        u64 *out; // out + b*o_bs + c*o_ps + i*n
        long long o_bs, o_ps;
        Base base;
        int logn, L;
        __device__ __forceinline__ bool skip(int) const { return false; }
        __device__ __forceinline__ int pid(int row) const { return row % L; }
        __device__ __forceinline__ u64 *rowp(int row) const { return R + (static_cast<long long>(row) << logn); }
        __device__ __forceinline__ const u64 *direct(int row, const PrimeDev &) const { return rowp(row); }
        __device__ __forceinline__ u64 load1(int row, int idx, const PrimeDev &) const { return rowp(row)[idx]; }
        __device__ __forceinline__ void load8(int row, int idx0, u64 (&a)[8], const PrimeDev &) const
        {
#pragma unroll
            for (int j = 0; j < 8; j++)
                a[j] = rowp(row)[idx0 + j];
        }
        __device__ __forceinline__ u64 *mid(int row) const { return rowp(row); }
        __device__ __forceinline__ void store1(int row, int idx, u64 v, const PrimeDev &P) const
        {
            const int i = row % L, bc = row / L, b = bc >> 1, c = bc & 1;
            const u64 t = csub(csub(v, P.q2), P.q);
            out[b * o_bs + c * o_ps + (static_cast<long long>(i) << logn) + idx] =
                finish(base, b, c, i, logn, idx, csub(t + base.get(b, c, i, idx, P.q), P.q), P);
        }
        __device__ __forceinline__ void store8(int row, int idx0, u64 (&a)[8], const PrimeDev &P) const
        {
            const int i = row % L, bc = row / L, b = bc >> 1, c = bc & 1;
            ulonglong2 *op_ = reinterpret_cast<ulonglong2 *>(out + b * o_bs + c * o_ps + (static_cast<long long>(i) << logn) + idx0);
            const bool has_base = base.present && !(c == 1 && base.c1_zero);
            const bool base_plain = has_base && base.s.plain();
            const ulonglong2 *bp = base_plain ? reinterpret_cast<const ulonglong2 *>(base.s.row(b, i) + c * base.pstride + idx0) : nullptr;
#pragma unroll
            for (int h = 0; h < 4; h++)
            {
                u64 r0 = csub(csub(a[2 * h], P.q2), P.q), r1 = csub(csub(a[2 * h + 1], P.q2), P.q);
                if (base_plain)
                {
                    const ulonglong2 bv = bp[h];
                    r0 = csub(r0 + bv.x, P.q), r1 = csub(r1 + bv.y, P.q);
                }
                else if (has_base)
                {
                    r0 = csub(r0 + base.get(b, c, i, idx0 + 2 * h, P.q), P.q);
                    r1 = csub(r1 + base.get(b, c, i, idx0 + 2 * h + 1, P.q), P.q);
                }
                finish2(base, b, c, i, logn, idx0, h, r0, r1, P);
                op_[h] = make_ulonglong2(r0, r1);
            }
        }
    };

    // ------------------------------------------------------------------------------------------------ host side ----
    void ksint_init(Context &c)
    {
        c.ksint.ready = false;
        if (c.logn < 12 || c.k < 2)
            return;
        const sbh::KsIntHost h = sbh::build_ksint(c.n, c.q.data(), c.k);
        if (h.S == 0 || h.S > kKsMaxS)
            return;
        KsInt &d = c.ksint;
        d.prm.S = h.S, d.prm.r = h.r, d.prm.logn = c.logn;
        d.max_digits = h.max_digits; // the 64-bit sums of ks32_mac / ks32_mac_tile: deeper levels take the 64-bit path
        for (int t = 0; t < h.S; t++)
        {
            d.prm.p[t] = h.p[t], d.prm.mu[t] = h.mu[t], d.prm.c2[t] = h.c2[t];
            d.prm.inv60[t] = static_cast<uint32_t>((u64(1) << 60) / h.p[t]);
            d.prm.red[t] = make_uint2(h.red[2 * t], h.red[2 * t + 1]);
            d.prm.c1[t] = make_uint2(h.c1[2 * t], h.c1[2 * t + 1]);
        }
        d.d_fwd_outer = upload<uint2>(c, h.fwd_outer);
        d.d_inv_outer = upload<uint2>(c, h.inv_outer);
        d.d_fwd_local = upload<uint2>(c, h.fwd_local);
        d.d_inv_local = upload<uint2>(c, h.inv_local);
        d.d_punct = upload<u64>(c, h.punct_mod_q);
        d.d_neg = upload<u64>(c, h.neg_mod_q);
        {
            std::vector<u64> hm(c.k);
            for (size_t i = 0; i < c.k; i++)
                hm[i] = (c.q[c.k - 1] >> 1) % c.q[i];
            d.d_half_mod = upload<u64>(c, hm);
        }
        cuda_check(cudaFuncSetAttribute(ks32_fwd_local, cudaFuncAttributeMaxDynamicSharedMemorySize, kKsLocalSmem), "smem attr");
        cuda_check(cudaFuncSetAttribute(ks32_inv_local, cudaFuncAttributeMaxDynamicSharedMemorySize, kKsLocalSmem), "smem attr");
        if (const char *e = std::getenv("SB200_KS_FUSE_CRT"))
            d.fuse_crt = std::atoi(e) != 0;
        if (const char *e = std::getenv("SB200_KS_FUSE_NTT"))
            d.fuse_ntt = std::atoi(e) != 0;
        if (const char *e = std::getenv("SB200_KS_MAC_TILE"))
            d.mac_tile = std::atoi(e) != 0;
        if (const char *e = std::getenv("SB200_KS_MAC_MMA"))
            d.mac_mma = std::atoi(e) != 0;
        d.ready = true;
    }

    // the digit slab holds ceil(B / TB) * TB ciphertexts (register tiles of the product kernel); the per-ciphertext figure counts one
    // ciphertext of padding per real one only through ksint_bytes_fixed (at most TB - 1 rows per digit and prime)
    size_t ksint_bytes_per_ct(const Context &c, size_t L)
    {
        const size_t S = c.ksint.prm.S;
        return c.n * (std::max(S * L * 4, 2 * L * 8) + 2 * (L + 1) * S * 4);
    }
    size_t ksint_bytes_fixed(const Context &c, size_t L) { return c.n * c.ksint.prm.S * L * 4 * (kMacTB - 1); }
    KsIntScratch ksint_carve(const Context &c, size_t L, size_t B, void *base)
    {
        const size_t S = c.ksint.prm.S, Bpad = (B + kMacTB - 1) / kMacTB * kMacTB;
        KsIntScratch s;
        unsigned char *p = static_cast<unsigned char *>(base);
        s.Dh = reinterpret_cast<uint32_t *>(p);
        s.R = reinterpret_cast<u64 *>(p);
        p += c.n * std::max(S * L * 4 * Bpad, 2 * L * 8 * B);
        s.Acc = reinterpret_cast<uint32_t *>(p);
        return s;
    }

    template <bool PLAIN>
    static void launch_fwd_outer(Context &c, Src dsrc, int L, int rows, uint32_t *Dh, RowMap map, cudaStream_t st)
    {
        const KsInt &d = c.ksint;
        const unsigned grid = static_cast<unsigned>(rows) * 16u;
        switch (d.prm.r)
        {
        case 0: ks32_fwd_outer<0, PLAIN><<<grid, 256, 0, st>>>(dsrc, L, c.d_primes.get(), d.prm, d.d_fwd_outer.get(), Dh, map); break;
        case 1: ks32_fwd_outer<1, PLAIN><<<grid, 256, 0, st>>>(dsrc, L, c.d_primes.get(), d.prm, d.d_fwd_outer.get(), Dh, map); break;
        case 2: ks32_fwd_outer<2, PLAIN><<<grid, 256, 0, st>>>(dsrc, L, c.d_primes.get(), d.prm, d.d_fwd_outer.get(), Dh, map); break;
        case 3: ks32_fwd_outer<3, PLAIN><<<grid, 256, 0, st>>>(dsrc, L, c.d_primes.get(), d.prm, d.d_fwd_outer.get(), Dh, map); break;
        case 4: ks32_fwd_outer<4, PLAIN><<<grid, 256, 0, st>>>(dsrc, L, c.d_primes.get(), d.prm, d.d_fwd_outer.get(), Dh, map); break;
        case 5: ks32_fwd_outer<5, PLAIN><<<grid, 256, 0, st>>>(dsrc, L, c.d_primes.get(), d.prm, d.d_fwd_outer.get(), Dh, map); break;
        default: throw std::logic_error("unsupported transform size");
        }
    }

    // rows of 64-bit words (dsrc rows (b, J), J < L) -> Dh[t][map.rows_out][n], transformed modulo every auxiliary prime
    // (outer = false: the outer pass has been run, by ks32_intt_fwd_outer)
    static void ksint_forward(Context &c, Src dsrc, int L, int rows, uint32_t *Dh, RowMap map, cudaStream_t st, bool outer = true)
    {
        const KsInt &d = c.ksint;
        const double n = static_cast<double>(c.n), S = d.prm.S;
        const bool plain = dsrc.perm == nullptr && dsrc.ginv == 0;
        if (outer)
        {
            c.stats.begin("ks32_fwd_outer", 0, rows * n * (8.0 + 4.0 * S), st, 0, 0);
            c.stats.work32(0.5 * rows * n * S * d.prm.r, 0);
            plain ? launch_fwd_outer<true>(c, dsrc, L, rows, Dh, map, st) : launch_fwd_outer<false>(c, dsrc, L, rows, Dh, map, st);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "ks32_fwd_outer");
        }
        // (padding rows of the digit layout are transformed too: a few uninitialised rows whose products are never stored)
        const unsigned grid = static_cast<unsigned>((map.rows_out + kRowsPerCta - 1) / kRowsPerCta * (d.prm.S << d.prm.r));
        c.stats.begin("ks32_fwd_local", 0, rows * n * 8.0 * S, st, 0, 0);
        c.stats.work32(0.5 * rows * n * S * 12, 0);
        ks32_fwd_local<<<grid, 256, kKsLocalSmem, st>>>(Dh, map.rows_out, 1, map.rows_out, d.prm, d.d_fwd_local.get());
        c.stats.end(st);
        cuda_check(cudaGetLastError(), "ks32_fwd_local");
    }

    void ksint_prepare_key(Context &c, KSwitchKey &key, cudaStream_t st)
    {
        if (!c.ksint.ready || key.d_key32)
            return;
        const size_t rows = key.digits * 2 * c.k, words = rows * c.n, S = c.ksint.prm.S;
        // + 8 rows: the last register tile of the product kernel may read (and discard) up to 7 rows past the end
        DevBuf<uint32_t> key32(S * words + 8 * c.n);
        cuda_check(cudaMemsetAsync(key32.get() + S * words, 0, 8 * c.n * sizeof(uint32_t), st), "memset");
        // coefficient form of every key row (row % k = its prime), then the digit path's forward transforms: khat[t][row][n]
        DevBuf<u64> tmp(words);
        struct Quiet // a one-time conversion, not part of any timed operation: no profile records until the scope ends
        {
            LaunchStats &s;
            bool prof;
            ~Quiet() { s.profiling = prof; }
        } quiet{ c.stats, c.stats.profiling };
        c.stats.profiling = false;
        cuda_check(cudaMemcpyAsync(tmp.get(), key.d_key.get(), words * sizeof(u64), cudaMemcpyDeviceToDevice, st), "key copy");
        op_ntt(c, true, c.k, 2, key.digits, tmp.get(), st);
        ksint_forward(c, Src{ tmp.get(), 0, nullptr, 0, c.logn }, static_cast<int>(rows), static_cast<int>(rows), key32.get(),
                      RowMap{ 2, static_cast<int>(c.k), static_cast<int>(rows) }, st);
        cuda_check(cudaStreamSynchronize(st), "synchronize");
        key.d_key32 = std::move(key32);
    }

    template <int R>
    static void launch_inv_outer_r(uint32_t *data, unsigned grid, const KsInt &d, cudaStream_t st)
    {
        ks32_inv_outer<R><<<grid, 256, 0, st>>>(data, d.prm, d.d_inv_outer.get());
    }

    static void launch_inverse(Context &c, uint32_t *data, int arows, cudaStream_t st, bool outer = true);

    template <int LOGNA>
    static void launch_intt_fwd_outer_logna(Context &c, const OpKsIntt &op, int rows, uint32_t *Dh, RowMap map, cudaStream_t st)
    {
        const dim3 grid(static_cast<unsigned>(rows), static_cast<unsigned>((1 << kLocalLog) / (kTile >> LOGNA)));
        ks32_intt_fwd_outer<LOGNA><<<grid, kColThreads, 0, st>>>(op, c.d_primes.get(), c.ksint.prm, c.ksint.d_fwd_outer.get(), Dh, map);
    }
    // the target's inverse transforms (CKKS / BGV: NTT form); fused: their column passes end in the forward outer pass
    static void ksint_target_intt(Context &c, const OpKsIntt &op, int rows, uint32_t *Dh, RowMap map, bool fused, cudaStream_t st)
    {
        cuda_check(launch_ntt_inv(op, rows, c.logn, c.d_primes.get(), st, c.stats, "ks_target_intt", -1, fused), "ks intt");
        if (!fused)
            return;
        const double n = static_cast<double>(c.n), S = c.ksint.prm.S;
        // bytes and butterflies: the inverse column pass's read, ks32_fwd_outer's writes and 32-bit butterflies
        c.stats.begin("ks_target_intt_aux", 1, rows * n * (8.0 + 4.0 * S), st, 0.5 * rows * n * (c.logn - kLocalLog));
        c.stats.work32(0.5 * rows * n * S * c.ksint.prm.r, 0);
        switch (c.logn)
        {
        case 13: launch_intt_fwd_outer_logna<5>(c, op, rows, Dh, map, st); break;
        case 14: launch_intt_fwd_outer_logna<6>(c, op, rows, Dh, map, st); break;
        case 15: launch_intt_fwd_outer_logna<7>(c, op, rows, Dh, map, st); break;
        case 16: launch_intt_fwd_outer_logna<8>(c, op, rows, Dh, map, st); break;
        default: throw std::logic_error("unsupported transform size");
        }
        c.stats.end(st);
        cuda_check(cudaGetLastError(), "ks32_intt_fwd_outer");
    }

    template <class Base>
    void ksint_core(Context &c, size_t L, size_t B, const KsIntScratch &s, Src target, u64 *D, const KSwitchKey &key, Base base,
                    u64 *out, long long o_bs, cudaStream_t st)
    {
        const KsInt &d = c.ksint;
        if (!d.ready || !key.d_key32)
            throw std::logic_error("integer key-switching path is not initialised");
        const int Li = static_cast<int>(L), ki = static_cast<int>(c.k), Bi = static_cast<int>(B), S = d.prm.S;
        const double n = static_cast<double>(c.n);
        const int rows = Bi * Li, nic = 2 * (Li + 1), arows = Bi * nic;
        const bool fuse_crt = d.fuse_crt && d.prm.r >= 1 && d.prm.r <= 4;
        // CKKS / BGV at n = 8192 .. 65536: the path's entry and exit ride in the column passes of the 64-bit transforms
        const bool fuse_ntt = d.fuse_ntt && c.scheme != 1 && d.prm.r >= 1 && d.prm.r <= 4;
        // (1) digits -> auxiliary primes, forward transforms
        const int nbt = (Bi + kMacTB - 1) / kMacTB, Bpad = nbt * kMacTB;
        const RowMap map{ 1, Bpad, Li * Bpad };
        Src dsrc = target;
        if (c.scheme != 1)
        {
            ksint_target_intt(c, OpKsIntt{ target, D, c.logn, Li }, rows, s.Dh, map, fuse_ntt, st);
            dsrc = Src{ D, static_cast<long long>(L * c.n), nullptr, 0, c.logn };
        }
        ksint_forward(c, dsrc, Li, rows, s.Dh, map, st, !fuse_ntt);
        // (2) products with the key, summed over the digits
        {
            // one pass over the key + the transformed digits in, the sums out
            c.stats.begin("ks32_mac", 0, 4.0 * n * S * (static_cast<double>(Li) * 2 * (Li + 1) + rows + arows), st);
            // integer-pipe multiply-accumulates only: the tensor-core kernel's products are not work against the mac32 ceiling (DESIGN 4)
            if (launch_mac_logn(s, key.d_key32.get(), d, d.mac_mma, Li, ki, static_cast<int>(key.digits), Bi, nbt, static_cast<int>(c.logn), st) != 2)
                c.stats.work32(0, static_cast<double>(arows) * Li * S * n);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "ks32_mac");
        }
        // (3) inverse transforms of the sums; the outer stages ride in the reconstruction kernel (fuse_crt) or run as their own pass
        launch_inverse(c, s.Acc, arows, st, !fuse_crt);
        // (4) exact integers -> residues mod q_I, mod-down by the special prime in coefficient form
        const long long o_ps = static_cast<long long>(L) * c.n;
        if (!o_bs)
            o_bs = 2 * o_ps;
        {
            CrtArgs<> A{}; // the base enters only in MODE 1 (BFV), through Ab below
            A.Acc = s.Acc, A.punct = d.d_punct.get(), A.neg = d.d_neg.get(), A.primes = c.d_primes.get();
            A.inv_top = c.d_invq.get() + (c.k - 1) * c.k;
            A.half_mod = d.d_half_mod.get();
            A.R = s.R, A.out = out, A.o_bs = o_bs, A.o_ps = o_ps, A.base = base, A.L = Li, A.k = ki;
            A.total = static_cast<long long>(B) * 2 * c.n;
            if (c.scheme == 3)
            {
                A.qtop_mod = c.d_qmod.get() + (c.k - 1) * c.k;
                A.t = c.t, A.t_ratio = c.t_ratio;
                A.inv_top_mod_t = Tw{ c.inv_q_mod_t[c.k - 1], sbh::shoup(c.inv_q_mod_t[c.k - 1], c.t) };
            }
            if (fuse_ntt && fuse_crt)
            {
                // (4 + 5) the special prime's value in place, then the result's forward column passes reconstruct their own inputs
                c.stats.begin("ks32_inv_crt_top", 0, n * B * 2 * (4.0 * S + 8.0), st);
                c.stats.work32(0.5 * B * 2 * S * n * d.prm.r, 0);
                c.scheme == 3 ? launch_crt_ntt<3>(A, d, s.R, B, c.fast_q, true, c.logn, st) : launch_crt_ntt<0>(A, d, s.R, B, c.fast_q, true, c.logn, st);
                c.stats.end(st);
                cuda_check(cudaGetLastError(), "ks32_crt_kernel");
                const double rrows = 2.0 * B * L;
                c.stats.begin("ks32_inv_crt_ntt", 0, n * rrows * (4.0 * S + 16.0), st, 0.5 * rrows * n * (c.logn - kLocalLog));
                c.stats.work32(0.5 * rrows * S * n * d.prm.r, 0);
                c.scheme == 3 ? launch_crt_ntt<3>(A, d, s.R, B, c.fast_q, false, c.logn, st) : launch_crt_ntt<0>(A, d, s.R, B, c.fast_q, false, c.logn, st);
                c.stats.end(st);
                cuda_check(cudaGetLastError(), "ks32_inv_crt_ntt");
                OpAddBaseFwd<Base> op{ s.R, out, o_bs, o_ps, base, c.logn, Li };
                cuda_check(launch_ntt_fwd(op, static_cast<int>(B * 2 * L), c.logn, c.d_primes.get(), st, c.stats, "ks_result_ntt", -1, c.fast_q, true),
                           "ks result ntt");
                return;
            }
            c.stats.begin("ks32_crt", 0, n * B * 2 * (4.0 * S * (L + 1) + 8.0 * L), st);
            if (fuse_crt)
                c.stats.work32(0.5 * arows * S * n * d.prm.r, 0);
            if (c.scheme == 3)
                launch_crt<3>(A, d, fuse_crt, B, c.logn, st);
            else if (c.scheme == 1)
            {
                if constexpr (Base::kPlain) // BFV: a plaintext product of a coefficient-form result is a convolution
                    throw std::logic_error("the key switch's plaintext product needs an NTT-form result (CKKS / BGV)");
                else
                {
                    CrtArgs<Base> Ab{ A.Acc, A.punct, A.neg, A.primes, A.inv_top, A.half_mod, A.qtop_mod, A.t, A.t_ratio, A.inv_top_mod_t,
                                      A.R, A.out, A.o_bs, A.o_ps, base, A.L, A.k, A.total };
                    launch_crt<1>(Ab, d, fuse_crt, B, c.logn, st);
                }
            }
            else
                launch_crt<0>(A, d, fuse_crt, B, c.logn, st);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "ks32_crt_kernel");
        }
        // (5) CKKS / BGV: back to NTT form, added into the ciphertext
        if (c.scheme != 1)
        {
            OpAddBaseFwd<Base> op{ s.R, out, o_bs, o_ps, base, c.logn, Li };
            cuda_check(launch_ntt_fwd(op, static_cast<int>(B * 2 * L), c.logn, c.d_primes.get(), st, c.stats, "ks_result_ntt", -1, c.fast_q), "ks result ntt");
        }
    }
    template void ksint_core<BaseSrc>(Context &, size_t, size_t, const KsIntScratch &, Src, u64 *, const KSwitchKey &, BaseSrc, u64 *, long long,
                                      cudaStream_t);
    template void ksint_core<BaseAddSrc>(Context &, size_t, size_t, const KsIntScratch &, Src, u64 *, const KSwitchKey &, BaseAddSrc, u64 *,
                                         long long, cudaStream_t);
    template void ksint_core<BasePlainSrc<false>>(Context &, size_t, size_t, const KsIntScratch &, Src, u64 *, const KSwitchKey &,
                                                  BasePlainSrc<false>, u64 *, long long, cudaStream_t);
    template void ksint_core<BasePlainSrc<true>>(Context &, size_t, size_t, const KsIntScratch &, Src, u64 *, const KSwitchKey &,
                                                 BasePlainSrc<true>, u64 *, long long, cudaStream_t);

    static void launch_inverse(Context &c, uint32_t *data, int arows, cudaStream_t st, bool outer)
    {
        const KsInt &d = c.ksint;
        const int S = d.prm.S;
        const double n = static_cast<double>(c.n);
        const unsigned grid = static_cast<unsigned>((arows + kRowsPerCta - 1) / kRowsPerCta * (S << d.prm.r));
        c.stats.begin("ks32_inv_local", 0, 8.0 * arows * S * n, st);
        c.stats.work32(0.5 * arows * S * n * 12, 0);
        ks32_inv_local<<<grid, 256, kKsLocalSmem, st>>>(data, arows, S, 1, d.prm, d.d_inv_local.get());
        c.stats.end(st);
        cuda_check(cudaGetLastError(), "ks32_inv_local");
        if (d.prm.r > 0 && outer)
        {
            const unsigned g1 = static_cast<unsigned>(arows) * S * 16u;
            c.stats.begin("ks32_inv_outer", 0, 8.0 * arows * S * n, st);
            c.stats.work32(0.5 * arows * S * n * d.prm.r, 0);
            switch (d.prm.r)
            {
            case 1: launch_inv_outer_r<1>(data, g1, d, st); break;
            case 2: launch_inv_outer_r<2>(data, g1, d, st); break;
            case 3: launch_inv_outer_r<3>(data, g1, d, st); break;
            case 4: launch_inv_outer_r<4>(data, g1, d, st); break;
            case 5: launch_inv_outer_r<5>(data, g1, d, st); break;
            default: throw std::logic_error("unsupported transform size");
            }
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "ks32_inv_outer");
        }
    }

    void ksint_selftest_transform(Context &c, bool inverse, const u64 *h_rows, size_t rows, uint32_t *h_io)
    {
        if (!c.ksint.ready)
            throw std::logic_error("integer key-switching path is not available for this context");
        const size_t S = c.ksint.prm.S, out_bytes = S * rows * c.n * sizeof(uint32_t), in_bytes = rows * c.n * sizeof(u64);
        unsigned char *base = static_cast<unsigned char *>(c.ensure_scratch(out_bytes + in_bytes));
        uint32_t *d32 = reinterpret_cast<uint32_t *>(base);
        if (inverse)
        {
            cuda_check(cudaMemcpy(d32, h_io, out_bytes, cudaMemcpyHostToDevice), "upload");
            launch_inverse(c, d32, static_cast<int>(rows), nullptr);
        }
        else
        {
            u64 *d64 = reinterpret_cast<u64 *>(base + out_bytes);
            cuda_check(cudaMemcpy(d64, h_rows, in_bytes, cudaMemcpyHostToDevice), "upload");
            ksint_forward(c, Src{ d64, 0, nullptr, 0, c.logn }, static_cast<int>(rows), static_cast<int>(rows), d32,
                          RowMap{ 0, 0, static_cast<int>(rows) }, nullptr);
        }
        cuda_check(cudaMemcpy(h_io, d32, out_bytes, cudaMemcpyDeviceToHost), "download");
    }

    int ksint_selftest_product(Context &c, const uint32_t *h_Dh, const uint32_t *h_key, int L, int B, uint32_t *h_Acc, int mma)
    {
        if (!c.ksint.ready)
            throw std::logic_error("integer key-switching path is not available for this context");
        if (L < 1 || B < 1 || static_cast<size_t>(L) > c.ksint.max_digits)
            throw std::invalid_argument("product: 1 <= L <= max_digits and B >= 1");
        const KsInt &d = c.ksint;
        const size_t S = d.prm.S, n = c.n, Bpad = (B + kMacTB - 1) / kMacTB * kMacTB, k = L + 1;
        const size_t dh_words = S * L * Bpad * n, key_words = S * L * 2 * k * n, acc_words = B * 2 * k * S * n;
        // + 8 key rows of slack, as ksint_prepare_key allocates them
        uint32_t *base = static_cast<uint32_t *>(c.ensure_scratch((dh_words + key_words + 8 * n + acc_words) * sizeof(uint32_t)));
        KsIntScratch s;
        s.Dh = base;
        uint32_t *key = base + dh_words;
        s.Acc = key + key_words + 8 * n;
        cuda_check(cudaMemset(s.Dh, 0, dh_words * sizeof(uint32_t)), "memset");
        cuda_check(cudaMemcpy2D(s.Dh, Bpad * n * sizeof(uint32_t), h_Dh, B * n * sizeof(uint32_t), B * n * sizeof(uint32_t), S * L,
                                cudaMemcpyHostToDevice), "upload");
        cuda_check(cudaMemcpy(key, h_key, key_words * sizeof(uint32_t), cudaMemcpyHostToDevice), "upload");
        cuda_check(cudaMemset(key + key_words, 0, 8 * n * sizeof(uint32_t)), "memset");
        const int ran = launch_mac_logn(s, key, d, mma != 0, L, static_cast<int>(k), L, B, static_cast<int>(Bpad / kMacTB), static_cast<int>(c.logn), nullptr);
        cuda_check(cudaGetLastError(), "ks32_mac");
        cuda_check(cudaMemcpy(h_Acc, s.Acc, acc_words * sizeof(uint32_t), cudaMemcpyDeviceToHost), "download");
        return ran;
    }

    // ---- arithmetic ceilings of this path, measured in process: the butterflies / multiply-accumulates on registers only ----
    template <int KIND>
    __global__ void __launch_bounds__(256, 4) ks32_selftest_bfly(uint32_t *d, uint32_t p, int rounds)
    {
        __shared__ uint2 ts[256];
        const P32 P = make_p32(p);
        {
            const uint32_t w = (threadIdx.x * 2654435761u + 12345u) % p;
            ts[threadIdx.x] = make_uint2(w, static_cast<uint32_t>((static_cast<u64>(w) << 32) / p));
        }
        __syncthreads();
        uint32_t a[16];
#pragma unroll
        for (int j = 0; j < 16; j++)
            a[j] = d[(static_cast<size_t>(blockIdx.x) * 16 + j) * 256 + threadIdx.x] % p;
        const int lane = threadIdx.x & 31;
        for (int r = 0; r < rounds; r++)
        {
            const uint2 *t = ts + ((r * 7 + lane) & 127); // per-lane twiddles from shared memory, as the local passes read them
            auto tw = [&](int lvl, int g) { return t[(1 << lvl) - 1 + g]; };
            if (KIND == 0)
                radix_fwd<4>(a, tw, P);
            else
                radix_inv<4>(a, tw, P);
        }
#pragma unroll
        for (int j = 0; j < 16; j++)
            d[(static_cast<size_t>(blockIdx.x) * 16 + j) * 256 + threadIdx.x] = a[j];
    }
    // PAIRED: two products per accumulator and round, as the product kernel consumes its digits (ptxas adds both with one three-input
    // 64-bit add); THREADS x MINB: the launch shape (128 x 4: the register-tile kernel's; 512 x 1: the key-tile kernel's)
    template <int THREADS, int MINB, bool PAIRED>
    __global__ void __launch_bounds__(THREADS, MINB) ks32_selftest_mac(uint32_t *d, int rounds)
    {
        uint32_t dv[4], kv[8];
        u64 acc[4][8];
#pragma unroll
        for (int i = 0; i < 4; i++)
            dv[i] = d[(static_cast<size_t>(blockIdx.x) * 12 + i) * THREADS + threadIdx.x] >> 3;
#pragma unroll
        for (int r = 0; r < 8; r++)
            kv[r] = d[(static_cast<size_t>(blockIdx.x) * 12 + 4 + r) * THREADS + threadIdx.x] >> 3;
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
            for (int r = 0; r < 8; r++)
                acc[i][r] = 0;
        for (int q = 0; q < rounds; q++)
        {
            uint32_t d0[4], k0[8], d1[4], k1[8]; // operands change every round
#pragma unroll
            for (int i = 0; i < 4; i++)
                d0[i] = dv[i] + q, d1[i] = dv[i] ^ q;
#pragma unroll
            for (int r = 0; r < 8; r++)
                k0[r] = kv[r] ^ q, k1[r] = kv[r] + q;
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int r = 0; r < 8; r++)
                {
                    asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[i][r]) : "r"(d0[i]), "r"(k0[r]));
                    if (PAIRED)
                        asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[i][r]) : "r"(d1[i]), "r"(k1[r]));
                }
        }
        u64 x = 0;
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
            for (int r = 0; r < 8; r++)
                x ^= acc[i][r];
        d[static_cast<size_t>(blockIdx.x) * 12 * THREADS + threadIdx.x] = static_cast<uint32_t>(x) ^ static_cast<uint32_t>(x >> 32);
    }
    double ksint_selftest_rate(Context &c, int kind, cudaStream_t st)
    {
        if (!c.ksint.ready)
            throw std::logic_error("integer key-switching path is not available for this context");
        int sms = 0;
        cuda_check(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c.device), "device attribute");
        const int rounds = 512;
        const size_t words = static_cast<size_t>(sms) * 4 * 16 * 256;
        uint32_t *d = static_cast<uint32_t *>(c.ensure_scratch(words * sizeof(uint32_t)));
        cuda_check(cudaMemsetAsync(d, 0x5a, words * sizeof(uint32_t), st), "memset");
        cudaEvent_t e0 = c.stats.get_event(), e1 = c.stats.get_event();
        double ops = 0;
        auto run = [&](auto launch) {
            launch();
            cuda_check(cudaEventRecord(e0, st), "record");
            launch();
            cuda_check(cudaEventRecord(e1, st), "record");
            cuda_check(cudaEventSynchronize(e1), "synchronize");
            cuda_check(cudaGetLastError(), "selftest kernel");
        };
        switch (kind)
        {
        case 0: // forward butterflies at the local passes' launch shape (256 threads x 4 CTAs per SM): 32 per thread and round
            ops = static_cast<double>(sms) * 4 * 8 * rounds * 32.0;
            run([&] { ks32_selftest_bfly<0><<<sms * 4, 256, 0, st>>>(d, c.ksint.prm.p[0], rounds); });
            break;
        case 1:
            ops = static_cast<double>(sms) * 4 * 8 * rounds * 32.0;
            run([&] { ks32_selftest_bfly<1><<<sms * 4, 256, 0, st>>>(d, c.ksint.prm.p[0], rounds); });
            break;
        case 2: // multiply-accumulates, one product per accumulator and round, 128 threads x 4 CTAs per SM: 32 per thread and round
            ops = static_cast<double>(sms) * 4 * 4 * rounds * 32.0;
            run([&] { ks32_selftest_mac<128, 4, false><<<sms * 4, 128, 0, st>>>(d, rounds); });
            break;
        case 3: // the same at the key-tile kernel's launch shape (512 threads x 1 CTA per SM)
            ops = static_cast<double>(sms) * 16 * rounds * 32.0;
            run([&] { ks32_selftest_mac<512, 1, false><<<sms, 512, 0, st>>>(d, rounds); });
            break;
        case 4: // two products per accumulator and round (the product kernel's form), 128 x 4
            ops = static_cast<double>(sms) * 4 * 4 * rounds * 64.0;
            run([&] { ks32_selftest_mac<128, 4, true><<<sms * 4, 128, 0, st>>>(d, rounds); });
            break;
        case 5: // two products per accumulator and round, 512 x 1
            ops = static_cast<double>(sms) * 16 * rounds * 64.0;
            run([&] { ks32_selftest_mac<512, 1, true><<<sms, 512, 0, st>>>(d, rounds); });
            break;
        default: throw std::invalid_argument("unknown selftest");
        }
        float ms = 0;
        cuda_check(cudaEventElapsedTime(&ms, e0, e1), "cudaEventElapsedTime");
        c.stats.pool.push_back(e0);
        c.stats.pool.push_back(e1);
        return ops / (ms * 1e-3);
    }
} // namespace sb
