// seal_b200/csrc/sb_bfv.cu -- BFV ciphertext multiplication (BEHZ RNS variant) on the device.
//
// Reproduces Evaluator::bfv_multiply (evaluator.cpp:395-567) and the RNSTool steps it calls (util/rns.cpp):
//   (1) fastbconv_m_tilde  rns.cpp:1086-1131     \  behz_lift_kernel: one thread per coefficient, the L residues
//   (2) sm_mrq             rns.cpp:979-1039      /  staged in shared memory, FastBConv as 128-bit dot products
//   (3) NTT over q and Bsk                          batched transforms (sb_ntt.cuh)
//   (4) dyadic tensor      evaluator.cpp:497-541    tensor_kernel (both bases in one launch)
//   (5) INTT, (6) times t  evaluator.cpp:545-556    fused: the store of the inverse transform multiplies by t
//   (7) fast_floor         rns.cpp:1041-1084     \  behz_floor_sk_kernel: one thread per coefficient
//   (8) fastbconv_sk       rns.cpp:903-977       /
// FastBConv is the reference's inexact conversion sum_i [x_i (q/q_i)^-1]_{q_i} (q/q_i) mod p  (rns.cpp:418-463): the
// sum is a residue mod p, so accumulation order is free and results are word-identical.
#include "sb_engine.cuh"
#include <algorithm>

namespace sb
{
    struct BehzDev
    {
        sbh::BehzLevel host;
        int L = 0, nB = 0, nS = 0;
        // device arrays
        DevBuf<int> pids_bsk;          // prime ids of Bsk                         [nS]
        DevBuf<Tw> lift_c;             // m_tilde * (q/q_i)^-1 mod q_i             [L]
        DevBuf<Tw> inv_punc_q;         //                                          [L]
        DevBuf<u64> q_to_bsk;          //                                          [nS][L]
        DevBuf<uint32_t> q_to_mt;      // (q/q_i) mod 2^32                         [L]
        DevBuf<Tw> prod_q_mod_bsk, inv_mt_mod_bsk, inv_q_mod_bsk, t_mod_bsk; // [nS]
        DevBuf<Tw> t_mod_q, prod_b_mod_q, neg_prod_b_mod_q;                  // [L]
        DevBuf<Tw> inv_punc_b;         //                                          [nB]
        DevBuf<u64> b_to_q;            //                                          [L][nB]
        DevBuf<u64> b_to_msk;          //                                          [nB]
        Tw inv_b_mod_msk{};
        uint32_t neg_inv_q_mod_mt = 0;
    };

    static BehzDev &behz_dev(Context &c, size_t L)
    {
        if (c.scheme != 1)
            throw std::logic_error("BEHZ base exists for BFV contexts only");
        if (L < 1 || L > c.k)
            throw std::invalid_argument("encrypted is not valid for encryption parameters");
        check_bfv_multiply_level(c, L);
        auto it = c.behz.find(L);
        if (it != c.behz.end())
            return *it->second;
        auto d = std::make_shared<BehzDev>();
        d->host = sbh::build_behz(c.n, c.q, L, c.t);
        const sbh::BehzLevel &h = d->host;
        d->L = static_cast<int>(L), d->nB = static_cast<int>(h.nB), d->nS = static_cast<int>(h.nBsk);
        // Bsk primes are prefixes of the context-wide auxiliary list [m_sk, gamma, B_0, ...]
        std::vector<int> pids;
        for (size_t i = 0; i < h.nB; i++)
        {
            if (2 + i >= c.aux.size() || c.aux[2 + i] != h.B[i])
                throw std::logic_error("auxiliary base mismatch");
            pids.push_back(static_cast<int>(c.k + 2 + i));
        }
        pids.push_back(static_cast<int>(c.k + 0));
        d->pids_bsk = upload<int>(c, pids);
        std::vector<sbh::TwPair> lift;
        std::vector<uint32_t> qmt;
        for (size_t i = 0; i < L; i++)
        {
            u64 v = sbh::mulmod(h.mtilde_mod_q[i].w, h.inv_punc_q[i].w, c.q[i]);
            lift.push_back(sbh::TwPair{ v, sbh::shoup(v, c.q[i]) });
            qmt.push_back(static_cast<uint32_t>(h.q_to_mtilde[i]));
        }
        d->lift_c = upload<Tw>(c, lift);
        d->inv_punc_q = upload<Tw>(c, h.inv_punc_q);
        d->q_to_bsk = upload<u64>(c, h.q_to_Bsk);
        d->q_to_mt = upload<uint32_t>(c, qmt);
        d->prod_q_mod_bsk = upload<Tw>(c, h.prod_q_mod_Bsk);
        d->inv_mt_mod_bsk = upload<Tw>(c, h.inv_mtilde_mod_Bsk);
        d->inv_q_mod_bsk = upload<Tw>(c, h.inv_q_mod_Bsk);
        d->t_mod_bsk = upload<Tw>(c, h.t_mod_Bsk);
        d->t_mod_q = upload<Tw>(c, h.t_mod_q);
        d->prod_b_mod_q = upload<Tw>(c, h.prod_B_mod_q);
        d->neg_prod_b_mod_q = upload<Tw>(c, h.neg_prod_B_mod_q);
        d->inv_punc_b = upload<Tw>(c, h.inv_punc_B);
        d->b_to_q = upload<u64>(c, h.B_to_q);
        d->b_to_msk = upload<u64>(c, h.B_to_msk);
        d->inv_b_mod_msk.w = h.inv_B_mod_msk.w, d->inv_b_mod_msk.wq = h.inv_B_mod_msk.wq;
        d->neg_inv_q_mod_mt = static_cast<uint32_t>(h.neg_inv_q_mod_mtilde);
        c.behz[L] = d;
        return *d;
    }

    const sbh::BehzLevel &behz_host(Context &c, size_t L)
    {
        return behz_dev(c, L).host;
    }

    // ---- (1)+(2): lift the s1+s2 input polynomials from base q to base Bsk, removing the q-overflow ----------------
    // grid = (n/TH, s1+s2, B); dynamic smem = L*TH words
    constexpr int kBehzThreads = 128;
    __global__ void __launch_bounds__(kBehzThreads) behz_lift_kernel(const u64 *__restrict__ a, const u64 *__restrict__ b, u64 *__restrict__ XS,
                                                                      const PrimeDev *__restrict__ primes, const int *__restrict__ pids_bsk,
                                                                      const Tw *__restrict__ lift_c, const u64 *__restrict__ q_to_bsk,
                                                                      const uint32_t *__restrict__ q_to_mt, const Tw *__restrict__ prod_q_mod_bsk,
                                                                      const Tw *__restrict__ inv_mt_mod_bsk, uint32_t neg_inv_q_mod_mt, int logn,
                                                                      int L, int nS, int s1, int s2)
    {
        extern __shared__ u64 sm[];
        const int n = 1 << logn, idx = blockIdx.x * blockDim.x + threadIdx.x, p4 = blockIdx.y, bb = blockIdx.z;
        if (idx >= n)
            return;
        const u64 *src = (p4 < s1 ? a + ((static_cast<long long>(bb) * s1 + p4) * L << logn)
                                  : b + ((static_cast<long long>(bb) * s2 + (p4 - s1)) * L << logn)) + idx;
        u64 *t = sm + threadIdx.x;
        uint32_t ymt = 0;
        for (int i = 0; i < L; i++)
        {
            const u64 qi = primes[i].q;
            u64 ti = mul_shoup(src[static_cast<long long>(i) << logn], lift_c[i], qi); // [x m~ (q/q_i)^-1]_{q_i}
            t[i * blockDim.x] = ti;
            ymt += static_cast<uint32_t>(ti) * q_to_mt[i]; // FastBConv to {m~ = 2^32}: only the low 32 bits matter
        }
        const uint32_t r = ymt * neg_inv_q_mod_mt; // rns.cpp:1016-1017 (mod 2^32)
        u64 *dst = XS + ((static_cast<long long>(bb) * (s1 + s2) + p4) * nS << logn) + idx;
        for (int s = 0; s < nS; s++)
        {
            const PrimeDev P = primes[pids_bsk[s]];
            u64 lo = 0, hi = 0;
            for (int i = 0; i < L; i++)
                mac128(lo, hi, t[i * blockDim.x], q_to_bsk[s * L + i]);
            u64 y = barrett128(lo, hi, P.q, P.ratio_lo, P.ratio_hi);
            u64 rc = r;
            if (r >= 0x80000000u)
                rc += P.q - 0x100000000ull; // centred representative of r modulo the Bsk prime (rns.cpp:1027-1031)
            u64 v = csub(mul_shoup(rc, prod_q_mod_bsk[s], P.q) + y, P.q);
            dst[static_cast<long long>(s) << logn] = mul_shoup(v, inv_mt_mod_bsk[s], P.q);
        }
    }

    // ---- (4) tensor in an arbitrary base: X = [B][4][nb][n] (polys x0,x1,y0,y1) -> D = [B][3][nb][n] ---------------
    __global__ void __launch_bounds__(256) behz_tensor_kernel(const u64 *__restrict__ X, u64 *__restrict__ D, const PrimeDev *__restrict__ primes,
                                                               const int *__restrict__ pid_tab, int logn, int nb, long long total)
    {
        long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over B*nb*n
        if (e >= total)
            return;
        const long long poly = static_cast<long long>(nb) << logn;
        const long long bidx = e / poly, r = e % poly;
        const int i = static_cast<int>(r >> logn);
        const PrimeDev P = primes[pid_tab ? pid_tab[i] : i];
        const u64 *px = X + bidx * 4 * poly + r;
        u64 x0 = px[0], x1 = px[poly], y0 = px[2 * poly], y1 = px[3 * poly];
        u64 *po = D + bidx * 3 * poly + r;
        po[0] = mulmod_barrett(x0, y0, P);
        u64 lo = 0, hi = 0;
        mac128(lo, hi, x0, y1);
        mac128(lo, hi, x1, y0);
        po[poly] = barrett128(lo, hi, P.q, P.ratio_lo, P.ratio_hi);
        po[2 * poly] = mulmod_barrett(x1, y1, P);
    }

    // ---- (7)+(8): divide by q and floor into Bsk, then Shenoy-Kumaresan back to base q -----------------------------
    // grid = (n/TH, s1+s2-1, B); dynamic smem = (max(L, nS) + nS) * TH words
    __global__ void __launch_bounds__(kBehzThreads) behz_floor_sk_kernel(
        const u64 *__restrict__ DQ, const u64 *__restrict__ DS, u64 *__restrict__ out, const PrimeDev *__restrict__ primes,
        const int *__restrict__ pids_bsk, const Tw *__restrict__ inv_punc_q, const u64 *__restrict__ q_to_bsk, const Tw *__restrict__ inv_q_mod_bsk,
        const Tw *__restrict__ inv_punc_b, const u64 *__restrict__ b_to_q, const u64 *__restrict__ b_to_msk, Tw inv_b_mod_msk,
        const Tw *__restrict__ prod_b_mod_q, const Tw *__restrict__ neg_prod_b_mod_q, int logn, int L, int nB, int nS)
    {
        extern __shared__ u64 sm[];
        const int n = 1 << logn, idx = blockIdx.x * blockDim.x + threadIdx.x, p = blockIdx.y, bb = blockIdx.z;
        if (idx >= n)
            return;
        const int TH = blockDim.x, W = L > nS ? L : nS;
        u64 *t = sm + threadIdx.x;          // [W]  t_i, later u_i
        u64 *f = sm + W * TH + threadIdx.x; // [nS] f_s
        const int nout = gridDim.y;
        const u64 *dq = DQ + ((static_cast<long long>(bb) * nout + p) * L << logn) + idx;
        const u64 *ds = DS + ((static_cast<long long>(bb) * nout + p) * nS << logn) + idx;
        for (int i = 0; i < L; i++)
            t[i * TH] = mul_shoup(dq[static_cast<long long>(i) << logn], inv_punc_q[i], primes[i].q);
        // fast_floor: f_s = (d_s - FastBConv_{q->s}(d)) q^-1 mod Bsk_s   (rns.cpp:1074-1083)
        for (int s = 0; s < nS; s++)
        {
            const PrimeDev P = primes[pids_bsk[s]];
            u64 lo = 0, hi = 0;
            for (int i = 0; i < L; i++)
                mac128(lo, hi, t[i * TH], q_to_bsk[s * L + i]);
            u64 conv = barrett128(lo, hi, P.q, P.ratio_lo, P.ratio_hi);
            f[s * TH] = mul_shoup(ds[static_cast<long long>(s) << logn] + P.q - conv, inv_q_mod_bsk[s], P.q);
        }
        // fastbconv_sk (rns.cpp:932-976)
        for (int i = 0; i < nB; i++)
            t[i * TH] = mul_shoup(f[i * TH], inv_punc_b[i], primes[pids_bsk[i]].q);
        const PrimeDev M = primes[pids_bsk[nB]]; // m_sk
        u64 alpha;
        {
            u64 lo = 0, hi = 0;
            for (int i = 0; i < nB; i++)
                mac128(lo, hi, t[i * TH], b_to_msk[i]);
            u64 conv = barrett128(lo, hi, M.q, M.ratio_lo, M.ratio_hi);
            alpha = mul_shoup(conv + M.q - f[nB * TH], inv_b_mod_msk, M.q);
        }
        const bool neg = alpha > (M.q >> 1); // rns.cpp:964
        u64 *o = out + ((static_cast<long long>(bb) * nout + p) * L << logn) + idx;
        for (int j = 0; j < L; j++)
        {
            const PrimeDev P = primes[j];
            u64 lo = 0, hi = 0;
            for (int i = 0; i < nB; i++)
                mac128(lo, hi, t[i * TH], b_to_q[j * nB + i]);
            u64 y = barrett128(lo, hi, P.q, P.ratio_lo, P.ratio_hi);
            u64 corr = neg ? mul_shoup(M.q - alpha, prod_b_mod_q[j], P.q) : mul_shoup(alpha, neg_prod_b_mod_q[j], P.q);
            o[static_cast<long long>(j) << logn] = csub(y + corr, P.q);
        }
    }

    // ---- NTT functors ------------------------------------------------------------------------------------------------
    // forward transform of the s1+s2 input polys in base q: rows (b, p4, i) -> XQ[b][p4][i]
    struct OpBfvFwdQ
    {
        const u64 *a, *b;
        u64 *XQ;
        int logn, L, s1, s2;
        __device__ __forceinline__ bool skip(int) const { return false; }
        __device__ __forceinline__ int pid(int row) const { return row % L; }
        __device__ __forceinline__ const u64 *direct(int row, const PrimeDev &) const
        {
            const int i = row % L, bp = row / L, p4 = bp % (s1 + s2), bb = bp / (s1 + s2);
            return p4 < s1 ? a + (((static_cast<long long>(bb) * s1 + p4) * L + i) << logn)
                           : b + (((static_cast<long long>(bb) * s2 + (p4 - s1)) * L + i) << logn);
        }
        __device__ __forceinline__ u64 load1(int row, int idx, const PrimeDev &P) const { return direct(row, P)[idx]; }
        __device__ __forceinline__ void load8(int, int, u64 (&)[8], const PrimeDev &) const {}
        __device__ __forceinline__ u64 *mid(int row) const { return XQ + (static_cast<long long>(row) << logn); }
        __device__ __forceinline__ void store1(int row, int idx, u64 v, const PrimeDev &P) const { mid(row)[idx] = csub(csub(v, P.q2), P.q); }
        __device__ __forceinline__ void store8(int row, int idx0, u64 (&v)[8], const PrimeDev &P) const
        {
            ulonglong2 *p = reinterpret_cast<ulonglong2 *>(mid(row) + idx0);
#pragma unroll
            for (int j = 0; j < 4; j++)
                p[j] = make_ulonglong2(csub(csub(v[2 * j], P.q2), P.q), csub(csub(v[2 * j + 1], P.q2), P.q));
        }
    };

    // in-place inverse transform whose store multiplies by t (steps 5+6)
    struct OpBfvInvMulT
    {
        u64 *data;
        const Tw *t_mod; // per base element
        const int *pid_tab;
        int logn, nb;
        __device__ __forceinline__ bool skip(int) const { return false; }
        __device__ __forceinline__ int pid(int row) const
        {
            int i = row % nb;
            return pid_tab ? pid_tab[i] : i;
        }
        __device__ __forceinline__ u64 *rowp(int row) const { return data + (static_cast<long long>(row) << logn); }
        __device__ __forceinline__ const u64 *direct(int row, const PrimeDev &) const { return rowp(row); }
        __device__ __forceinline__ u64 load1(int row, int idx, const PrimeDev &) const { return rowp(row)[idx]; }
        __device__ __forceinline__ void load8(int row, int idx0, u64 (&a)[8], const PrimeDev &) const
        {
            const ulonglong2 *p = reinterpret_cast<const ulonglong2 *>(rowp(row) + idx0);
#pragma unroll
            for (int j = 0; j < 4; j++)
            {
                ulonglong2 v = p[j];
                a[2 * j] = v.x, a[2 * j + 1] = v.y;
            }
        }
        __device__ __forceinline__ u64 *mid(int row) const { return rowp(row); }
        __device__ __forceinline__ void store1(int row, int idx, u64 v, const PrimeDev &P) const
        {
            rowp(row)[idx] = mul_shoup(v, t_mod[row % nb], P.q);
        }
        __device__ __forceinline__ void store8(int row, int idx0, u64 (&a)[8], const PrimeDev &P) const
        {
#pragma unroll
            for (int j = 0; j < 8; j++)
                store1(row, idx0 + j, a[j], P);
        }
    };

    void op_ntt_rows(Context &c, bool inverse, u64 *d, size_t rows, size_t L, const int *pid_tab, cudaStream_t st);

    // Every term of the three FastBConv dot products (q -> Bsk in the lift and in fast_floor, B -> q and B -> m_sk in
    // fastbconv_sk) is below 2^122, so with at most 64 terms no 128-bit sum can wrap whatever the constants are.  The same limit
    // keeps the shared memory of behz_floor_sk_kernel, (max(L, |Bsk|) + |Bsk|) * 128 words, below what a block may use.
    void check_bfv_multiply_level(const Context &c, size_t L)
    {
        if (c.scheme == 1 && L >= 1 && L <= c.k && sbh::behz_base_size(c.q, L, c.t) > kBfvMultiplyMaxBase)
            throw std::invalid_argument("BFV multiplication supports at most 64 primes per level (and in its auxiliary base B)");
    }

    void op_bfv_multiply(Context &c, size_t L, size_t batch, const u64 *a, const u64 *b, u64 *out3, cudaStream_t st)
    {
        op_bfv_multiply(c, L, 2, 2, batch, a, b, out3, st);
    }

    // evaluator.cpp:395-567 for ciphertext sizes s1 x s2 -> s1+s2-1 (the BEHZ steps run per polynomial, :453-522, :524-560)
    void op_bfv_multiply(Context &c, size_t L, size_t s1, size_t s2, size_t batch, const u64 *a, const u64 *b, u64 *out3, cudaStream_t st)
    {
        check_sizes(s1, s2);
        check_bfv_multiply_level(c, L);
        BehzDev &d = behz_dev(c, L);
        const int n = static_cast<int>(c.n), Li = d.L, nS = d.nS, nB = d.nB;
        const size_t nin = s1 + s2, nout = s1 + s2 - 1;
        // scratch per ciphertext: XQ nin*L, XS nin*nS, DQ nout*L, DS nout*nS rows
        const size_t rows_per_ct = (nin + nout) * (L + nS);
        const size_t per = rows_per_ct * c.n * sizeof(u64);
        size_t chunk = std::min(batch, std::max<size_t>(1, c.scratch_budget / per));
        chunk = std::min<size_t>(chunk, std::max<size_t>(1, (size_t(1) << 30) / (nin * (L + nS) * c.n)));
        chunk = std::min<size_t>(chunk, 65535);
        const int TH = std::min(n, kBehzThreads);
        const size_t smem_lift = static_cast<size_t>(Li) * TH * sizeof(u64);
        const size_t smem_floor = static_cast<size_t>(std::max(Li, nS) + nS) * TH * sizeof(u64);
        cuda_check(cudaFuncSetAttribute(behz_lift_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_lift)), "smem attr");
        cuda_check(cudaFuncSetAttribute(behz_floor_sk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_floor)),
                   "smem attr");
        for (size_t b0 = 0; b0 < batch; b0 += chunk)
        {
            const size_t B = std::min(chunk, batch - b0);
            u64 *XQ = static_cast<u64 *>(c.ensure_scratch(per * B));
            u64 *XS = XQ + B * nin * L * c.n, *DQ = XS + B * nin * nS * c.n, *DS = DQ + B * nout * L * c.n;
            const u64 *pa = a + b0 * s1 * L * c.n, *pb = b + b0 * s2 * L * c.n;
            {
                OpBfvFwdQ op{ pa, pb, XQ, c.logn, Li, static_cast<int>(s1), static_cast<int>(s2) };
                cuda_check(launch_ntt_fwd(op, static_cast<int>(B * nin * L), c.logn, c.d_primes.get(), st, c.stats, "bfv_ntt_q", -1, c.fast_q), "bfv ntt q");
            }
            {
                dim3 grid((n + TH - 1) / TH, static_cast<unsigned>(nin), static_cast<unsigned>(B));
                c.stats.begin("behz_lift", 0, 8.0 * n * B * nin * (L + nS), st);
                behz_lift_kernel<<<grid, TH, smem_lift, st>>>(pa, pb, XS, c.d_primes.get(), d.pids_bsk.get(), d.lift_c.get(), d.q_to_bsk.get(), d.q_to_mt.get(), d.prod_q_mod_bsk.get(),
                                                              d.inv_mt_mod_bsk.get(), d.neg_inv_q_mod_mt, c.logn, Li, nS, static_cast<int>(s1),
                                                              static_cast<int>(s2));
                c.stats.end(st);
                cuda_check(cudaGetLastError(), "behz_lift_kernel");
            }
            op_ntt_rows(c, false, XS, B * nin * nS, nS, d.pids_bsk.get(), st);
            if (s1 != 2 || s2 != 2)
            {
                launch_tensor_general(c, XQ, static_cast<long long>(nin * L) * n, XQ + s1 * L * c.n, static_cast<long long>(nin * L) * n, DQ,
                                      nullptr, L, s1, s2, B, st);
                launch_tensor_general(c, XS, static_cast<long long>(nin) * nS * n, XS + s1 * nS * c.n, static_cast<long long>(nin) * nS * n, DS,
                                      d.pids_bsk.get(), nS, s1, s2, B, st);
            }
            else
            {
                long long tq = static_cast<long long>(B) * L * n, ts = static_cast<long long>(B) * nS * n;
                c.stats.begin("behz_tensor", 0, 56.0 * tq, st);
                behz_tensor_kernel<<<static_cast<unsigned>((tq + 255) / 256), 256, 0, st>>>(XQ, DQ, c.d_primes.get(), nullptr, c.logn, Li, tq);
                c.stats.end(st);
                c.stats.begin("behz_tensor", 0, 56.0 * ts, st);
                behz_tensor_kernel<<<static_cast<unsigned>((ts + 255) / 256), 256, 0, st>>>(XS, DS, c.d_primes.get(), d.pids_bsk.get(), c.logn, nS, ts);
                c.stats.end(st);
                cuda_check(cudaGetLastError(), "behz_tensor_kernel");
            }
            {
                OpBfvInvMulT oq{ DQ, d.t_mod_q.get(), nullptr, c.logn, Li };
                cuda_check(launch_ntt_inv(oq, static_cast<int>(B * nout * L), c.logn, c.d_primes.get(), st, c.stats, "bfv_intt_q"), "bfv intt q");
                OpBfvInvMulT os{ DS, d.t_mod_bsk.get(), d.pids_bsk.get(), c.logn, nS };
                cuda_check(launch_ntt_inv(os, static_cast<int>(B * nout * nS), c.logn, c.d_primes.get(), st, c.stats, "bfv_intt_bsk"), "bfv intt bsk");
            }
            {
                dim3 grid((n + TH - 1) / TH, static_cast<unsigned>(nout), static_cast<unsigned>(B));
                c.stats.begin("behz_floor_sk", 0, 8.0 * n * B * nout * (2 * L + nS), st);
                behz_floor_sk_kernel<<<grid, TH, smem_floor, st>>>(DQ, DS, out3 + b0 * nout * L * c.n, c.d_primes.get(), d.pids_bsk.get(), d.inv_punc_q.get(), d.q_to_bsk.get(),
                                                                  d.inv_q_mod_bsk.get(), d.inv_punc_b.get(), d.b_to_q.get(), d.b_to_msk.get(), d.inv_b_mod_msk,
                                                                  d.prod_b_mod_q.get(), d.neg_prod_b_mod_q.get(), c.logn, Li, nB, nS);
                c.stats.end(st);
                cuda_check(cudaGetLastError(), "behz_floor_sk_kernel");
            }
        }
    }
} // namespace sb
