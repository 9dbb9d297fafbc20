// seal_b200/csrc/sb_plainsum.cu -- sums of products in one pass over NTT-form operands:
//   plaintext products: destination j = add_many over i of multiply_plain(ct_i, plain_{j K + i}) (a plaintext matrix times a
//     vector of ciphertexts);
//   ciphertext products: destination j = add_many over i of multiply(lhs_{j K + i}, rhs_i), size-2 operands (the lazy-
//     relinearization idiom: inner products, encrypted-matrix x encrypted-vector by diagonals).
//
// Reference behaviour being reproduced (paths under /root/reference/native/src/seal/):
//   evaluator.cpp:1975-2195 multiply_plain (the four NTT-form cases) -> operands brought to NTT form, then plain_sum_kernel
//   evaluator.cpp:569-841   ckks_multiply / bgv_multiply (size 2 x 2)  -> multiply_sum_kernel
//   evaluator.cpp:395-567   bfv_multiply (BEHZ)                        -> op_bfv_multiply into scratch, chunks of terms, then fold
//   evaluator.cpp:155-262   add_inplace / add_many (BGV balancing)   -> one constant per term, applied with a Shoup product
#include "sb_engine.cuh"
#include <algorithm>

namespace sb
{
    namespace
    {
        struct SumTerm // one ciphertext operand [B][size][L][n], in pairs of words
        {
            const ulonglong2 *ct;
            long long size;
        };
        struct SumPlain // one NTT-form plaintext operand [count][L][n], in pairs; member_stride = 0 when shared by the batch
        {
            const ulonglong2 *p;
            long long member_stride;
        };

        // One thread owns one pair of coefficients (16-byte accesses) of one member for MT outputs and two polynomials
        // (grid: x = pairs of coefficients, y = member, z = output tile x polynomial pair).  For every term the ciphertext pair of
        // each polynomial is loaded once and each of the tile's plaintext pairs once; the products go into 128-bit accumulators,
        // which are reduced once every `window` terms: the largest count with q - 1 + window (q - 1)^2 < 2^128 at the level's largest
        // prime, at most kPlainSumWindow (256, which every prime below 2^60 allows; 64 at 61 bits; DESIGN 3.4).
        template <int MT>
        __global__ void __launch_bounds__(128) plain_sum_kernel(const SumTerm *__restrict__ terms, const SumPlain *__restrict__ plains,
                                                                const Tw *__restrict__ consts, ulonglong2 *const *__restrict__ outs,
                                                                const PrimeDev *__restrict__ primes, int logn, int L, int K, int M, int out_size,
                                                                int groups, int window, int accumulate, long long b0, long long half)
        {
            const long long r = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
            if (r >= half)
                return;
            const long long b = b0 + blockIdx.y;
            const int tile = static_cast<int>(blockIdx.z) / groups, p0 = 2 * (static_cast<int>(blockIdx.z) % groups), j0 = tile * MT;
            const int mt = min(MT, M - j0), np = min(2, out_size - p0);
            const int i = static_cast<int>((r * 2) >> logn);
            const PrimeDev P = primes[i];
            u64 acc[MT][2][4]; // [output][polynomial][lo0, hi0, lo1, hi1]
#pragma unroll
            for (int j = 0; j < MT; j++)
#pragma unroll
                for (int s = 0; s < 2; s++)
                {
                    ulonglong2 v = make_ulonglong2(0, 0);
                    if (accumulate && j < mt && s < np) // a partial sum of an earlier launch: canonical words
                        v = outs[j0 + j][(b * out_size + p0 + s) * half + r];
                    acc[j][s][0] = v.x, acc[j][s][1] = 0, acc[j][s][2] = v.y, acc[j][s][3] = 0;
                }
            for (int t = 0, since = 0; t < K; t++)
            {
                const SumTerm T = terms[t];
                ulonglong2 x[2];
                bool has[2];
#pragma unroll
                for (int s = 0; s < 2; s++)
                {
                    has[s] = s < np && p0 + s < T.size;
                    x[s] = make_ulonglong2(0, 0);
                    if (has[s])
                    {
                        const ulonglong2 v = T.ct[(b * T.size + p0 + s) * half + r];
                        x[s] = make_ulonglong2(canon_in(v.x, P), canon_in(v.y, P));
                        if (consts)
                        {
                            const Tw w = consts[static_cast<long long>(t) * L + i];
                            x[s] = make_ulonglong2(mul_shoup(x[s].x, w, P.q), mul_shoup(x[s].y, w, P.q));
                        }
                    }
                }
                if (has[0] || has[1])
#pragma unroll
                    for (int j = 0; j < MT; j++)
                        if (j < mt)
                        {
                            const SumPlain R = plains[static_cast<long long>(j0 + j) * K + t];
                            ulonglong2 y = R.p[b * R.member_stride + r];
                            y = make_ulonglong2(canon_in(y.x, P), canon_in(y.y, P));
#pragma unroll
                            for (int s = 0; s < 2; s++)
                                if (has[s])
                                {
                                    mac128(acc[j][s][0], acc[j][s][1], x[s].x, y.x);
                                    mac128(acc[j][s][2], acc[j][s][3], x[s].y, y.y);
                                }
                        }
                if (++since == window)
                {
                    since = 0;
#pragma unroll
                    for (int j = 0; j < MT; j++)
#pragma unroll
                        for (int s = 0; s < 2; s++)
                        {
                            acc[j][s][0] = barrett128(acc[j][s][0], acc[j][s][1], P.q, P.ratio_lo, P.ratio_hi), acc[j][s][1] = 0;
                            acc[j][s][2] = barrett128(acc[j][s][2], acc[j][s][3], P.q, P.ratio_lo, P.ratio_hi), acc[j][s][3] = 0;
                        }
                }
            }
#pragma unroll
            for (int j = 0; j < MT; j++)
#pragma unroll
                for (int s = 0; s < 2; s++)
                    if (j < mt && s < np)
                        outs[j0 + j][(b * out_size + p0 + s) * half + r] =
                            make_ulonglong2(barrett128(acc[j][s][0], acc[j][s][1], P.q, P.ratio_lo, P.ratio_hi),
                                            barrett128(acc[j][s][2], acc[j][s][3], P.q, P.ratio_lo, P.ratio_hi));
        }

        // One thread owns one pair of coefficients (16-byte accesses) of one member for MT outputs (grid: x = pairs of coefficients,
        // y = member, z = output tile).  For every term the right-hand pair of both polynomials is loaded once per tile and each
        // left-hand pair once, both reduced as they load (canon_in); the fold's constant of the term scales the left-hand words.
        // c0 += a0 b0, c1 += a0 b1 + a1 b0, c2 += a1 b1 go into 128-bit accumulators, which are reduced once every `window` terms:
        // the largest count with q - 1 + 2 window (q - 1)^2 < 2^128 at the level's largest prime, at most kMultiplySumWindow
        // (128 below 2^60, 32 at 61 bits; DESIGN 3.4).  Squares (a left operand that is the right one) need nothing special.
        template <int MT>
        __global__ void __launch_bounds__(128) multiply_sum_kernel(const ulonglong2 *const *__restrict__ rhs, const ulonglong2 *const *__restrict__ lhs,
                                                                   const Tw *__restrict__ consts, ulonglong2 *const *__restrict__ outs,
                                                                   const PrimeDev *__restrict__ primes, int logn, int L, int K, int M, int window,
                                                                   long long b0, long long half)
        {
            const long long r = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
            if (r >= half)
                return;
            const long long b = b0 + blockIdx.y;
            const int j0 = static_cast<int>(blockIdx.z) * MT, mt = min(MT, M - j0);
            const int i = static_cast<int>((r * 2) >> logn);
            const PrimeDev P = primes[i];
            u64 acc[MT][3][4]; // [output][polynomial][lo0, hi0, lo1, hi1]
#pragma unroll
            for (int j = 0; j < MT; j++)
#pragma unroll
                for (int s = 0; s < 3; s++)
                    acc[j][s][0] = acc[j][s][1] = acc[j][s][2] = acc[j][s][3] = 0;
            const long long o0 = (b * 2) * half + r, o1 = o0 + half;
            for (int t = 0, since = 0; t < K; t++)
            {
                const ulonglong2 *R = rhs[t];
                ulonglong2 y0 = R[o0], y1 = R[o1];
                y0 = make_ulonglong2(canon_in(y0.x, P), canon_in(y0.y, P)), y1 = make_ulonglong2(canon_in(y1.x, P), canon_in(y1.y, P));
                Tw w{};
                if (consts)
                    w = consts[static_cast<long long>(t) * L + i];
#pragma unroll
                for (int j = 0; j < MT; j++)
                    if (j < mt)
                    {
                        const ulonglong2 *X = lhs[static_cast<long long>(j0 + j) * K + t];
                        ulonglong2 x0 = X[o0], x1 = X[o1];
                        x0 = make_ulonglong2(canon_in(x0.x, P), canon_in(x0.y, P)), x1 = make_ulonglong2(canon_in(x1.x, P), canon_in(x1.y, P));
                        if (consts)
                        {
                            x0 = make_ulonglong2(mul_shoup(x0.x, w, P.q), mul_shoup(x0.y, w, P.q));
                            x1 = make_ulonglong2(mul_shoup(x1.x, w, P.q), mul_shoup(x1.y, w, P.q));
                        }
                        mac128(acc[j][0][0], acc[j][0][1], x0.x, y0.x), mac128(acc[j][0][2], acc[j][0][3], x0.y, y0.y);
                        mac128(acc[j][1][0], acc[j][1][1], x0.x, y1.x), mac128(acc[j][1][2], acc[j][1][3], x0.y, y1.y);
                        mac128(acc[j][1][0], acc[j][1][1], x1.x, y0.x), mac128(acc[j][1][2], acc[j][1][3], x1.y, y0.y);
                        mac128(acc[j][2][0], acc[j][2][1], x1.x, y1.x), mac128(acc[j][2][2], acc[j][2][3], x1.y, y1.y);
                    }
                if (++since == window)
                {
                    since = 0;
#pragma unroll
                    for (int j = 0; j < MT; j++)
#pragma unroll
                        for (int s = 0; s < 3; s++)
                        {
                            acc[j][s][0] = barrett128(acc[j][s][0], acc[j][s][1], P.q, P.ratio_lo, P.ratio_hi), acc[j][s][1] = 0;
                            acc[j][s][2] = barrett128(acc[j][s][2], acc[j][s][3], P.q, P.ratio_lo, P.ratio_hi), acc[j][s][3] = 0;
                        }
                }
            }
#pragma unroll
            for (int j = 0; j < MT; j++)
                if (j < mt)
#pragma unroll
                    for (int s = 0; s < 3; s++)
                        outs[j0 + j][(b * 3 + s) * half + r] = make_ulonglong2(barrett128(acc[j][s][0], acc[j][s][1], P.q, P.ratio_lo, P.ratio_hi),
                                                                               barrett128(acc[j][s][2], acc[j][s][3], P.q, P.ratio_lo, P.ratio_hi));
        }

        size_t align16(size_t bytes) { return (bytes + 15) & ~size_t(15); }

        // add_many's left fold acc = acc e1_t +/- x_t e2_t (the factors of unscaled steps are 1), unrolled: term t enters the sum
        // times +/- e2_t prod_{u > t} e1_u.  The residues are exact, so the constants are formed mod q_i on the host: [K][L], with
        // `any` false when every constant is 1 (the kernels then skip them).
        std::vector<Tw> fold_constants(const Context &c, size_t L, size_t K, const int *modes, const u64 *factors, bool &any)
        {
            std::vector<Tw> cst(K * L);
            any = false;
            for (size_t i = 0; i < L; i++)
            {
                const u64 q = c.q[i];
                u64 tail = 1; // prod_{u > t} e1_u mod q
                for (size_t t = K; t-- > 0;)
                {
                    const int m = t && modes ? modes[t - 1] : 0;
                    u64 v = (m & 2) ? factors[2 * (t - 1) + 1] % q : 1;
                    v = static_cast<u64>(static_cast<unsigned __int128>(v) * tail % q);
                    if ((m & 1) && v)
                        v = q - v;
                    cst[t * L + i] = Tw{ v, sbh::shoup(v, q) };
                    any |= v != 1;
                    if (m & 2)
                        tail = static_cast<u64>(static_cast<unsigned __int128>(tail) * (factors[2 * (t - 1)] % q) % q);
                }
            }
            return cst;
        }

        // the reduction window of a level: a carried residue plus `window` terms of `products` products of words below q each stay
        // below 2^128 at the level's largest prime, at most `cap`
        int sum_window(const Context &c, size_t L, int products, int cap)
        {
            u64 qmax = 0;
            for (size_t i = 0; i < L; i++)
                qmax = std::max(qmax, c.q[i]);
            const unsigned __int128 sq = static_cast<unsigned __int128>(qmax - 1) * (qmax - 1) * static_cast<unsigned>(products);
            return static_cast<int>(std::min<unsigned __int128>(cap, sq ? (~static_cast<unsigned __int128>(0) - (qmax - 1)) / sq : cap));
        }

        // the per-call tables of a sum kernel at the front of the scratch arena, each 16-byte aligned, and `rest` bytes behind them
        std::vector<unsigned char *> sum_tables(Context &c, const std::vector<size_t> &bytes, size_t rest)
        {
            size_t total = 0;
            for (size_t b : bytes)
                total += align16(b);
            auto *p = static_cast<unsigned char *>(c.ensure_scratch(total + rest));
            std::vector<unsigned char *> out;
            for (size_t b : bytes)
                out.push_back(p), p += align16(b);
            out.push_back(p);
            return out;
        }

        template <class T>
        void upload_table(T *d, const T *h, size_t count, cudaStream_t st, const char *what)
        {
            if (count)
                cuda_check(cudaMemcpyAsync(d, h, count * sizeof(T), cudaMemcpyHostToDevice, st), what);
        }
    } // namespace

    void op_multiply_plain_sum(Context &c, size_t L, size_t batch, size_t K, size_t M, const size_t *sizes, const u64 *const *cts,
                               const size_t *plain_counts, const u64 *const *plains, bool ct_ntt, bool plain_ntt, const int *modes,
                               const u64 *factors, u64 *const *outs, cudaStream_t st)
    {
        const size_t ln = L * c.n, half = ln / 2;
        size_t out_size = 0;
        for (size_t t = 0; t < K; t++)
            out_size = std::max(out_size, sizes[t]);
        bool any = false;
        const std::vector<Tw> cst = fold_constants(c, L, K, modes, factors, any);
        // operands not in NTT form are transformed into scratch, a chunk of terms at a time; later chunks add to the partial sums
        auto conv_bytes = [&](size_t t) {
            size_t w = ct_ntt ? 0 : batch * sizes[t] * ln;
            for (size_t j = 0; j < M && !plain_ntt; j++)
                w += plain_counts[j * K + t] * ln;
            return w * sizeof(u64);
        };
        std::vector<std::pair<size_t, size_t>> chunks;
        size_t most = 0, max_k = 0;
        for (size_t t0 = 0; t0 < K;)
        {
            size_t t1 = t0 + 1, bytes = conv_bytes(t0);
            while (t1 < K && bytes + conv_bytes(t1) <= c.scratch_budget)
                bytes += conv_bytes(t1++);
            chunks.emplace_back(t0, t1);
            most = std::max(most, bytes), max_k = std::max(max_k, t1 - t0);
            t0 = t1;
        }
        const std::vector<unsigned char *> tabs =
            sum_tables(c, { max_k * sizeof(SumTerm), M * max_k * sizeof(SumPlain), M * sizeof(u64 *), any ? max_k * L * sizeof(Tw) : 0 }, most);
        auto *d_terms = reinterpret_cast<SumTerm *>(tabs[0]);
        auto *d_plains = reinterpret_cast<SumPlain *>(tabs[1]);
        auto *d_outs = reinterpret_cast<ulonglong2 **>(tabs[2]);
        Tw *d_cst = any ? reinterpret_cast<Tw *>(tabs[3]) : nullptr;
        u64 *conv = reinterpret_cast<u64 *>(tabs[4]);
        std::vector<ulonglong2 *> h_outs(M);
        for (size_t j = 0; j < M; j++)
            h_outs[j] = reinterpret_cast<ulonglong2 *>(outs[j]);
        upload_table(d_outs, h_outs.data(), M, st, "upload output table");

        const int window = sum_window(c, L, 1, kPlainSumWindow);
        const int MT = M >= 3 ? 4 : static_cast<int>(M), groups = static_cast<int>((out_size + 1) / 2);
        const size_t tiles = (M + MT - 1) / MT;
        for (const auto &ch : chunks)
        {
            const size_t t0 = ch.first, k = ch.second - ch.first;
            std::vector<SumTerm> h_terms(k);
            std::vector<SumPlain> h_plains(M * k);
            u64 *w = conv;
            double words = 0;
            for (size_t t = t0; t < t0 + k; t++)
            {
                const u64 *ct = cts[t];
                if (!ct_ntt) // BFV coefficient form: the chain's sb200_ntt_forward, on a copy
                {
                    const size_t n_ct = batch * sizes[t] * ln;
                    cuda_check(cudaMemcpyAsync(w, ct, n_ct * sizeof(u64), cudaMemcpyDeviceToDevice, st), "copy");
                    op_ntt(c, false, L, sizes[t], batch, w, st);
                    ct = w, w += n_ct;
                }
                h_terms[t - t0] = SumTerm{ reinterpret_cast<const ulonglong2 *>(ct), static_cast<long long>(sizes[t]) };
                words += static_cast<double>(tiles * batch * sizes[t]);
                for (size_t j = 0; j < M; j++)
                {
                    const size_t pc = plain_counts[j * K + t];
                    const u64 *p = plains[j * K + t];
                    if (!plain_ntt) // transform_to_ntt_inplace(Plaintext&): lift and transform
                    {
                        op_plain_to_ntt(c, L, pc, p, nullptr, w, st);
                        p = w, w += pc * ln;
                    }
                    h_plains[j * k + (t - t0)] = SumPlain{ reinterpret_cast<const ulonglong2 *>(p), pc == 1 ? 0 : static_cast<long long>(half) };
                    words += static_cast<double>(pc * groups);
                }
            }
            // the plaintext table is indexed [output][term of this chunk]
            upload_table(d_terms, h_terms.data(), k, st, "upload term table");
            upload_table(d_plains, h_plains.data(), M * k, st, "upload plain table");
            if (any)
                upload_table(d_cst, cst.data() + t0 * L, k * L, st, "upload term constants");
            words += static_cast<double>((t0 ? 2 : 1) * M * batch * out_size);
            c.stats.begin("plain_sum", 0, 8.0 * words * static_cast<double>(ln), st);
            for (size_t b0 = 0; b0 < batch; b0 += 65535)
            {
                const dim3 grid(static_cast<unsigned>((half + 127) / 128), static_cast<unsigned>(std::min<size_t>(65535, batch - b0)),
                                static_cast<unsigned>(tiles * groups));
                const int args_k = static_cast<int>(k), args_m = static_cast<int>(M), os = static_cast<int>(out_size), acc = t0 ? 1 : 0;
                const auto hl = static_cast<long long>(half), bb = static_cast<long long>(b0);
                if (MT == 1)
                    plain_sum_kernel<1><<<grid, 128, 0, st>>>(d_terms, d_plains, d_cst, d_outs, c.d_primes.get(), c.logn, static_cast<int>(L), args_k,
                                                              args_m, os, groups, window, acc, bb, hl);
                else if (MT == 2)
                    plain_sum_kernel<2><<<grid, 128, 0, st>>>(d_terms, d_plains, d_cst, d_outs, c.d_primes.get(), c.logn, static_cast<int>(L), args_k,
                                                              args_m, os, groups, window, acc, bb, hl);
                else
                    plain_sum_kernel<4><<<grid, 128, 0, st>>>(d_terms, d_plains, d_cst, d_outs, c.d_primes.get(), c.logn, static_cast<int>(L), args_k,
                                                              args_m, os, groups, window, acc, bb, hl);
                cuda_check(cudaGetLastError(), "plain_sum_kernel");
            }
            c.stats.end(st);
        }
        if (!ct_ntt) // the chain's sb200_ntt_inverse, once per output instead of once per term
            for (size_t j = 0; j < M; j++)
                op_ntt(c, true, L, out_size, batch, outs[j], st);
    }

    void op_multiply_sum(Context &c, size_t L, size_t batch, size_t K, size_t M, const u64 *const *lhs, const u64 *const *rhs, const int *modes,
                         const u64 *factors, u64 *const *outs, cudaStream_t st)
    {
        const size_t ln = L * c.n, half = ln / 2;
        if (c.scheme == SB200_SCHEME_BFV)
        {
            // BEHZ rounds every product, so the sum is not one rounding: the chain's op_bfv_multiply runs into the aux arena, a chunk
            // of terms at a time (as many size-3 products as the scratch budget holds), and op_add_many folds each chunk into the
            // output, whose partial sum is operand 0 of every fold after the first.  The fold's steps keep their place in the whole
            // chain, so its words do not depend on where it is cut.
            const size_t per = batch * 3 * ln;
            const size_t k = std::max<size_t>(1, std::min(K, c.scratch_budget / (per * sizeof(u64))));
            u64 *prod = static_cast<u64 *>(c.ensure_aux(k * per * sizeof(u64)));
            std::vector<int> all(K > 1 ? K - 1 : 1, SB200_FOLD_ADD);
            if (modes)
                std::copy(modes, modes + (K - 1), all.begin());
            for (size_t j = 0; j < M; j++)
                for (size_t t0 = 0; t0 < K; t0 += k)
                {
                    const size_t kk = std::min(k, K - t0);
                    std::vector<const u64 *> ops;
                    if (t0)
                        ops.push_back(outs[j]);
                    for (size_t t = t0; t < t0 + kk; t++)
                    {
                        u64 *p = prod + (t - t0) * per;
                        op_bfv_multiply(c, L, batch, lhs[j * K + t], rhs[t], p, st);
                        ops.push_back(p);
                    }
                    const size_t step0 = t0 ? t0 - 1 : 0; // the fold step of ops[1]
                    const std::vector<size_t> sizes(ops.size(), 3);
                    op_add_many(c, L, batch, ops.size(), sizes.data(), ops.data(), all.data() + step0, factors ? factors + 2 * step0 : nullptr,
                                outs[j], st);
                }
            return;
        }
        bool any = false;
        const std::vector<Tw> cst = fold_constants(c, L, K, modes, factors, any);
        const std::vector<unsigned char *> tabs = sum_tables(c, { K * sizeof(u64 *), M * K * sizeof(u64 *), M * sizeof(u64 *), any ? K * L * sizeof(Tw) : 0 }, 0);
        auto *d_rhs = reinterpret_cast<const ulonglong2 **>(tabs[0]);
        auto *d_lhs = reinterpret_cast<const ulonglong2 **>(tabs[1]);
        auto *d_outs = reinterpret_cast<ulonglong2 **>(tabs[2]);
        Tw *d_cst = any ? reinterpret_cast<Tw *>(tabs[3]) : nullptr;
        std::vector<const ulonglong2 *> h_rhs(K), h_lhs(M * K);
        std::vector<ulonglong2 *> h_outs(M);
        for (size_t t = 0; t < K; t++)
            h_rhs[t] = reinterpret_cast<const ulonglong2 *>(rhs[t]);
        for (size_t x = 0; x < M * K; x++)
            h_lhs[x] = reinterpret_cast<const ulonglong2 *>(lhs[x]);
        for (size_t j = 0; j < M; j++)
            h_outs[j] = reinterpret_cast<ulonglong2 *>(outs[j]);
        upload_table(d_rhs, h_rhs.data(), K, st, "upload right-hand table");
        upload_table(d_lhs, h_lhs.data(), M * K, st, "upload left-hand table");
        upload_table(d_outs, h_outs.data(), M, st, "upload output table");
        if (any)
            upload_table(d_cst, cst.data(), K * L, st, "upload term constants");

        const int window = sum_window(c, L, 2, kMultiplySumWindow);
        const int MT = M >= kMultiplySumTile ? kMultiplySumTile : static_cast<int>(M);
        const size_t tiles = (M + MT - 1) / MT;
        // per member: every right-hand pair once per output tile, every left-hand pair once, three output polynomials
        const double words = static_cast<double>(batch) * static_cast<double>(2 * K * tiles + 2 * M * K + 3 * M);
        c.stats.begin("multiply_sum", 0, 8.0 * words * static_cast<double>(ln), st);
        for (size_t b0 = 0; b0 < batch; b0 += 65535)
        {
            const dim3 grid(static_cast<unsigned>((half + 127) / 128), static_cast<unsigned>(std::min<size_t>(65535, batch - b0)), static_cast<unsigned>(tiles));
            const int args_l = static_cast<int>(L), args_k = static_cast<int>(K), args_m = static_cast<int>(M);
            const auto hl = static_cast<long long>(half), bb = static_cast<long long>(b0);
            if (MT == 1)
                multiply_sum_kernel<1><<<grid, 128, 0, st>>>(d_rhs, d_lhs, d_cst, d_outs, c.d_primes.get(), c.logn, args_l, args_k, args_m, window, bb, hl);
            else
                multiply_sum_kernel<kMultiplySumTile><<<grid, 128, 0, st>>>(d_rhs, d_lhs, d_cst, d_outs, c.d_primes.get(), c.logn, args_l, args_k, args_m,
                                                                              window, bb, hl);
            cuda_check(cudaGetLastError(), "multiply_sum_kernel");
        }
        c.stats.end(st);
    }
} // namespace sb
