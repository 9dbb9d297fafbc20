// seal_b200/csrc/sb_plainsum.cu -- sums of plaintext products: destination j = add_many over i of multiply_plain(ct_i, plain_{j K + i})
// in one pass over NTT-form operands (a plaintext matrix times a vector of ciphertexts).
//
// Reference behaviour being reproduced (paths under /root/reference/native/src/seal/):
//   evaluator.cpp:1975-2195 multiply_plain (the four NTT-form cases) -> operands brought to NTT form, then plain_sum_kernel
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

        size_t align16(size_t bytes) { return (bytes + 15) & ~size_t(15); }
    } // namespace

    void op_multiply_plain_sum(Context &c, size_t L, size_t batch, size_t K, size_t M, const size_t *sizes, const u64 *const *cts,
                               const size_t *plain_counts, const u64 *const *plains, bool ct_ntt, bool plain_ntt, const int *modes,
                               const u64 *factors, u64 *const *outs, cudaStream_t st)
    {
        const size_t ln = L * c.n, half = ln / 2;
        size_t out_size = 0;
        for (size_t t = 0; t < K; t++)
            out_size = std::max(out_size, sizes[t]);
        // add_many's left fold acc = acc e1_t +/- x_t e2_t (the factors of unscaled steps are 1), unrolled: term t enters the sum
        // times +/- e2_t prod_{u > t} e1_u.  The residues are exact, so the constants are formed mod q_i on the host.
        std::vector<Tw> cst(K * L);
        bool any = false;
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
        const size_t tab_bytes = align16(max_k * sizeof(SumTerm)) + align16(M * max_k * sizeof(SumPlain)) + align16(M * sizeof(u64 *)) +
                                 (any ? align16(max_k * L * sizeof(Tw)) : 0);
        auto *base = static_cast<unsigned char *>(c.ensure_scratch(tab_bytes + most));
        auto *d_terms = reinterpret_cast<SumTerm *>(base);
        auto *d_plains = reinterpret_cast<SumPlain *>(base + align16(max_k * sizeof(SumTerm)));
        auto *d_outs = reinterpret_cast<ulonglong2 **>(reinterpret_cast<unsigned char *>(d_plains) + align16(M * max_k * sizeof(SumPlain)));
        Tw *d_cst = any ? reinterpret_cast<Tw *>(reinterpret_cast<unsigned char *>(d_outs) + align16(M * sizeof(u64 *))) : nullptr;
        u64 *conv = reinterpret_cast<u64 *>(base + tab_bytes);
        std::vector<ulonglong2 *> h_outs(M);
        for (size_t j = 0; j < M; j++)
            h_outs[j] = reinterpret_cast<ulonglong2 *>(outs[j]);
        cuda_check(cudaMemcpyAsync(d_outs, h_outs.data(), M * sizeof(u64 *), cudaMemcpyHostToDevice, st), "upload output table");

        // the reduction window of this level: a carried residue plus `window` products of words below q stay below 2^128
        u64 qmax = 0;
        for (size_t i = 0; i < L; i++)
            qmax = std::max(qmax, c.q[i]);
        const unsigned __int128 sq = static_cast<unsigned __int128>(qmax - 1) * (qmax - 1);
        const int window = static_cast<int>(std::min<unsigned __int128>(kPlainSumWindow, sq ? (~static_cast<unsigned __int128>(0) - (qmax - 1)) / sq : kPlainSumWindow));
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
            cuda_check(cudaMemcpyAsync(d_terms, h_terms.data(), k * sizeof(SumTerm), cudaMemcpyHostToDevice, st), "upload term table");
            cuda_check(cudaMemcpyAsync(d_plains, h_plains.data(), M * k * sizeof(SumPlain), cudaMemcpyHostToDevice, st), "upload plain table");
            if (any)
                cuda_check(cudaMemcpyAsync(d_cst, cst.data() + t0 * L, k * L * sizeof(Tw), cudaMemcpyHostToDevice, st), "upload term constants");
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
} // namespace sb
