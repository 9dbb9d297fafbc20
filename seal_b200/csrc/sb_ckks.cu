// seal_b200/csrc/sb_ckks.cu -- CKKSEncoder::encode / decode on the device (ckks.h:455-807), the producer / consumer of the
// NTT-form plaintexts the evaluator works on.
//
// Floating point with an integer contract: the reference runs a double-precision complex FFT (util/dwthandler.h) over the slot
// values, rounds every coefficient to an integer and reduces it modulo each prime, so a plaintext is only reproducible bit for
// bit if every floating-point operation is the reference's, in the reference's order.  Each butterfly below is therefore written
// with the round-to-nearest intrinsics (__dadd_rn / __dsub_rn / __dmul_rn: never contracted into FMA), a complex product is
// (ac - bd, ad + bc) exactly as std::complex multiplies (with its Annex G recovery of infinities when both parts are NaN), the scaling by scale / n is merged into the last stage as
// DWTHandler::transform_from_rev does, and the root tables come from the host (sbh::ckks_tables: std::polar on one eighth of the
// circle + symmetry, util/croots.cpp).  The butterflies of one stage are independent, so the parallel schedule does not change
// any value.  After the transform the three decomposition branches of the reference (coefficients below 2^64, below 2^128,
// multi-precision) all reduce the same exact integer |round(c)| = mantissa * 2^exponent; one kernel does that for every size.
//
// Schedule: the stages with gap < 2^kFftLocalLog run in shared memory on contiguous blocks of 2^(kFftLocalLog+1)... (one CTA per block
// of 2048 points, 1024 threads, one butterfly per thread per stage); the remaining log n - 11 stages are one streaming kernel
// each.  At n = 65536 that is 6 passes over 1 MB per plaintext: noise next to the 31 NTTs that follow.
#include "sb_engine.cuh"
#include <cmath>
#include <cstring>

namespace sb
{
    namespace
    {
        constexpr int kFftLocalLog = 11; // points per CTA of the shared-memory part: 2^11 complex doubles = 32 KB

        __device__ __forceinline__ double2 cadd(double2 a, double2 b)
        {
            return make_double2(__dadd_rn(a.x, b.x), __dadd_rn(a.y, b.y));
        }
        __device__ __forceinline__ double2 csubd(double2 a, double2 b)
        {
            return make_double2(__dsub_rn(a.x, b.x), __dsub_rn(a.y, b.y));
        }
        // C99 Annex G (G.5.1) recovery of a complex product whose parts both came out NaN, as std::complex<double> multiplies under
        // g++: an infinite factor is boxed to +-1 / +-0 with the other factor's NaNs made 0 (or, when only a partial product overflowed,
        // every NaN is made 0), then the product is recomputed times infinity.  Reached only by non-finite operands.
        __device__ __noinline__ double2 cmul_recover(double2 p, double a, double b, double c, double d, bool overflowed)
        {
            bool recalc = false;
            if (isinf(a) || isinf(b))
            {
                a = copysign(isinf(a) ? 1.0 : 0.0, a), b = copysign(isinf(b) ? 1.0 : 0.0, b);
                c = isnan(c) ? copysign(0.0, c) : c, d = isnan(d) ? copysign(0.0, d) : d;
                recalc = true;
            }
            if (isinf(c) || isinf(d))
            {
                c = copysign(isinf(c) ? 1.0 : 0.0, c), d = copysign(isinf(d) ? 1.0 : 0.0, d);
                a = isnan(a) ? copysign(0.0, a) : a, b = isnan(b) ? copysign(0.0, b) : b;
                recalc = true;
            }
            if (!recalc && overflowed)
            {
                a = isnan(a) ? copysign(0.0, a) : a, b = isnan(b) ? copysign(0.0, b) : b;
                c = isnan(c) ? copysign(0.0, c) : c, d = isnan(d) ? copysign(0.0, d) : d;
                recalc = true;
            }
            if (!recalc)
                return p;
            const double inf = __longlong_as_double(0x7ff0000000000000ll);
            return make_double2(__dmul_rn(inf, __dsub_rn(__dmul_rn(a, c), __dmul_rn(b, d))), __dmul_rn(inf, __dadd_rn(__dmul_rn(a, d), __dmul_rn(b, c))));
        }
        __device__ __forceinline__ double2 cmul(double2 a, double2 r) // std::complex product: (ac - bd, ad + bc), Annex G on NaN
        {
            const double ac = __dmul_rn(a.x, r.x), bd = __dmul_rn(a.y, r.y), ad = __dmul_rn(a.x, r.y), bc = __dmul_rn(a.y, r.x);
            const double2 p = make_double2(__dsub_rn(ac, bd), __dadd_rn(ad, bc));
            if (isnan(p.x) && isnan(p.y))
                return cmul_recover(p, a.x, a.y, r.x, r.y, isinf(ac) || isinf(bd) || isinf(ad) || isinf(bc));
            return p;
        }
        __device__ __forceinline__ double2 cscale(double2 a, double s)
        {
            return make_double2(__dmul_rn(a.x, s), __dmul_rn(a.y, s));
        }

        // values [B][count] (complex: (re, im) pairs; real: one double) -> V[b][map[i]] = v, V[b][map[i + slots]] = conj(v).
        // broadcast: values [B], member b's one value in every slot (CKKSEncoder::encode of one complex number, ckks.h:794-800)
        __global__ void __launch_bounds__(256) ckks_scatter_kernel(const double *__restrict__ values, int is_complex, int broadcast, long long count,
                                                                   const uint32_t *__restrict__ map, double2 *__restrict__ V, int logn,
                                                                   long long total, int *flags)
        {
            const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
            if (e >= total)
                return;
            const long long b = e / count, i = e % count, src = broadcast ? b : e;
            const long long n = 1ll << logn, slots = n >> 1;
            double re, im = 0.0;
            if (is_complex)
                re = values[2 * src], im = values[2 * src + 1];
            else
                re = values[src];
            if (!isfinite(re) || !isfinite(im))
                atomicOr(flags, 1); // "values must be finite"
            V[b * n + map[i]] = make_double2(re, im);
            V[b * n + map[i + slots]] = make_double2(re, -im);
        }

        // DWTHandler::transform_from_rev, the stages with gap < 2^local (gap = 1, 2, ...): stage with gap g has m = n / 2g groups, group i
        // uses inv_roots[n - 2m + i + 1]; the stage with m == 1 (only reached here when n <= 2^kFftLocalLog) carries the scalar
        __global__ void __launch_bounds__(1024) ckks_ifft_local_kernel(double2 *__restrict__ V, const double2 *__restrict__ inv_roots, int logn,
                                                                       int local, double scalar)
        {
            extern __shared__ double2 sm[];
            const long long n = 1ll << logn;
            const int pts = 1 << local, t = threadIdx.x;
            const long long blocks_per_poly = n >> local;
            const long long poly = blockIdx.x / blocks_per_poly, blk = blockIdx.x % blocks_per_poly;
            double2 *base = V + poly * n + blk * pts;
            for (int i = t; i < pts; i += blockDim.x)
                sm[i] = base[i];
            __syncthreads();
            for (int s = 0; s < local; s++)
            {
                const int gap = 1 << s;
                const long long m = n >> (s + 1);
                for (int w = t; w < pts / 2; w += blockDim.x)
                {
                    const int g = w >> s, j = w & (gap - 1), xi = (g << (s + 1)) + j;
                    const long long gi = (blk << (local - s - 1)) + g; // group index within the polynomial
                    const double2 r = inv_roots[n - 2 * m + gi + 1];
                    const double2 u = sm[xi], v = sm[xi + gap];
                    if (m > 1)
                    {
                        sm[xi] = cadd(u, v);
                        sm[xi + gap] = cmul(csubd(u, v), r);
                    }
                    else
                    {
                        sm[xi] = cscale(cadd(u, v), scalar);
                        sm[xi + gap] = cmul(csubd(u, v), cscale(r, scalar));
                    }
                }
                __syncthreads();
            }
            for (int i = t; i < pts; i += blockDim.x)
                base[i] = sm[i];
        }

        // one stage (gap = 2^s) over global memory; LAST: the scaled stage (m == 1)
        template <bool LAST>
        __global__ void __launch_bounds__(256) ckks_ifft_stage_kernel(double2 *__restrict__ V, const double2 *__restrict__ inv_roots, int logn, int s,
                                                                      double scalar, long long total)
        {
            const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over B * n / 2 butterflies
            if (e >= total)
                return;
            const long long n = 1ll << logn, half = n >> 1, poly = e / half, w = e % half;
            const long long gap = 1ll << s, m = n >> (s + 1), g = w >> s, j = w & (gap - 1);
            double2 *x = V + poly * n + (g << (s + 1)) + j, *y = x + gap;
            const double2 r = inv_roots[n - 2 * m + g + 1];
            const double2 u = *x, v = *y;
            if (!LAST)
            {
                *x = cadd(u, v);
                *y = cmul(csubd(u, v), r);
            }
            else
            {
                *x = cscale(cadd(u, v), scalar);
                *y = cmul(csubd(u, v), cscale(r, scalar));
            }
        }

        // max |Re c| (as the bit pattern of a non-negative double: ordered like the integers) and the NaN flag (ckks.h:525-545)
        __global__ void __launch_bounds__(256) ckks_max_kernel(const double2 *__restrict__ V, long long total, unsigned long long *max_bits, int *flags)
        {
            const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
            double a = 0.0;
            if (e < total)
                a = fabs(V[e].x);
            if (isnan(a))
            {
                atomicOr(flags, 2);
                a = 0.0;
            }
            unsigned long long bits = static_cast<unsigned long long>(__double_as_longlong(a));
            for (int o = 16; o; o >>= 1)
            {
                const unsigned long long other = __shfl_xor_sync(0xffffffffu, bits, o);
                bits = other > bits ? other : bits;
            }
            if ((threadIdx.x & 31) == 0 && bits)
                atomicMax(max_bits, bits);
        }

        // round(c) of a finite double as sign and magnitude, |round(c)| = mant * 2^ex exactly.  The reference's three decomposition
        // branches (below 2^64, below 2^128, multi-precision: ckks.h:556-668 for vectors, ckks.cpp:152-226 for one real) all reduce
        // this same integer, so every encoder reduces it through ckks_decompose + ckks_residue
        struct CkksCoeff
        {
            u64 mant;
            int ex;
            bool negative;
        };
        __device__ __forceinline__ CkksCoeff ckks_decompose(double c)
        {
            double d = round(c); // half away from zero, like std::round
            CkksCoeff k{ 0, 0, static_cast<bool>(signbit(d)) };
            d = fabs(d);
            if (d >= 1.0)
            {
                if (d < 18446744073709551616.0)
                    k.mant = __double2ull_rz(d);
                else
                {
                    const long long bits = __double_as_longlong(d);
                    k.ex = static_cast<int>((bits >> 52) & 0x7ff) - 1075; // d = (2^52 + fraction) * 2^ex, ex >= 12 here
                    k.mant = (static_cast<u64>(bits) & 0xFFFFFFFFFFFFFull) | (1ull << 52);
                }
            }
            return k;
        }
        // round(c) mod q, canonical; a negative value is negated modulo q with 0 kept as 0 (negate_uint_mod)
        __device__ __forceinline__ u64 ckks_residue(const CkksCoeff &k, const PrimeDev &P)
        {
            u64 r = barrett64(k.mant, P.q, P.ratio_hi);
            for (int left = k.ex; left > 0; left -= 32) // times 2^ex, 32 bits at a time (large coefficients only)
                r = mulmod_barrett(r, 1ull << (left >= 32 ? 32 : left), P);
            return k.negative && r ? P.q - r : r;
        }

        // round(Re c) -> residues modulo every prime of the level (ckks.h:556-668)
        __global__ void __launch_bounds__(256) ckks_reduce_kernel(const double2 *__restrict__ V, u64 *__restrict__ out, const PrimeDev *__restrict__ primes,
                                                                  int logn, int L, long long total)
        {
            const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over B * n
            if (e >= total)
                return;
            const long long n = 1ll << logn, b = e >> logn, i = e & (n - 1);
            const CkksCoeff k = ckks_decompose(V[e].x);
            u64 *dst = out + b * L * n + i;
            for (int j = 0; j < L; j++)
            {
                const PrimeDev P = primes[j];
                dst[static_cast<long long>(j) * n] = ckks_residue(k, P);
            }
        }

        // CKKSEncoder::encode of one real (kind kCkksScalarReal: value * scale, ckks.cpp:75-230) or one int64 (kCkksScalarInt64,
        // ckks.cpp:232-287) per member: the plaintext is the constant polynomial, so in NTT form every word of row (b, j) of out
        // [B][L][n] is the same residue.  One CTA per row: thread 0 computes the residue once, then the CTA writes the row with
        // 16-byte stores (VEC; 8-byte stores when out is not 16-byte aligned).  A pure write stream of B L n 8 bytes.
        template <bool VEC>
        __global__ void __launch_bounds__(256) ckks_fill_kernel(const u64 *__restrict__ values, int kind, double scale, const PrimeDev *__restrict__ primes,
                                                                int logn, int L, u64 *__restrict__ out)
        {
            __shared__ u64 word;
            const long long row = blockIdx.x, n = 1ll << logn;
            if (threadIdx.x == 0)
            {
                const long long b = row / L;
                const PrimeDev P = primes[row % L];
                const u64 v = values[b];
                if (kind == kCkksScalarInt64)
                    // the reference adds q_j to the two's-complement word of a negative value before its Barrett reduction. For |v| > q_j
                    // that 64-bit sum does not wrap, so the word is (2^64 - |v|) mod q_j rather than -|v| mod q_j: kept, to be bit-exact
                    word = barrett64(static_cast<long long>(v) < 0 ? v + P.q : v, P.q, P.ratio_hi);
                else
                    word = ckks_residue(ckks_decompose(__dmul_rn(__longlong_as_double(static_cast<long long>(v)), scale)), P);
            }
            __syncthreads();
            const u64 w = word;
            if (VEC)
            {
                ulonglong2 *dst = reinterpret_cast<ulonglong2 *>(out + row * n);
                const ulonglong2 w2 = make_ulonglong2(w, w);
                for (long long i = threadIdx.x; i < n / 2; i += blockDim.x)
                    dst[i] = w2;
            }
            else
            {
                u64 *dst = out + row * n;
                for (long long i = threadIdx.x; i < n; i += blockDim.x)
                    dst[i] = w;
            }
        }

        // ---- decode ----
        // RNSBase::compose (rns.cpp:321-352) of one coefficient (crt_compose, sb_device.cuh) + the conversion to double (ckks.h:740-778).
        // big = [Q (L) | threshold (L) | punctured (L * L)] words; one thread per coefficient, the L-word integers in local memory
        __global__ void __launch_bounds__(128) ckks_compose_kernel(const u64 *__restrict__ coef, const u64 *__restrict__ big, const Tw *__restrict__ invp,
                                                                   const PrimeDev *__restrict__ primes, double2 *__restrict__ V, int logn, int L,
                                                                   double inv_scale, long long total)
        {
            const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over B * n
            if (e >= total)
                return;
            const long long n = 1ll << logn, b = e >> logn, i = e & (n - 1);
            const u64 *Q = big, *thr = big + L, *punct = big + 2 * L;
            u64 val[kCrtMaxWords];
            const u64 *src = coef + b * L * n + i;
            crt_compose([&](int j) { return src[static_cast<long long>(j) * n]; }, Q, punct, invp, primes, L, val);
            bool upper = true; // is_greater_than_or_equal_uint(value, upper_half_threshold)
            for (int w = L - 1; w >= 0; w--)
                if (val[w] != thr[w])
                {
                    upper = val[w] > thr[w];
                    break;
                }
            // the reference accumulates word by word in doubles, the words of Q - value taken WORDWISE (no borrow): keep that
            double acc = 0.0, s64 = inv_scale;
            for (int w = 0; w < L; w++, s64 = __dmul_rn(s64, 18446744073709551616.0))
            {
                if (upper)
                {
                    if (val[w] > Q[w])
                    {
                        const u64 diff = val[w] - Q[w];
                        acc = __dadd_rn(acc, __dmul_rn(__ull2double_rn(diff), s64));
                    }
                    else
                    {
                        const u64 diff = Q[w] - val[w];
                        acc = __dsub_rn(acc, diff ? __dmul_rn(__ull2double_rn(diff), s64) : 0.0);
                    }
                }
                else
                    acc = __dadd_rn(acc, val[w] ? __dmul_rn(__ull2double_rn(val[w]), s64) : 0.0);
            }
            V[e] = make_double2(acc, 0.0);
        }

        // DWTHandler::transform_to_rev: stage with m groups (gap = n / 2m), group i uses roots[m + i]; u, v = y r; x = u + v, y = u - v
        __global__ void __launch_bounds__(256) ckks_fft_stage_kernel(double2 *__restrict__ V, const double2 *__restrict__ roots, int logn, int s,
                                                                     long long total)
        {
            const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
            if (e >= total)
                return;
            const long long n = 1ll << logn, half = n >> 1, poly = e / half, w = e % half;
            const long long gap = 1ll << s, m = n >> (s + 1), g = w >> s, j = w & (gap - 1);
            double2 *x = V + poly * n + (g << (s + 1)) + j, *y = x + gap;
            const double2 u = *x, v = cmul(*y, roots[m + g]);
            *x = cadd(u, v);
            *y = csubd(u, v);
        }
        // the stages with gap < 2^local (gap = 2^(local-1) ... 1) in shared memory
        __global__ void __launch_bounds__(1024) ckks_fft_local_kernel(double2 *__restrict__ V, const double2 *__restrict__ roots, int logn, int local)
        {
            extern __shared__ double2 sm[];
            const long long n = 1ll << logn;
            const int pts = 1 << local, t = threadIdx.x;
            const long long blocks_per_poly = n >> local;
            const long long poly = blockIdx.x / blocks_per_poly, blk = blockIdx.x % blocks_per_poly;
            double2 *base = V + poly * n + blk * pts;
            for (int i = t; i < pts; i += blockDim.x)
                sm[i] = base[i];
            __syncthreads();
            for (int s = local - 1; s >= 0; s--)
            {
                const int gap = 1 << s;
                const long long m = n >> (s + 1);
                for (int w = t; w < pts / 2; w += blockDim.x)
                {
                    const int g = w >> s, j = w & (gap - 1), xi = (g << (s + 1)) + j;
                    const long long gi = (blk << (local - s - 1)) + g;
                    const double2 u = sm[xi], v = cmul(sm[xi + gap], roots[m + gi]);
                    sm[xi] = cadd(u, v);
                    sm[xi + gap] = csubd(u, v);
                }
                __syncthreads();
            }
            for (int i = t; i < pts; i += blockDim.x)
                base[i] = sm[i];
        }
        // destination[i] = res[map[i]], i < n / 2 (ckks.h:782-785)
        __global__ void __launch_bounds__(256) ckks_gather_kernel(const double2 *__restrict__ V, const uint32_t *__restrict__ map, double2 *__restrict__ out,
                                                                  int logn, long long total)
        {
            const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over B * n / 2
            if (e >= total)
                return;
            const long long slots = 1ll << (logn - 1), b = e / slots, i = e % slots;
            out[e] = V[(b << logn) + map[i]];
        }

        unsigned grid_for(long long total, int threads)
        {
            return static_cast<unsigned>((total + threads - 1) / threads);
        }
    } // namespace

    Context::CkksEncoder &ckks_encoder(Context &c)
    {
        if (c.ckks.d_stat)
            return c.ckks;
        if (c.scheme != 2)
            throw std::invalid_argument("unsupported scheme");
        const sbh::CkksTables t = sbh::ckks_tables(c.n);
        Context::CkksEncoder enc;
        enc.d_roots = upload<double2>(c, t.roots);
        enc.d_inv_roots = upload<double2>(c, t.inv_roots);
        enc.d_map = upload<uint32_t>(c, sbh::batch_index_map(c.n)); // matrix_reps_index_map_: the same map BatchEncoder uses
        enc.d_stat = DevBuf<u64>(2);
        c.table_bytes += enc.d_stat.bytes();
        return c.ckks = std::move(enc);
    }

    // values: device, [B][count] complex (re, im) pairs or reals; plain: device, [B][L][n] NTT form.  Synchronises the stream once
    // (the reference's "encoded values are too large" check needs the largest coefficient before the plaintext is produced).
    void op_ckks_encode(Context &c, size_t L, size_t B, const double *values, size_t count, bool is_complex, double scale, u64 *plain,
                        cudaStream_t st, bool broadcast)
    {
        auto &enc = ckks_encoder(c);
        if (L < 1 || L > c.k)
            throw std::invalid_argument("parms_id is not valid for encryption parameters");
        if (count > c.n / 2)
            throw std::invalid_argument("values_size is too large");
        if (count && !values)
            throw std::invalid_argument("values cannot be null");
        const int total_bits = crt_level(c, L).total_bits;
        // ckks.h:494-499
        if (!std::isnormal(scale) || scale <= 0 || (static_cast<int>(std::log2(scale)) + 1 >= total_bits))
            throw std::invalid_argument("scale out of bounds");
        if (!B)
            return;
        const long long n = static_cast<long long>(c.n), logn = c.logn;
        double2 *V = static_cast<double2 *>(c.ensure_aux(B * c.n * sizeof(double2)));
        cuda_check(cudaMemsetAsync(V, 0, B * c.n * sizeof(double2), st), "memset");
        cuda_check(cudaMemsetAsync(enc.d_stat.get(), 0, 16, st), "memset");
        unsigned long long *d_max = enc.d_stat.get();
        int *d_flags = reinterpret_cast<int *>(d_max + 1);
        if (count)
        {
            const long long total = static_cast<long long>(B) * static_cast<long long>(count);
            c.stats.begin("ckks_scatter", 0, 48.0 * total, st);
            ckks_scatter_kernel<<<grid_for(total, 256), 256, 0, st>>>(values, is_complex ? 1 : 0, broadcast ? 1 : 0, static_cast<long long>(count),
                                                                      enc.d_map.get(), V, static_cast<int>(logn), total, d_flags);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "ckks_scatter_kernel");
        }
        const double fix = scale / static_cast<double>(c.n); // ckks.h:522
        const int local = static_cast<int>(std::min<long long>(logn, kFftLocalLog));
        c.stats.begin("ckks_ifft_local", 0, 32.0 * B * n, st);
        ckks_ifft_local_kernel<<<static_cast<unsigned>(B * (c.n >> local)), std::min(1024, 1 << (local > 0 ? local - 1 : 0)),
                                 (size_t(1) << local) * sizeof(double2), st>>>(V, enc.d_inv_roots.get(), static_cast<int>(logn), local, fix);
        c.stats.end(st);
        cuda_check(cudaGetLastError(), "ckks_ifft_local_kernel");
        const long long bflies = static_cast<long long>(B) * (n / 2);
        for (int s = local; s < logn; s++)
        {
            c.stats.begin("ckks_ifft_stage", s, 32.0 * B * n, st);
            if (s + 1 < logn)
                ckks_ifft_stage_kernel<false><<<grid_for(bflies, 256), 256, 0, st>>>(V, enc.d_inv_roots.get(), static_cast<int>(logn), s, fix, bflies);
            else
                ckks_ifft_stage_kernel<true><<<grid_for(bflies, 256), 256, 0, st>>>(V, enc.d_inv_roots.get(), static_cast<int>(logn), s, fix, bflies);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "ckks_ifft_stage_kernel");
        }
        const long long total = static_cast<long long>(B) * n;
        c.stats.begin("ckks_max", 0, 16.0 * total, st);
        ckks_max_kernel<<<grid_for(total, 256), 256, 0, st>>>(V, total, d_max, d_flags);
        c.stats.end(st);
        cuda_check(cudaGetLastError(), "ckks_max_kernel");
        struct
        {
            unsigned long long max_bits;
            int flags, pad;
        } stat;
        cuda_check(cudaMemcpyAsync(&stat, enc.d_stat.get(), 16, cudaMemcpyDeviceToHost, st), "status D2H");
        cuda_check(cudaStreamSynchronize(st), "synchronize");
        if (stat.flags & 1)
            throw std::invalid_argument("values must be finite");
        double max_coeff;
        std::memcpy(&max_coeff, &stat.max_bits, sizeof(double));
        // ckks.h:533-553
        if ((stat.flags & 2) || !std::isfinite(max_coeff))
            throw std::invalid_argument("encoded values are too large");
        const int max_coeff_bit_count = static_cast<int>(std::ceil(std::log2(std::max(max_coeff, 1.0)))) + 1;
        if (max_coeff_bit_count >= total_bits)
            throw std::invalid_argument("encoded values are too large");
        c.stats.begin("ckks_reduce", 0, (16.0 + 8.0 * L) * total, st);
        ckks_reduce_kernel<<<grid_for(total, 256), 256, 0, st>>>(V, plain, c.d_primes.get(), static_cast<int>(logn), static_cast<int>(L), total);
        c.stats.end(st);
        cuda_check(cudaGetLastError(), "ckks_reduce_kernel");
        op_ntt(c, false, L, 1, B, plain, st);
    }

    void check_ckks_scalar(const Context &c, size_t L, int kind, double scale)
    {
        if (kind != kCkksScalarReal && kind != kCkksScalarComplex && kind != kCkksScalarInt64)
            throw std::invalid_argument("kind must be SB200_CKKS_SCALAR_REAL, SB200_CKKS_SCALAR_COMPLEX or SB200_CKKS_SCALAR_INT64");
        if (c.scheme != 2)
            throw std::invalid_argument("unsupported scheme"); // ckks.cpp:22-25
        if (L < 1 || L > c.k)
            throw std::invalid_argument("parms_id is not valid for encryption parameters");
        const int total_bits = sbh::product_bit_count(c.q.data(), L);
        // one real: ckks.cpp:96-101 (isfinite, no +1); one complex: the vector path's test, ckks.h:494-499
        if (kind == kCkksScalarReal && (!std::isfinite(scale) || scale <= 0 || static_cast<int>(std::log2(scale)) >= total_bits))
            throw std::invalid_argument("scale out of bounds");
        if (kind == kCkksScalarComplex && (!std::isnormal(scale) || scale <= 0 || static_cast<int>(std::log2(scale)) + 1 >= total_bits))
            throw std::invalid_argument("scale out of bounds");
    }

    void check_ckks_scalar_values(const Context &c, size_t L, size_t B, int kind, const u64 *h_values, double scale)
    {
        const int total_bits = sbh::product_bit_count(c.q.data(), L);
        for (size_t b = 0; b < B; b++)
        {
            if (kind == kCkksScalarInt64) // ckks.cpp:253-257; |INT64_MIN| = 2^63, which llabs yields on two's-complement targets
            {
                const u64 v = h_values[b], mag = static_cast<int64_t>(v) < 0 ? 0 - v : v;
                if ((mag ? 64 - __builtin_clzll(mag) : 0) + 2 >= total_bits)
                    throw std::invalid_argument("encoded value is too large");
            }
            else if (kind == kCkksScalarReal) // ckks.cpp:103-124; value * scale is the kernel's product (one IEEE multiply)
            {
                double value;
                std::memcpy(&value, h_values + b, sizeof(double));
                if (!std::isfinite(value))
                    throw std::invalid_argument("value must be finite");
                const double p = value * scale;
                if (!std::isfinite(p))
                    throw std::invalid_argument("encoded value is too large");
                const int coeff_bit_count = std::fabs(p) < 1.0 ? 2 : static_cast<int>(std::log2(std::fabs(p))) + 2;
                if (coeff_bit_count >= total_bits)
                    throw std::invalid_argument("encoded value is too large");
            }
        }
    }

    void op_ckks_encode_scalar(Context &c, size_t L, size_t B, int kind, const u64 *values, double scale, u64 *plain, cudaStream_t st)
    {
        check_ckks_scalar(c, L, kind, scale);
        if (!B)
            return;
        if (kind == kCkksScalarComplex) // ckks.h:794-800: slots copies through the vector path, read from one pair per member
        {
            op_ckks_encode(c, L, B, reinterpret_cast<const double *>(values), c.n / 2, true, scale, plain, st, true);
            return;
        }
        std::vector<u64> h(B);
        cuda_check(cudaMemcpyAsync(h.data(), values, B * sizeof(u64), cudaMemcpyDeviceToHost, st), "values D2H");
        cuda_check(cudaStreamSynchronize(st), "synchronize");
        check_ckks_scalar_values(c, L, B, kind, h.data(), scale);
        const unsigned rows = static_cast<unsigned>(B * L);
        c.stats.begin("ckks_fill", 0, 8.0 * B * L * c.n, st);
        if (reinterpret_cast<uintptr_t>(plain) % sizeof(ulonglong2) == 0)
            ckks_fill_kernel<true><<<rows, 256, 0, st>>>(values, kind, scale, c.d_primes.get(), c.logn, static_cast<int>(L), plain);
        else
            ckks_fill_kernel<false><<<rows, 256, 0, st>>>(values, kind, scale, c.d_primes.get(), c.logn, static_cast<int>(L), plain);
        c.stats.end(st);
        cuda_check(cudaGetLastError(), "ckks_fill_kernel");
    }

    // plain: device [B][L][n] NTT form, scale = Plaintext::scale(); values out: device [B][n/2] complex (re, im)
    void op_ckks_decode(Context &c, size_t L, size_t B, const u64 *plain, double scale, double *values, cudaStream_t st)
    {
        auto &enc = ckks_encoder(c);
        if (L < 1 || L > c.k || L > static_cast<size_t>(kCrtMaxWords))
            throw std::invalid_argument("plain is not valid for encryption parameters");
        auto &lv = crt_level(c, L);
        // ckks.h:712-716
        if (!std::isnormal(scale) || scale <= 0 || (static_cast<int>(std::log2(scale)) >= lv.total_bits))
            throw std::invalid_argument("scale out of bounds");
        if (!B)
            return;
        const long long n = static_cast<long long>(c.n), logn = c.logn, total = static_cast<long long>(B) * n;
        const size_t coef_bytes = B * L * c.n * sizeof(u64);
        unsigned char *arena = static_cast<unsigned char *>(c.ensure_aux(coef_bytes + B * c.n * sizeof(double2)));
        u64 *coef = reinterpret_cast<u64 *>(arena);
        double2 *V = reinterpret_cast<double2 *>(arena + coef_bytes);
        cuda_check(cudaMemcpyAsync(coef, plain, coef_bytes, cudaMemcpyDeviceToDevice, st), "copy");
        op_ntt(c, true, L, 1, B, coef, st);
        const double inv_scale = 1.0 / scale;
        c.stats.begin("ckks_compose", 0, (8.0 * L + 16.0) * total, st);
        ckks_compose_kernel<<<grid_for(total, 128), 128, 0, st>>>(coef, lv.d_big.get(), lv.d_invp.get(), c.d_primes.get(), V, static_cast<int>(logn), static_cast<int>(L),
                                                                  inv_scale, total);
        c.stats.end(st);
        cuda_check(cudaGetLastError(), "ckks_compose_kernel");
        const int local = static_cast<int>(std::min<long long>(logn, kFftLocalLog));
        const long long bflies = static_cast<long long>(B) * (n / 2);
        for (int s = static_cast<int>(logn) - 1; s >= local; s--)
        {
            c.stats.begin("ckks_fft_stage", s, 32.0 * B * n, st);
            ckks_fft_stage_kernel<<<grid_for(bflies, 256), 256, 0, st>>>(V, enc.d_roots.get(), static_cast<int>(logn), s, bflies);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "ckks_fft_stage_kernel");
        }
        c.stats.begin("ckks_fft_local", 0, 32.0 * B * n, st);
        ckks_fft_local_kernel<<<static_cast<unsigned>(B * (c.n >> local)), std::min(1024, 1 << (local > 0 ? local - 1 : 0)),
                                (size_t(1) << local) * sizeof(double2), st>>>(V, enc.d_roots.get(), static_cast<int>(logn), local);
        c.stats.end(st);
        cuda_check(cudaGetLastError(), "ckks_fft_local_kernel");
        c.stats.begin("ckks_gather", 0, 16.0 * total, st);
        ckks_gather_kernel<<<grid_for(total / 2, 256), 256, 0, st>>>(V, enc.d_map.get(), reinterpret_cast<double2 *>(values), static_cast<int>(logn), total / 2);
        c.stats.end(st);
        cuda_check(cudaGetLastError(), "ckks_gather_kernel");
    }
} // namespace sb
