// seal_b200/csrc/sb_engine.cu -- device context, fused prologue/epilogue functors and the operation drivers for
// NTT, CKKS multiply, hybrid key switching (relinearize / apply_galois), rescale and modulus switching.
//
// Reference behaviour being reproduced (paths under /root/reference/native/src/seal/):
//   evaluator.cpp:569-708   ckks_multiply            -> ckks_tensor_kernel
//   evaluator.cpp:2561-2867 switch_key_inplace       -> key_switch_chunk(): INTT(target) | integer path (sb_ksint.cu) or digit NTTs | MAC | mod-down
//   evaluator.cpp:1144-1199 relinearize_internal     -> op_relinearize / op_multiply_relinearize
//   evaluator.cpp:2384-2502 apply_galois_inplace     -> op_apply_galois (permutation fused into the loads)
//   evaluator.cpp:1201-1294 + rns.cpp:789-901        -> op_rescale / op_mod_switch
#include "sb_engine.cuh"
#include "sb_src.cuh"
#include <algorithm>
#include <cstdlib>
#include <cstring>

#ifndef SB_MAC_MIN_BLOCKS
#define SB_MAC_MIN_BLOCKS 2 // CTAs per SM the fused key-switch kernel is register-tuned for
#endif

namespace sb
{
    void cuda_check(cudaError_t e, const char *what)
    {
        if (e != cudaSuccess)
            throw CudaError(std::string(what) + ": " + cudaGetErrorString(e));
    }

    // ------------------------------------------------------------------------------------------- context ----
    void *Context::ensure_scratch(size_t bytes)
    {
        scratch.grow(bytes);
        scratch_used = bytes;
        return scratch.get();
    }

    void Context::wipe_scratch(cudaStream_t st)
    {
        if (scratch && scratch_used)
            cuda_check(cudaMemsetAsync(scratch.get(), 0, std::min(scratch_used, scratch.bytes()), st), "wipe scratch");
    }

    void Context::wipe_aux(cudaStream_t st)
    {
        if (aux_buf && aux_used)
            cuda_check(cudaMemsetAsync(aux_buf.get(), 0, std::min(aux_used, aux_buf.bytes()), st), "wipe aux");
    }

    void *Context::ensure_aux(size_t bytes)
    {
        aux_buf.grow(bytes);
        aux_used = bytes;
        return aux_buf.get();
    }

    const uint32_t *Context::galois_table(uint32_t elt)
    {
        auto it = galois_tables.find(elt);
        if (it == galois_tables.end())
            it = galois_tables.emplace(elt, upload<uint32_t>(*this, sbh::galois_table_ntt(n, elt))).first;
        return it->second.get();
    }

    static Tw to_tw(const sbh::TwPair &p)
    {
        Tw t;
        t.w = p.w;
        t.wq = p.wq;
        return t;
    }

    static void upload_prime(Context &c, const sbh::PrimeTables &pt, std::vector<PrimeDev> &hp)
    {
        static_assert(sizeof(sbh::TwPair) == sizeof(Tw), "layout");
        c.d_fwd.push_back(upload<Tw>(c, pt.fwd));
        c.d_inv.push_back(upload<Tw>(c, pt.inv));
        PrimeDev d;
        d.q = pt.q;
        d.q2 = 2 * pt.q;
        d.q4 = 4 * pt.q;
        d.nq = 0ull - pt.q;
        d.zero = 0;
        d.ratio_lo = pt.ratio_lo;
        d.ratio_hi = pt.ratio_hi;
        d.inv_n = to_tw(pt.inv_n);
        d.inv_n_w = to_tw(pt.inv_n_w);
        d.fwd = c.d_fwd.back().get();
        d.inv = c.d_inv.back().get();
        {
            int bits = 0;
            while (bits < 64 && (pt.q >> bits))
                bits++;
            d.sh = bits - 2;
            d.mu = static_cast<u64>((static_cast<unsigned __int128>(1) << (bits + 62)) / pt.q);
            d.pad_ = 0;
        }
        hp.push_back(d);
    }

    std::unique_ptr<Context> make_context(int scheme, size_t n, const u64 *moduli, size_t k, u64 t, int device)
    {
        if (scheme != 1 && scheme != 2 && scheme != 3)
            throw std::invalid_argument("unsupported scheme");
        if (n < 2 || (n & (n - 1)) || n > 131072)
            throw std::invalid_argument("poly_modulus_degree is invalid");
        if (k < 1 || k > 256)
            throw std::invalid_argument("coeff_modulus size is invalid");
        int ndev = 0;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
            throw CudaError("no CUDA device available (libseal_b200 has no CPU fallback)");
        if (device < 0 || device >= ndev)
            throw std::invalid_argument("device index out of range");
        cuda_check(cudaSetDevice(device), "cudaSetDevice");
        cudaDeviceProp prop;
        cuda_check(cudaGetDeviceProperties(&prop, device), "cudaGetDeviceProperties");
        if (prop.major != 9 || prop.minor != 0)
            throw CudaError("libseal_b200 is built for sm_90a (H100) only; found compute capability " +
                            std::to_string(prop.major) + "." + std::to_string(prop.minor));

        auto c = std::make_unique<Context>();
        c->scheme = scheme, c->n = n, c->k = k, c->t = t, c->device = device, c->logn = sbh::ilog2(n);
        if (const char *e = std::getenv("SB200_SCRATCH_MB"))
            c->scratch_budget = static_cast<size_t>(std::max(64L, std::atol(e))) << 20;
        for (size_t i = 0; i < k; i++)
        {
            if (moduli[i] >> 61)
                throw std::invalid_argument("coeff_modulus primes must be below 2^61");
            for (size_t j = 0; j < i; j++)
                if (moduli[j] == moduli[i])
                    throw std::invalid_argument("coeff_modulus primes must be distinct");
            c->q.push_back(moduli[i]);
            if (moduli[i] >> 57)
                c->fast_q = false; // the guard-free forward butterflies need (4 + 4*17) q < 2^64
        }
        if (scheme == 1)
        {
            if (t < 2 || (t >> 60))
                throw std::invalid_argument("plain_modulus is invalid");
            // all levels use prefixes of one auxiliary list: [m_sk, gamma, B_0, B_1, ...]  (rns.cpp:626-632); the key level (L = k)
            // may need k + 1 primes of B, and BFV multiplication takes at most kBfvMultiplyMaxBase
            size_t max_nb = std::min(k + 1, kBfvMultiplyMaxBase);
            c->aux = sbh::get_primes(2 * static_cast<u64>(n), 61, max_nb + 2);
        }
        if (scheme == 3)
        {
            // BGV: q_j^-1 mod t for every prime (RNSTool::inv_q_last_mod_t of each level, rns.cpp:778-787)
            if (t < 2 || (t >> 60))
                throw std::invalid_argument("plain_modulus is invalid");
            c->t_ratio = static_cast<u64>((static_cast<unsigned __int128>(1) << 64) / t);
            for (size_t j = 0; j < k; j++)
            {
                u64 v = 0;
                if (!sbh::invmod(c->q[j] % t, t, v))
                    throw std::logic_error("invalid rns bases");
                c->inv_q_mod_t.push_back(v);
            }
        }
        std::vector<PrimeDev> hp;
        c->tabs.resize(k + c->aux.size());
        for (size_t i = 0; i < k; i++)
            c->tabs[i].build(n, c->q[i]);
        for (size_t i = 0; i < c->aux.size(); i++)
            if (i != 1) // gamma is only used by decryption
                c->tabs[k + i].build(n, c->aux[i]);
        if (scheme != 2 && t > 2 && (t - 1) % (2 * n) == 0 && sbh::is_prime(t))
        {
            // plain_ntt_tables (context.cpp:374-394): batching is available, t gets transform tables of its own
            c->t_pid = static_cast<int>(c->tabs.size());
            c->tabs.emplace_back();
            c->tabs.back().build(n, t);
        }
        for (size_t i = 0; i < c->tabs.size(); i++)
        {
            if (c->tabs[i].q == 0)
            {
                c->d_fwd.emplace_back();
                c->d_inv.emplace_back();
                hp.push_back(PrimeDev{});
                continue;
            }
            upload_prime(*c, c->tabs[i], hp);
        }
        c->nprimes = hp.size();
        c->d_primes = upload<PrimeDev>(*c, hp);
        // q_j^-1 mod q_i (rns.cpp:767-776 for every level at once)
        std::vector<Tw> invq(k * k);
        for (size_t j = 0; j < k; j++)
            for (size_t i = 0; i < k; i++)
            {
                Tw tw{ 0, 0 };
                if (i != j)
                {
                    u64 v = 0;
                    if (!sbh::invmod(c->q[j] % c->q[i], c->q[i], v))
                        throw std::logic_error("invalid rns bases");
                    tw.w = v;
                    tw.wq = sbh::shoup(v, c->q[i]);
                }
                invq[j * k + i] = tw;
            }
        c->d_invq = upload<Tw>(*c, invq);
        if (c->t_pid >= 0)
        {
            const auto map = sbh::batch_index_map(n);
            std::vector<uint32_t> inv(n);
            for (size_t i = 0; i < n; i++)
                inv[map[i]] = static_cast<uint32_t>(i);
            c->d_batch_inv_map = upload<uint32_t>(*c, inv);
        }
        for (size_t L = 1; L <= k; L++)
        {
            std::array<u64, 4> id;
            sbw::parms_id(scheme, n, c->q.data(), L, scheme == 2 ? 0 : t, id.data());
            c->parms_ids.push_back(id);
        }
        if (scheme == 3)
        {
            // q_j mod q_i with its Shoup quotient (the "k * q_last" term of the BGV mod-down, rns.cpp:1222-1224)
            std::vector<Tw> qmod(k * k);
            for (size_t j = 0; j < k; j++)
                for (size_t i = 0; i < k; i++)
                {
                    const u64 v = c->q[j] % c->q[i];
                    qmod[j * k + i] = Tw{ v, sbh::shoup(v, c->q[i]) };
                }
            c->d_qmod = upload<Tw>(*c, qmod);
        }
        if (const char *e = std::getenv("SB200_KS_ALGO"))
            c->ks_algo = std::atoi(e);
        if (const char *e = std::getenv("SB200_KS_MIN_DIGITS"))
            c->ks_min_digits = static_cast<size_t>(std::atoi(e));
        ksint_init(*c);
        return c;
    }

    // -------------------------------------------------------------------------------------- NTT functors ----
    struct OpBase
    {
        int logn;
        __device__ __forceinline__ bool skip(int) const { return false; }
    };

    // plain slab transform, in place: Evaluator::transform_to_ntt_inplace / transform_from_ntt_inplace
    template <bool INVERSE>
    struct OpSlab
    {
        u64 *data;
        int logn, L;
        const int *pid_tab; // optional prime-id table (BEHZ bases); null = identity
        __device__ __forceinline__ bool skip(int) const { return false; }
        __device__ __forceinline__ int pid(int row) const
        {
            int i = row % L;
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
        __device__ __forceinline__ u64 canon(u64 v, const PrimeDev &P) const
        {
            return INVERSE ? csub(v, P.q) : csub(csub(v, P.q2), P.q);
        }
        __device__ __forceinline__ void store1(int row, int idx, u64 v, const PrimeDev &P) const
        {
            rowp(row)[idx] = canon(v, P);
        }
        __device__ __forceinline__ void store8(int row, int idx0, u64 (&a)[8], const PrimeDev &P) const
        {
            ulonglong2 *p = reinterpret_cast<ulonglong2 *>(rowp(row) + idx0);
#pragma unroll
            for (int j = 0; j < 4; j++)
                p[j] = make_ulonglong2(canon(a[2 * j], P), canon(a[2 * j + 1], P));
        }
    };

    void op_ntt_rows(Context &c, bool inverse, u64 *d, size_t rows, size_t L, const int *pid_tab, cudaStream_t st)
    {
        if (inverse)
        {
            OpSlab<true> op{ d, c.logn, static_cast<int>(L), pid_tab };
            cuda_check(launch_ntt_inv(op, static_cast<int>(rows), c.logn, c.d_primes.get(), st, c.stats), "ntt_inv");
        }
        else
        {
            OpSlab<false> op{ d, c.logn, static_cast<int>(L), pid_tab };
            cuda_check(launch_ntt_fwd(op, static_cast<int>(rows), c.logn, c.d_primes.get(), st, c.stats, "ntt_fwd", -1, c.fast_q && !pid_tab), "ntt_fwd");
        }
    }

    void op_ntt(Context &c, bool inverse, size_t L, size_t size, size_t batch, u64 *d, cudaStream_t st)
    {
        // keep grid.x below 2^31 and launches reasonably sized
        const size_t rows = batch * size * L, max_rows = size_t(1) << 20;
        for (size_t r0 = 0; r0 < rows; r0 += max_rows - (max_rows % L))
        {
            size_t cnt = std::min(rows - r0, max_rows - (max_rows % L));
            op_ntt_rows(c, inverse, d + r0 * c.n, cnt, L, nullptr, st);
        }
    }

    // ------------------------------------------------------------------------------------ CKKS multiply ----
    // (x0 y0, x0 y1 + x1 y0, x1 y1) per prime per coefficient; evaluator.cpp:634-662.
    // FUSED: poly 0,1 go to out (stride 2 polys) and poly 2 to c2 ([b][L][n]) -- the key-switch target.
    // two consecutive coefficients per thread (16-byte accesses); residues are below their modulus (valid ciphertexts), so every
    // 128-bit value reduced here is below 2 q^2 and barrett_wide applies
    template <bool FUSED>
    __global__ void __launch_bounds__(256) ckks_tensor_kernel(const u64 *__restrict__ a, const u64 *__restrict__ b, u64 *out, u64 *c2,
                                                               const PrimeDev *__restrict__ primes, int logn, int L, long long total)
    {
        long long e = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 2; // over batch*L*n
        if (e >= total)
            return;
        const long long poly = static_cast<long long>(L) << logn;
        const long long bidx = e / poly, r = e % poly;
        const int i = static_cast<int>(r >> logn);
        const PrimeDev P = primes[i];
        const u64 *pa = a + bidx * 2 * poly + r, *pb = b + bidx * 2 * poly + r;
        ulonglong2 x0 = *reinterpret_cast<const ulonglong2 *>(pa), x1 = *reinterpret_cast<const ulonglong2 *>(pa + poly);
        ulonglong2 y0 = *reinterpret_cast<const ulonglong2 *>(pb), y1 = *reinterpret_cast<const ulonglong2 *>(pb + poly);
        x0 = make_ulonglong2(canon_in(x0.x, P), canon_in(x0.y, P)), x1 = make_ulonglong2(canon_in(x1.x, P), canon_in(x1.y, P));
        y0 = make_ulonglong2(canon_in(y0.x, P), canon_in(y0.y, P)), y1 = make_ulonglong2(canon_in(y1.x, P), canon_in(y1.y, P));
        auto mid = [&](u64 p0, u64 p1, u64 q0, u64 q1) {
            u64 lo = 0, hi = 0;
            mac128(lo, hi, p0, q1);
            mac128(lo, hi, p1, q0);
            return barrett_wide(lo, hi, P);
        };
        const ulonglong2 d0 = make_ulonglong2(mulmod_wide(x0.x, y0.x, P), mulmod_wide(x0.y, y0.y, P));
        const ulonglong2 d1 = make_ulonglong2(mid(x0.x, x1.x, y0.x, y1.x), mid(x0.y, x1.y, y0.y, y1.y));
        const ulonglong2 d2 = make_ulonglong2(mulmod_wide(x1.x, y1.x, P), mulmod_wide(x1.y, y1.y, P));
        if (FUSED)
        {
            u64 *po = out + bidx * 2 * poly + r;
            *reinterpret_cast<ulonglong2 *>(po) = d0, *reinterpret_cast<ulonglong2 *>(po + poly) = d1;
            *reinterpret_cast<ulonglong2 *>(c2 + bidx * poly + r) = d2;
        }
        else
        {
            u64 *po = out + bidx * 3 * poly + r;
            *reinterpret_cast<ulonglong2 *>(po) = d0, *reinterpret_cast<ulonglong2 *>(po + poly) = d1;
            *reinterpret_cast<ulonglong2 *>(po + 2 * poly) = d2;
        }
    }

    static void launch_tensor(Context &c, bool fused, size_t L, size_t batch, const u64 *a, const u64 *b, u64 *out, u64 *c2,
                              cudaStream_t st)
    {
        long long total = static_cast<long long>(batch) * L * c.n;
        unsigned blocks = static_cast<unsigned>((total / 2 + 255) / 256);
        c.stats.begin("ckks_tensor", 0, 7.0 * 8.0 * total, st); // 4 reads + 3 writes per coefficient (SURVEY 8d)
        if (fused)
            ckks_tensor_kernel<true><<<blocks, 256, 0, st>>>(a, b, out, c2, c.d_primes.get(), c.logn, static_cast<int>(L), total);
        else
            ckks_tensor_kernel<false><<<blocks, 256, 0, st>>>(a, b, out, c2, c.d_primes.get(), c.logn, static_cast<int>(L), total);
        c.stats.end(st);
        cuda_check(cudaGetLastError(), "ckks_tensor_kernel");
    }

    // general-size tensor in an arbitrary base (evaluator.cpp:664-700 / :796-833 NTT-form schemes, :524-560 BFV):
    // out[k] = sum_{i+j=k} x_i * y_j for 0 <= k < s1+s2-1.  x = [B][s1][nb][n] at xa (+ b*xa_bs), y likewise; the prime of
    // row i is pid_tab[i] (or i).  The words are canonicalised on the way in (canon_in: the reference's dyadic products accept any
    // 64-bit representative), so at most min(s1,s2) <= 16 products below q^2 < 2^122 meet in one 128-bit sum.
    __global__ void __launch_bounds__(256) tensor_general_kernel(const u64 *__restrict__ xa, long long xa_bs, const u64 *__restrict__ xb,
                                                                  long long xb_bs, u64 *__restrict__ out, const PrimeDev *__restrict__ primes,
                                                                  const int *__restrict__ pid_tab, int logn, int nb, int s1, int s2,
                                                                  long long total)
    {
        long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over B*nb*n
        if (e >= total)
            return;
        const long long poly = static_cast<long long>(nb) << logn;
        const long long bidx = e / poly, r = e % poly;
        const int i = static_cast<int>(r >> logn);
        const PrimeDev P = primes[pid_tab ? pid_tab[i] : i];
        const u64 *px = xa + bidx * xa_bs + r, *py = xb + bidx * xb_bs + r;
        u64 *po = out + bidx * (s1 + s2 - 1) * poly + r;
        for (int k = 0; k < s1 + s2 - 1; k++)
        {
            const int i0 = k - (s2 - 1) > 0 ? k - (s2 - 1) : 0, i1 = k < s1 - 1 ? k : s1 - 1;
            u64 lo = 0, hi = 0;
            for (int a = i0; a <= i1; a++)
                mac128(lo, hi, canon_in(px[a * poly], P), canon_in(py[(k - a) * poly], P));
            po[k * poly] = barrett128(lo, hi, P.q, P.ratio_lo, P.ratio_hi);
        }
    }

    void launch_tensor_general(Context &c, const u64 *xa, long long xa_bs, const u64 *xb, long long xb_bs, u64 *out, const int *pid_tab,
                               size_t nb, size_t s1, size_t s2, size_t B, cudaStream_t st)
    {
        const long long total = static_cast<long long>(B) * nb * c.n;
        c.stats.begin("tensor_general", 0, 8.0 * total * (2.0 * (s1 + s2) - 1.0), st);
        tensor_general_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(
            xa, xa_bs, xb, xb_bs, out, c.d_primes.get(), pid_tab, c.logn, static_cast<int>(nb), static_cast<int>(s1), static_cast<int>(s2), total);
        c.stats.end(st);
        cuda_check(cudaGetLastError(), "tensor_general_kernel");
    }

    void check_sizes(size_t s1, size_t s2)
    {
        // Ciphertext sizes are bounded by SEAL_CIPHERTEXT_SIZE_MAX = 16 (defines.h), the product by the same bound (evaluator.cpp:588-596)
        if (s1 < 2 || s2 < 2 || s1 > 16 || s2 > 16 || s1 + s2 - 1 > 16)
            throw std::invalid_argument("invalid ciphertext sizes");
    }

    void op_ckks_multiply(Context &c, size_t L, size_t s1, size_t s2, size_t batch, const u64 *a, const u64 *b, u64 *out, cudaStream_t st)
    {
        if (s1 == 2 && s2 == 2)
            return op_ckks_multiply(c, L, batch, a, b, out, st);
        check_sizes(s1, s2);
        const size_t poly = L * c.n, step = std::max<size_t>(1, (size_t(1) << 31) / poly);
        for (size_t b0 = 0; b0 < batch; b0 += step)
        {
            const size_t nb = std::min(step, batch - b0);
            launch_tensor_general(c, a + b0 * s1 * poly, static_cast<long long>(s1 * poly), b + b0 * s2 * poly, static_cast<long long>(s2 * poly),
                                  out + b0 * (s1 + s2 - 1) * poly, nullptr, L, s1, s2, nb, st);
        }
    }

    // squaring (ckks_square / bgv_square, evaluator.cpp:1022-1142): (x0^2, 2 x0 x1, x1^2) -- three products and two input rows per
    // coefficient instead of four and four; the kernel is bound by HBM (5 rows moved instead of 7)
    __global__ void __launch_bounds__(256) ckks_square_kernel(const u64 *__restrict__ a, u64 *out, const PrimeDev *__restrict__ primes, int logn,
                                                               int L, long long total)
    {
        long long e = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 2; // over batch*L*n
        if (e >= total)
            return;
        const long long poly = static_cast<long long>(L) << logn;
        const long long bidx = e / poly, r = e % poly;
        const PrimeDev P = primes[static_cast<int>(r >> logn)];
        const u64 *pa = a + bidx * 2 * poly + r;
        ulonglong2 x0 = *reinterpret_cast<const ulonglong2 *>(pa), x1 = *reinterpret_cast<const ulonglong2 *>(pa + poly);
        x0 = make_ulonglong2(canon_in(x0.x, P), canon_in(x0.y, P)), x1 = make_ulonglong2(canon_in(x1.x, P), canon_in(x1.y, P));
        auto twice = [&](u64 p0, u64 p1) {
            const u64 m = mulmod_wide(p0, p1, P);
            return csub(m + m, P.q);
        };
        u64 *po = out + bidx * 3 * poly + r;
        *reinterpret_cast<ulonglong2 *>(po) = make_ulonglong2(mulmod_wide(x0.x, x0.x, P), mulmod_wide(x0.y, x0.y, P));
        *reinterpret_cast<ulonglong2 *>(po + poly) = make_ulonglong2(twice(x0.x, x1.x), twice(x0.y, x1.y));
        *reinterpret_cast<ulonglong2 *>(po + 2 * poly) = make_ulonglong2(mulmod_wide(x1.x, x1.x, P), mulmod_wide(x1.y, x1.y, P));
    }

    void op_ckks_multiply(Context &c, size_t L, size_t batch, const u64 *a, const u64 *b, u64 *out3, cudaStream_t st)
    {
        const size_t step = std::max<size_t>(1, (size_t(1) << 31) / (L * c.n));
        if (a == b)
        {
            for (size_t b0 = 0; b0 < batch; b0 += step)
            {
                const size_t nb = std::min(step, batch - b0);
                const long long total = static_cast<long long>(nb) * L * c.n;
                c.stats.begin("ckks_square", 0, 5.0 * 8.0 * total, st); // 2 reads + 3 writes per coefficient
                ckks_square_kernel<<<static_cast<unsigned>((total / 2 + 255) / 256), 256, 0, st>>>(a + b0 * 2 * L * c.n, out3 + b0 * 3 * L * c.n,
                                                                                                     c.d_primes.get(), c.logn, static_cast<int>(L), total);
                c.stats.end(st);
                cuda_check(cudaGetLastError(), "ckks_square_kernel");
            }
            return;
        }
        for (size_t b0 = 0; b0 < batch; b0 += step)
        {
            size_t nb = std::min(step, batch - b0);
            launch_tensor(c, false, L, nb, a + b0 * 2 * L * c.n, b + b0 * 2 * L * c.n, out3 + b0 * 3 * L * c.n, nullptr, st);
        }
    }

    // ---- add / sub / negate (evaluator.cpp:130-350: add_poly_coeffmod / sub_poly_coeffmod / negate_poly_coeffmod) ---------
    // MODE 0: a + b, 1: a - b, 2: -a; rows of n coefficients, prime of a row = row % L
    template <int MODE>
    __global__ void __launch_bounds__(256) linear_kernel(const ulonglong2 *__restrict__ a, const ulonglong2 *__restrict__ b, ulonglong2 *out,
                                                          const PrimeDev *__restrict__ primes, int logn, int L, long long total2)
    {
        long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over pairs of coefficients
        if (e >= total2)
            return;
        const u64 q = primes[static_cast<int>(((e * 2) >> logn) % L)].q;
        ulonglong2 x = a[e], y = MODE == 2 ? make_ulonglong2(0, 0) : b[e], r;
        if (MODE == 0)
            r = make_ulonglong2(csub(x.x + y.x, q), csub(x.y + y.y, q));
        else if (MODE == 1)
            r = make_ulonglong2(sub_borrow(x.x, y.x, q), sub_borrow(x.y, y.y, q));
        else
            r = make_ulonglong2(x.x ? q - x.x : 0, x.y ? q - x.y : 0);
        out[e] = r;
    }

    void op_linear(Context &c, int mode, size_t L, size_t size, size_t batch, const u64 *a, const u64 *b, u64 *out, cudaStream_t st)
    {
        if (c.n < 2 || size < 1)
            throw std::invalid_argument("encrypted is not valid for encryption parameters");
        const size_t per = size * L * c.n, step = std::max<size_t>(1, (size_t(1) << 32) / per);
        for (size_t b0 = 0; b0 < batch; b0 += step)
        {
            const size_t nb = std::min(step, batch - b0);
            const long long total2 = static_cast<long long>(nb * per / 2);
            const unsigned blocks = static_cast<unsigned>((total2 + 255) / 256);
            auto pa = reinterpret_cast<const ulonglong2 *>(a + b0 * per);
            auto pb = reinterpret_cast<const ulonglong2 *>(b ? b + b0 * per : nullptr);
            auto po = reinterpret_cast<ulonglong2 *>(out + b0 * per);
            c.stats.begin(mode == 0 ? "add" : mode == 1 ? "sub" : "negate", 0, (mode == 2 ? 16.0 : 24.0) * total2 * 2, st);
            if (mode == 0)
                linear_kernel<0><<<blocks, 256, 0, st>>>(pa, pb, po, c.d_primes.get(), c.logn, static_cast<int>(L), total2);
            else if (mode == 1)
                linear_kernel<1><<<blocks, 256, 0, st>>>(pa, pb, po, c.d_primes.get(), c.logn, static_cast<int>(L), total2);
            else
                linear_kernel<2><<<blocks, 256, 0, st>>>(pa, pb, po, c.d_primes.get(), c.logn, static_cast<int>(L), total2);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "linear_kernel");
        }
    }

    // ---- add_many: a left fold of add_inplace / sub_inplace steps in one pass (evaluator.cpp:155-262, :263-350) ------------
    // Operand j is [B][stride_j][L][n] with size_j polynomials present.  Every output word gets the word operations the reference's
    // chain of add_inplace / sub_inplace performs on it, in the chain's order, in registers: acc = x_0, then per step j >= 1
    //   scaled (BGV balancing, multiply_poly_scalar_coeffmod over the present polynomials): acc = acc * e1_j, y = x_j * e2_j (Shoup);
    //   add: acc = csub(acc + y, q);  sub: acc = sub_borrow(acc, y, q) (acc - y, plus q on a borrow);
    //   polynomial absent from every earlier operand: acc = y (add, set_poly_array) or -y (sub, negate_poly_coeffmod).
    // Absence is tracked, never stood in for by zero: csub(0 + y, q) != y for a word y >= q.
    struct FoldLaunch
    {
        const ulonglong2 *x[kFoldMaxOperands];
        int size[kFoldMaxOperands];   // polynomials present in operand j
        int stride[kFoldMaxOperands]; // polynomials per ciphertext in operand j's slab
        int mode[kFoldMaxOperands];   // step j (j >= 1): bit 0 sub, bit 1 scaled; the scalars of step j at tab[(j - 1) L + i]
        int count, polys, out_stride; // operands; polynomials written; polynomials per ciphertext of the output slab
    };

    __global__ void __launch_bounds__(256) fold_kernel(const __grid_constant__ FoldLaunch f, const Tw *__restrict__ tab, ulonglong2 *out,
                                                       const PrimeDev *__restrict__ primes, int logn, int L, long long total2)
    {
        const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over the batch's pairs of one polynomial
        if (e >= total2)
            return;
        const long long half = static_cast<long long>(L) << (logn - 1);
        const long long b = e / half, r = e - b * half;
        const int i = static_cast<int>((r * 2) >> logn);
        const u64 q = primes[i].q;
        for (int p = 0; p < f.polys; p++)
        {
            ulonglong2 acc = make_ulonglong2(0, 0);
            bool have = false;
            for (int j = 0; j < f.count; j++)
            {
                const int m = j ? f.mode[j] : 0;
                if (m & 2)
                {
                    const Tw e1 = tab[(2 * (j - 1)) * L + i], e2 = tab[(2 * (j - 1) + 1) * L + i];
                    if (have)
                        acc = make_ulonglong2(mul_shoup(acc.x, e1, q), mul_shoup(acc.y, e1, q));
                    if (p < f.size[j])
                    {
                        const ulonglong2 v = f.x[j][(b * f.stride[j] + p) * half + r];
                        const ulonglong2 y = make_ulonglong2(mul_shoup(v.x, e2, q), mul_shoup(v.y, e2, q));
                        acc = !have ? ((m & 1) ? make_ulonglong2(y.x ? q - y.x : 0, y.y ? q - y.y : 0) : y)
                              : (m & 1) ? make_ulonglong2(sub_borrow(acc.x, y.x, q), sub_borrow(acc.y, y.y, q))
                                        : make_ulonglong2(csub(acc.x + y.x, q), csub(acc.y + y.y, q));
                        have = true;
                    }
                }
                else if (p < f.size[j])
                {
                    const ulonglong2 y = f.x[j][(b * f.stride[j] + p) * half + r];
                    acc = !have ? ((m & 1) ? make_ulonglong2(y.x ? q - y.x : 0, y.y ? q - y.y : 0) : y)
                          : (m & 1) ? make_ulonglong2(sub_borrow(acc.x, y.x, q), sub_borrow(acc.y, y.y, q))
                                    : make_ulonglong2(csub(acc.x + y.x, q), csub(acc.y + y.y, q));
                    have = true;
                }
            }
            out[(b * f.out_stride + p) * half + r] = acc;
        }
    }

    void op_add_many(Context &c, size_t L, size_t batch, size_t count, const size_t *sizes, const u64 *const *ops, const int *modes,
                     const u64 *factors, u64 *out, cudaStream_t st)
    {
        size_t out_size = 0;
        bool scaled = false;
        for (size_t j = 0; j < count; j++)
        {
            out_size = std::max(out_size, sizes[j]);
            scaled |= j && (modes[j - 1] & 2);
        }
        // (e1_j, e2_j) mod q_i with their Shoup quotients: tab[(2 (j - 1) + {0, 1}) L + i]
        const Tw *d_tab = nullptr;
        if (scaled)
        {
            std::vector<Tw> tab(2 * (count - 1) * L);
            for (size_t j = 1; j < count; j++)
                if (modes[j - 1] & 2)
                    for (int h = 0; h < 2; h++)
                        for (size_t i = 0; i < L; i++)
                        {
                            const u64 v = factors[2 * (j - 1) + h] % c.q[i];
                            tab[(2 * (j - 1) + h) * L + i] = Tw{ v, sbh::shoup(v, c.q[i]) };
                        }
            auto *d = static_cast<Tw *>(c.ensure_scratch(tab.size() * sizeof(Tw)));
            cuda_check(cudaMemcpyAsync(d, tab.data(), tab.size() * sizeof(Tw), cudaMemcpyHostToDevice, st), "upload scalars");
            d_tab = d;
        }
        const long long half = static_cast<long long>(L * c.n / 2), total2 = static_cast<long long>(batch) * half;
        const unsigned blocks = static_cast<unsigned>((total2 + 255) / 256);
        // operand 0 of every launch after the first is the partial result in out (its present polynomials so far); the words do not
        // depend on where the fold is cut, since the accumulator of a word is that word
        size_t j0 = 0, acc_size = 0;
        while (j0 < count)
        {
            FoldLaunch f{};
            int k = 0;
            double words = 0;
            if (j0)
            {
                f.x[0] = reinterpret_cast<const ulonglong2 *>(out), f.size[0] = static_cast<int>(acc_size), f.stride[0] = static_cast<int>(out_size);
                words += static_cast<double>(acc_size);
                k = 1;
            }
            size_t polys = acc_size;
            const size_t first = j0;
            for (; k < kFoldMaxOperands && j0 < count; k++, j0++)
            {
                f.x[k] = reinterpret_cast<const ulonglong2 *>(ops[j0]);
                f.size[k] = f.stride[k] = static_cast<int>(sizes[j0]);
                // the scalars stay indexed by the step's place in the whole fold: shift the table so that launch slot k finds them
                f.mode[k] = j0 ? modes[j0 - 1] : 0;
                polys = std::max(polys, sizes[j0]);
                words += static_cast<double>(sizes[j0]);
            }
            f.count = k, f.polys = static_cast<int>(polys), f.out_stride = static_cast<int>(out_size);
            // slot k of this launch holds step (first - (first ? 1 : 0)) + k of the fold; its scalars start at that step's entry
            const size_t step0 = first ? first - 1 : 0;
            const Tw *t = d_tab ? d_tab + 2 * step0 * L : nullptr;
            c.stats.begin("add_many", 0, 8.0 * (words + static_cast<double>(polys)) * static_cast<double>(L * c.n) * static_cast<double>(batch), st);
            fold_kernel<<<blocks, 256, 0, st>>>(f, t, reinterpret_cast<ulonglong2 *>(out), c.d_primes.get(), c.logn, static_cast<int>(L), total2);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "fold_kernel");
            acc_size = polys;
        }
    }

    // ---- multiply_plain, NTT x NTT (evaluator.cpp:2157-2195: dyadic_product_coeffmod of every polynomial with the plaintext) ----
    // ct [B][size][L][n], plain [B][L][n] (one NTT-form plaintext per ciphertext, at the ciphertext's level)
    __global__ void __launch_bounds__(256) plain_mul_kernel(const ulonglong2 *__restrict__ a, const ulonglong2 *__restrict__ plain,
                                                             ulonglong2 *out, const PrimeDev *__restrict__ primes, int logn, int L, int size,
                                                             long long total2)
    {
        long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over pairs of coefficients
        if (e >= total2)
            return;
        const long long row = (e * 2) >> logn;
        const int i = static_cast<int>(row % L);
        const long long b = row / (static_cast<long long>(size) * L);
        const long long pe = (((b * L + i) << logn) >> 1) + (e & ((1ll << (logn - 1)) - 1));
        const PrimeDev &P = primes[i];
        const ulonglong2 x = a[e], y = plain[pe];
        out[e] = make_ulonglong2(mulmod_wide(canon_in(x.x, P), canon_in(y.x, P), P), mulmod_wide(canon_in(x.y, P), canon_in(y.y, P), P));
    }

    // One plaintext [L][n] for the whole batch.  A thread owns one pair of plaintext words and keeps them in registers while it
    // walks the rows of a group of G ciphertexts: MODE 0 multiplies every polynomial (dyadic_product_coeffmod, operands reduced on
    // the way in as plain_mul_kernel does), MODE 1 / 2 add to / subtract from c_0 only (add_poly_coeffmod / sub_poly_coeffmod, as
    // add_c0_kernel).  blockIdx.x is the ciphertext group, so the CTAs that read one plaintext slice run together and the slice
    // crosses HBM once per launch.  (The per-ciphertext kernels with a plaintext stride of 0 re-read the plaintext from HBM once L2
    // no longer holds it: at n = 65536 with 31 primes, 1.3x / 1.6x this kernel's time for multiply_plain / add_plain; DESIGN 7b.)
    template <int MODE>
    __global__ void __launch_bounds__(256) shared_plain_kernel(const ulonglong2 *__restrict__ a, const ulonglong2 *__restrict__ plain, ulonglong2 *out,
                                                                const PrimeDev *__restrict__ primes, int logn, int L, int size, int batch, int G)
    {
        const long long half = static_cast<long long>(L) << (logn - 1); // pairs of one polynomial
        const int b1 = min(batch, static_cast<int>(blockIdx.x + 1) * G), polys = MODE == 0 ? size : 1;
        // grid.y is capped at 65535 blocks and L n / 512 reaches 65536 at n = 131072 with 256 primes: the y blocks stride over the pairs
        for (long long p = static_cast<long long>(blockIdx.y) * blockDim.x + threadIdx.x; p < half; p += static_cast<long long>(gridDim.y) * blockDim.x)
        {
            const PrimeDev &P = primes[static_cast<int>(p >> (logn - 1))];
            ulonglong2 y = plain[p];
            if (MODE == 0)
                y = make_ulonglong2(canon_in(y.x, P), canon_in(y.y, P));
            for (int b = blockIdx.x * G; b < b1; b++)
                for (int s = 0; s < polys; s++)
                {
                    const long long e = (static_cast<long long>(b) * size + s) * half + p;
                    const ulonglong2 x = a[e];
                    if (MODE == 0)
                        out[e] = make_ulonglong2(mulmod_wide(canon_in(x.x, P), y.x, P), mulmod_wide(canon_in(x.y, P), y.y, P));
                    else if (MODE == 1)
                        out[e] = make_ulonglong2(csub(x.x + y.x, P.q), csub(x.y + y.y, P.q));
                    else
                        out[e] = make_ulonglong2(sub_borrow(x.x, y.x, P.q), sub_borrow(x.y, y.y, P.q));
                }
        }
    }

    static void launch_shared_plain(Context &c, int mode, const char *name, size_t L, size_t size, size_t batch, const u64 *a, const u64 *plain,
                                    u64 *out, cudaStream_t st)
    {
        constexpr int G = 8;
        const size_t half = L * c.n / 2, polys = mode == 0 ? size : 1;
        const dim3 grid(static_cast<unsigned>((batch + G - 1) / G), static_cast<unsigned>(std::min<size_t>((half + 255) / 256, 65535)));
        auto pa = reinterpret_cast<const ulonglong2 *>(a);
        auto pp = reinterpret_cast<const ulonglong2 *>(plain);
        auto po = reinterpret_cast<ulonglong2 *>(out);
        const int l = static_cast<int>(L), sz = static_cast<int>(size), nb = static_cast<int>(batch);
        c.stats.begin(name, 0, 8.0 * (2.0 * batch * polys + 1.0) * L * c.n, st);
        if (mode == 0)
            shared_plain_kernel<0><<<grid, 256, 0, st>>>(pa, pp, po, c.d_primes.get(), c.logn, l, sz, nb, G);
        else if (mode == 1)
            shared_plain_kernel<1><<<grid, 256, 0, st>>>(pa, pp, po, c.d_primes.get(), c.logn, l, sz, nb, G);
        else
            shared_plain_kernel<2><<<grid, 256, 0, st>>>(pa, pp, po, c.d_primes.get(), c.logn, l, sz, nb, G);
        c.stats.end(st);
        cuda_check(cudaGetLastError(), "shared_plain_kernel");
    }

    void op_multiply_plain(Context &c, size_t L, size_t size, size_t batch, bool shared, const u64 *a, const u64 *plain, u64 *out,
                           cudaStream_t st)
    {
        if (c.n < 2 || size < 1)
            throw std::invalid_argument("encrypted is not valid for encryption parameters");
        if (shared)
        {
            const size_t step = std::max<size_t>(1, (size_t(1) << 30) / (size * L * c.n));
            for (size_t b0 = 0; b0 < batch; b0 += step)
                launch_shared_plain(c, 0, "multiply_plain", L, size, std::min(step, batch - b0), a + b0 * size * L * c.n, plain,
                                    out + b0 * size * L * c.n, st);
            return;
        }
        const size_t per = size * L * c.n, step = std::max<size_t>(1, (size_t(1) << 32) / per);
        for (size_t b0 = 0; b0 < batch; b0 += step)
        {
            const size_t nb = std::min(step, batch - b0);
            const long long total2 = static_cast<long long>(nb * per / 2);
            const unsigned blocks = static_cast<unsigned>((total2 + 255) / 256);
            c.stats.begin("multiply_plain", 0, 8.0 * (2.0 * nb * per + nb * L * c.n), st);
            plain_mul_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<const ulonglong2 *>(a + b0 * per),
                                                     reinterpret_cast<const ulonglong2 *>(plain + b0 * L * c.n),
                                                     reinterpret_cast<ulonglong2 *>(out + b0 * per), c.d_primes.get(), c.logn, static_cast<int>(L),
                                                     static_cast<int>(size), total2);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "plain_mul_kernel");
        }
    }

    // ---- coefficient-form plaintexts (BFV / BGV): lift, transform, multiply_plain, add_plain / sub_plain ----------------
    const Context::PlainLevel &plain_level(Context &c, size_t L)
    {
        if (c.scheme == 2 || c.t < 2)
            throw std::invalid_argument("unsupported operation for scheme type");
        if (!c.d_t_mod_q)
        {
            std::vector<u64> tm(c.k);
            for (size_t i = 0; i < c.k; i++)
                tm[i] = c.t % c.q[i];
            c.d_t_mod_q = upload<u64>(c, tm);
            const unsigned __int128 ratio = ~static_cast<unsigned __int128>(0) / c.t; // floor((2^128 - 1) / t): at most 1 below floor(2^128 / t)
            c.t_ratio_lo = static_cast<u64>(ratio), c.t_ratio_hi = static_cast<u64>(ratio >> 64);
        }
        auto it = c.plain_levels.find(L);
        if (it != c.plain_levels.end())
            return it->second;
        Context::PlainLevel pl;
        unsigned __int128 acc = 1;
        for (size_t i = 0; i < L; i++)
            acc = acc * (c.q[i] % c.t) % c.t;
        pl.q_mod_t = static_cast<u64>(acc);
        // floor(q / t) = (q - (q mod t)) / t, and q = 0 mod q_i: floor(q / t) mod q_i = -(q mod t) * t^-1 mod q_i
        std::vector<Tw> delta(L);
        for (size_t i = 0; i < L; i++)
        {
            u64 inv = 0;
            if (!sbh::invmod(c.t % c.q[i], c.q[i], inv))
                throw std::logic_error("plain_modulus and coeff_modulus are not coprime");
            const u64 r = pl.q_mod_t % c.q[i];
            const u64 v = static_cast<u64>(static_cast<unsigned __int128>(r ? c.q[i] - r : 0) * inv % c.q[i]);
            delta[i] = Tw{ v, sbh::shoup(v, c.q[i]) };
        }
        pl.d_delta = upload<Tw>(c, delta);
        return c.plain_levels.emplace(L, std::move(pl)).first->second;
    }

    // per-ciphertext BGV correction factors -> device (behind the scratch words of this call); nullptr stays nullptr
    static const u64 *upload_cf(Context &c, const u64 *h_cf, size_t B, u64 *slot, cudaStream_t st)
    {
        if (!h_cf)
            return nullptr;
        cuda_check(cudaMemcpyAsync(slot, h_cf, B * sizeof(u64), cudaMemcpyHostToDevice, st), "upload correction factors");
        (void)c;
        return slot;
    }

    // forward transform of lifted plaintexts: rows (b, i) -> out[b][i][:]; cf (optional): plaintext times cf[b] mod t first
    struct OpPlainLift
    {
        const u64 *plain; // [B][n]
        const u64 *cf;    // [B] or nullptr
        const u64 *t_mod_q;
        u64 *out;         // [B][L][n]
        u64 t, t_ratio_lo, t_ratio_hi;
        int logn, L;
        __device__ __forceinline__ bool skip(int) const { return false; }
        __device__ __forceinline__ int pid(int row) const { return row % L; }
        __device__ __forceinline__ const u64 *direct(int, const PrimeDev &) const { return nullptr; }
        __device__ __forceinline__ u64 load1(int row, int idx, const PrimeDev &P) const
        {
            const int b = row / L;
            u64 v = plain[(static_cast<long long>(b) << logn) + idx];
            if (cf)
            {
                const u64 f = cf[b];
                v = barrett128(v * f, __umul64hi(v, f), t, t_ratio_lo, t_ratio_hi);
                v = csub(v, t); // the ratio may sit one below floor(2^128 / t)
            }
            return plain_lift(v, t, t_mod_q[row % L], P);
        }
        __device__ __forceinline__ void load8(int, int, u64 (&)[8], const PrimeDev &) const {}
        __device__ __forceinline__ u64 *mid(int row) const { return out + (static_cast<long long>(row) << logn); }
        __device__ __forceinline__ void store1(int row, int idx, u64 v, const PrimeDev &P) const { mid(row)[idx] = csub(csub(v, P.q2), P.q); }
        __device__ __forceinline__ void store8(int row, int idx0, u64 (&v)[8], const PrimeDev &P) const
        {
#pragma unroll
            for (int j = 0; j < 8; j++)
                store1(row, idx0 + j, v[j], P);
        }
    };

    static void plain_to_ntt_dev(Context &c, size_t L, size_t B, const u64 *plain, const u64 *d_cf, u64 *out, cudaStream_t st)
    {
        plain_level(c, L);
        OpPlainLift op{ plain, d_cf, c.d_t_mod_q.get(), out, c.t, c.t_ratio_lo, c.t_ratio_hi, c.logn, static_cast<int>(L) };
        cuda_check(launch_ntt_fwd(op, static_cast<int>(B * L), c.logn, c.d_primes.get(), st, c.stats, "plain_lift_ntt", -1, c.fast_q), "plain lift ntt");
    }

    void op_plain_to_ntt(Context &c, size_t L, size_t batch, const u64 *plain, const u64 *h_cf, u64 *out, cudaStream_t st)
    {
        const size_t step = std::max<size_t>(1, (size_t(1) << 30) / (L * c.n));
        for (size_t b0 = 0; b0 < batch; b0 += step)
        {
            const size_t B = std::min(step, batch - b0);
            const u64 *d_cf = nullptr;
            if (h_cf)
                d_cf = upload_cf(c, h_cf + b0, B, static_cast<u64 *>(c.ensure_scratch(B * sizeof(u64))), st);
            plain_to_ntt_dev(c, L, B, plain + b0 * c.n, d_cf, out + b0 * L * c.n, st);
        }
    }

    void op_multiply_plain_coeff(Context &c, size_t L, size_t size, size_t batch, bool shared, bool ct_ntt, const u64 *ct, const u64 *plain,
                                 u64 *out, cudaStream_t st)
    {
        if (size < 1)
            throw std::invalid_argument("encrypted is not valid for encryption parameters");
        const size_t per = size * L * c.n;
        // a shared plaintext is lifted and transformed once per call (L n scratch words); per-ciphertext plaintexts per chunk
        size_t chunk = shared ? batch : std::min(batch, std::max<size_t>(1, c.scratch_budget / (L * c.n * sizeof(u64))));
        chunk = std::min<size_t>(chunk, std::max<size_t>(1, (size_t(1) << 30) / per));
        u64 *T = nullptr;
        if (shared)
        {
            T = static_cast<u64 *>(c.ensure_scratch(L * c.n * sizeof(u64)));
            plain_to_ntt_dev(c, L, 1, plain, nullptr, T, st);
        }
        for (size_t b0 = 0; b0 < batch; b0 += chunk)
        {
            const size_t B = std::min(chunk, batch - b0);
            if (!shared)
            {
                T = static_cast<u64 *>(c.ensure_scratch(B * L * c.n * sizeof(u64)));
                plain_to_ntt_dev(c, L, B, plain + b0 * c.n, nullptr, T, st);
            }
            const u64 *in = ct + b0 * per;
            u64 *o = out + b0 * per;
            if (ct_ntt)
            {
                op_multiply_plain(c, L, size, B, shared, in, T, o, st); // evaluator.cpp:1999-2004
                continue;
            }
            // multiply_plain_normal (evaluator.cpp:2130-2143): ciphertext to NTT form, dyadic product, back
            if (o != in)
                cuda_check(cudaMemcpyAsync(o, in, B * per * sizeof(u64), cudaMemcpyDeviceToDevice, st), "copy");
            op_ntt(c, false, L, size, B, o, st);
            op_multiply_plain(c, L, size, B, shared, o, T, o, st);
            op_ntt(c, true, L, size, B, o, st);
        }
    }

    // BFV: c_0 +/- round(q * m / t) (multiply_add / multiply_sub_plain_with_scaling_variant, util/scalingvariant.cpp:70-160)
    // plain [B][n] (plain_bs = n) or one [n] for the whole batch (plain_bs = 0)
    __global__ void __launch_bounds__(256) bfv_add_plain_kernel(const u64 *__restrict__ plain, long long plain_bs, u64 *ct, long long ct_bs,
                                                                 const Tw *__restrict__ delta,
                                                                 const PrimeDev *__restrict__ primes, u64 t, u64 t_ratio_lo, u64 t_ratio_hi,
                                                                 u64 q_mod_t, int logn, int L, int subtract, long long total)
    {
        long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over B*n
        if (e >= total)
            return;
        const long long b = e >> logn;
        const int idx = static_cast<int>(e & ((1 << logn) - 1));
        const u64 m = plain[b * plain_bs + idx];
        const u64 fix = bfv_plain_fix(m, t, t_ratio_lo, t_ratio_hi, q_mod_t);
        u64 *dst = ct + b * ct_bs + idx;
        for (int i = 0; i < L; i++)
        {
            const PrimeDev P = primes[i];
            const u64 scaled = bfv_plain_scaled(m, fix, t, delta[i], P);
            const u64 x = dst[static_cast<long long>(i) << logn];
            dst[static_cast<long long>(i) << logn] = subtract ? sub_borrow(x, scaled, P.q) : csub(x + scaled, P.q);
        }
    }

    // c_0 +/- T, T = [B][L][n] NTT-form plaintexts: BGV's transformed plaintexts (evaluator.cpp:1838-1849), CKKS's own
    // (add_poly_coeffmod / sub_poly_coeffmod, :1831-1836, :1939-1944)
    __global__ void __launch_bounds__(256) add_c0_kernel(const u64 *__restrict__ T, u64 *ct, long long ct_bs, const PrimeDev *__restrict__ primes,
                                                          int logn, int L, int subtract, long long total)
    {
        long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over B*L*n
        if (e >= total)
            return;
        const long long poly = static_cast<long long>(L) << logn, b = e / poly, r = e % poly;
        const u64 q = primes[static_cast<int>(r >> logn)].q;
        u64 *p = ct + b * ct_bs + r;
        const u64 x = *p, y = T[e];
        *p = subtract ? sub_borrow(x, y, q) : csub(x + y, q);
    }

    static void launch_add_c0(Context &c, const char *name, size_t L, size_t size, size_t B, bool shared, bool subtract, const u64 *T, u64 *o,
                              cudaStream_t st)
    {
        if (shared)
            return launch_shared_plain(c, subtract ? 2 : 1, name, L, size, B, o, T, o, st);
        const long long total = static_cast<long long>(B * L * c.n);
        c.stats.begin(name, 0, 24.0 * total, st);
        add_c0_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(T, o, static_cast<long long>(size * L * c.n), c.d_primes.get(),
                                                                                  c.logn, static_cast<int>(L), subtract ? 1 : 0, total);
        c.stats.end(st);
        cuda_check(cudaGetLastError(), "add_c0_kernel");
    }

    void op_add_plain_coeff(Context &c, size_t L, size_t size, size_t batch, bool shared, bool subtract, const u64 *ct, const u64 *plain,
                            const u64 *h_cf, u64 *out, cudaStream_t st)
    {
        if (size < 1)
            throw std::invalid_argument("encrypted is not valid for encryption parameters");
        const Context::PlainLevel &pl = plain_level(c, L);
        const size_t per = size * L * c.n;
        if (out != ct)
            cuda_check(cudaMemcpyAsync(out, ct, batch * per * sizeof(u64), cudaMemcpyDeviceToDevice, st), "copy");
        size_t chunk = shared ? batch : std::min(batch, std::max<size_t>(1, c.scratch_budget / ((L * c.n + 1) * sizeof(u64))));
        chunk = std::min<size_t>(chunk, std::max<size_t>(1, (size_t(1) << 30) / (L * c.n)));
        u64 *T = nullptr;
        if (shared && c.scheme != 1) // BGV: NTT(lift(m cf mod t)) of the one plaintext, once per call
        {
            T = static_cast<u64 *>(c.ensure_scratch((L * c.n + 1) * sizeof(u64)));
            plain_to_ntt_dev(c, L, 1, plain, upload_cf(c, h_cf, 1, T + L * c.n, st), T, st);
        }
        for (size_t b0 = 0; b0 < batch; b0 += chunk)
        {
            const size_t B = std::min(chunk, batch - b0);
            u64 *o = out + b0 * per;
            if (c.scheme == 1)
            {
                const long long total = static_cast<long long>(B * c.n);
                c.stats.begin("bfv_add_plain", 0, 8.0 * ((shared ? c.n : total) + 2.0 * L * total), st);
                bfv_add_plain_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(
                    plain + (shared ? 0 : b0 * c.n), shared ? 0 : static_cast<long long>(c.n), o, static_cast<long long>(per), pl.d_delta.get(),
                    c.d_primes.get(), c.t, c.t_ratio_lo, c.t_ratio_hi, pl.q_mod_t, c.logn, static_cast<int>(L), subtract ? 1 : 0, total);
                c.stats.end(st);
                cuda_check(cudaGetLastError(), "bfv_add_plain_kernel");
                continue;
            }
            if (!shared)
            {
                T = static_cast<u64 *>(c.ensure_scratch((B * L * c.n + B) * sizeof(u64)));
                const u64 *d_cf = upload_cf(c, h_cf ? h_cf + b0 : nullptr, B, T + B * L * c.n, st);
                plain_to_ntt_dev(c, L, B, plain + b0 * c.n, d_cf, T, st);
            }
            launch_add_c0(c, "bgv_add_plain", L, size, B, shared, subtract, T, o, st);
        }
    }

    void op_add_plain_ntt(Context &c, size_t L, size_t size, size_t batch, bool shared, bool subtract, const u64 *ct, const u64 *plain, u64 *out,
                          cudaStream_t st)
    {
        if (c.scheme == 1) // evaluator.cpp:1774-1782, :1882-1890
            throw std::invalid_argument("BFV plain cannot be in NTT form");
        if (c.scheme == 3) // :1798-1806, :1906-1914
            throw std::invalid_argument("BGV plain cannot be in NTT form");
        if (c.n < 2 || size < 1)
            throw std::invalid_argument("encrypted is not valid for encryption parameters");
        const size_t per = size * L * c.n;
        if (out != ct)
            cuda_check(cudaMemcpyAsync(out, ct, batch * per * sizeof(u64), cudaMemcpyDeviceToDevice, st), "copy");
        const size_t chunk = std::max<size_t>(1, (size_t(1) << 30) / (L * c.n));
        for (size_t b0 = 0; b0 < batch; b0 += chunk)
        {
            const size_t B = std::min(chunk, batch - b0);
            launch_add_c0(c, subtract ? "ckks_sub_plain" : "ckks_add_plain", L, size, B, shared, subtract, plain + (shared ? 0 : b0 * L * c.n),
                          out + b0 * per, st);
        }
    }

    // ---- BatchEncoder (batchencoder.cpp:84-330): the slot permutation rides in the load (encode) or the store (decode) of a
    //      transform modulo t; rows = plaintexts
    struct OpBatchEncode
    {
        const u64 *values;        // [B][n] matrix slots
        const uint32_t *inv_map;  // coefficient index -> slot
        u64 *plain;               // [B][n]
        int logn, pid_t;
        __device__ __forceinline__ bool skip(int) const { return false; }
        __device__ __forceinline__ int pid(int) const { return pid_t; }
        __device__ __forceinline__ const u64 *direct(int, const PrimeDev &) const { return nullptr; }
        __device__ __forceinline__ u64 load1(int row, int idx, const PrimeDev &) const
        {
            return values[(static_cast<long long>(row) << logn) + inv_map[idx]];
        }
        __device__ __forceinline__ void load8(int row, int idx0, u64 (&a)[8], const PrimeDev &P) const
        {
#pragma unroll
            for (int j = 0; j < 8; j++)
                a[j] = load1(row, idx0 + j, P);
        }
        __device__ __forceinline__ u64 *mid(int row) const { return plain + (static_cast<long long>(row) << logn); }
        __device__ __forceinline__ void store1(int row, int idx, u64 v, const PrimeDev &P) const { mid(row)[idx] = csub(v, P.q); }
        __device__ __forceinline__ void store8(int row, int idx0, u64 (&a)[8], const PrimeDev &P) const
        {
#pragma unroll
            for (int j = 0; j < 8; j++)
                store1(row, idx0 + j, a[j], P);
        }
    };
    struct OpBatchDecode
    {
        const u64 *plain;         // [B][n] coefficients
        const uint32_t *inv_map;
        u64 *tmp;                 // [B][n] intermediate rows of the two-pass transform
        u64 *values;              // [B][n]
        int logn, pid_t;
        __device__ __forceinline__ bool skip(int) const { return false; }
        __device__ __forceinline__ int pid(int) const { return pid_t; }
        __device__ __forceinline__ const u64 *direct(int row, const PrimeDev &) const { return plain + (static_cast<long long>(row) << logn); }
        __device__ __forceinline__ u64 load1(int row, int idx, const PrimeDev &P) const { return direct(row, P)[idx]; }
        __device__ __forceinline__ void load8(int, int, u64 (&)[8], const PrimeDev &) const {}
        __device__ __forceinline__ u64 *mid(int row) const { return tmp + (static_cast<long long>(row) << logn); }
        __device__ __forceinline__ void store1(int row, int idx, u64 v, const PrimeDev &P) const
        {
            values[(static_cast<long long>(row) << logn) + inv_map[idx]] = csub(csub(v, P.q2), P.q);
        }
        __device__ __forceinline__ void store8(int row, int idx0, u64 (&a)[8], const PrimeDev &P) const
        {
#pragma unroll
            for (int j = 0; j < 8; j++)
                store1(row, idx0 + j, a[j], P);
        }
    };

    static void check_batching(const Context &c)
    {
        if (c.t_pid < 0)
            throw std::invalid_argument("encryption parameters are not valid for batching"); // batchencoder.cpp:27-30
    }
    void op_batch_encode(Context &c, size_t batch, const u64 *values, u64 *plain, cudaStream_t st)
    {
        check_batching(c);
        if (values == plain)
            throw std::invalid_argument("batch_encode: input and output must not alias");
        const size_t step = std::max<size_t>(1, (size_t(1) << 30) / c.n);
        for (size_t b0 = 0; b0 < batch; b0 += step)
        {
            const size_t B = std::min(step, batch - b0);
            OpBatchEncode op{ values + b0 * c.n, c.d_batch_inv_map.get(), plain + b0 * c.n, c.logn, c.t_pid };
            cuda_check(launch_ntt_inv(op, static_cast<int>(B), c.logn, c.d_primes.get(), st, c.stats, "batch_encode_intt"), "batch encode");
        }
    }
    void op_batch_decode(Context &c, size_t batch, const u64 *plain, u64 *values, cudaStream_t st)
    {
        check_batching(c);
        if (values == plain)
            throw std::invalid_argument("batch_decode: input and output must not alias");
        const size_t step = std::max<size_t>(1, std::min<size_t>((size_t(1) << 30) / c.n, c.scratch_budget / (c.n * sizeof(u64))));
        for (size_t b0 = 0; b0 < batch; b0 += step)
        {
            const size_t B = std::min(step, batch - b0);
            u64 *tmp = static_cast<u64 *>(c.ensure_scratch(B * c.n * sizeof(u64)));
            OpBatchDecode op{ plain + b0 * c.n, c.d_batch_inv_map.get(), tmp, values + b0 * c.n, c.logn, c.t_pid };
            cuda_check(launch_ntt_fwd(op, static_cast<int>(B), c.logn, c.d_primes.get(), st, c.stats, "batch_decode_ntt", -1, (c.t >> 57) == 0),
                       "batch decode");
        }
    }

    // ---- decryption (decryptor.cpp): phase = c_0 + sum c_p s^p, then per scheme ---------------------------------------
    void secret_key_create(Context &c, const u64 *h_sk, SecretKey &out)
    {
        out.d_pow = DevBuf<u64>(c.k * c.n, true);
        cuda_check(cudaMemcpy(out.d_pow.get(), h_sk, out.d_pow.bytes(), cudaMemcpyHostToDevice), "upload secret key");
        out.ctx = &c, out.powers = 1;
    }
    // Decryptor::compute_secret_key_array (decryptor.cpp:199-310): s^p = s^(p-1) * s, dyadic at the key level
    void ensure_key_powers(Context &c, SecretKey &sk, size_t powers, cudaStream_t st)
    {
        if (powers <= sk.powers)
            return;
        const size_t row = c.k * c.n;
        sk.d_pow.grow(powers * row, true); // the old powers are wiped as they are freed
        u64 *s = sk.d_pow.get();
        for (size_t p = sk.powers; p < powers; p++)
            op_multiply_plain(c, c.k, 1, 1, false, s + (p - 1) * row, s, s + p * row, st);
        sk.powers = powers;
    }

    // sum_{p>=1} src_p * s^p (+ c_0) per coefficient; rows of src: item b, poly p-1 at src + b*src_bs + (p-1)*L*n
    template <bool ADD_C0>
    __global__ void __launch_bounds__(256) phase_kernel(const u64 *__restrict__ src, long long src_bs, const u64 *__restrict__ c0, long long c0_bs,
                                                         const u64 *__restrict__ skpow, long long sk_ps, u64 *__restrict__ out,
                                                         const PrimeDev *__restrict__ primes, int logn, int L, int npow, long long total)
    {
        long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over B*L*n
        if (e >= total)
            return;
        const long long poly = static_cast<long long>(L) << logn, b = e / poly, r = e % poly;
        const PrimeDev P = primes[static_cast<int>(r >> logn)];
        u64 lo = 0, hi = 0;
        for (int p = 0; p < npow; p++)
            mac128(lo, hi, src[b * src_bs + p * poly + r], skpow[p * sk_ps + r]);
        u64 v = barrett128(lo, hi, P.q, P.ratio_lo, P.ratio_hi);
        if (ADD_C0)
            v = csub(v + c0[b * c0_bs + r], P.q);
        out[e] = v;
    }

    struct DecConst
    {
        Tw c;      // BFV: (t * gamma mod q_i) * (q/q_i)^-1 mod q_i;  BGV: (q/q_i)^-1 mod q_i
        u64 m_t;   // (q/q_i) mod t
        u64 m_g;   // (q/q_i) mod gamma (BFV)
        u64 pad;
    };
    static_assert(sizeof(DecConst) == 40 || sizeof(DecConst) == 48, "layout");

    __device__ __forceinline__ u64 mulmod_any(u64 a, u64 b, u64 m, u64 ratio_lo, u64 ratio_hi)
    {
        // the ratio may sit one below floor(2^128 / m): one more conditional subtraction
        return csub(barrett128(a * b, __umul64hi(a, b), m, ratio_lo, ratio_hi), m);
    }

    // BFV: RNSTool::decrypt_scale_and_round (rns.cpp:1133-1191) on phase = T (INTT of the key part) + c_0
    __global__ void __launch_bounds__(128) bfv_scale_round_kernel(const u64 *__restrict__ T, const u64 *__restrict__ c0, long long c0_bs,
                                                                   u64 *__restrict__ plain, const DecConst *__restrict__ dc,
                                                                   const PrimeDev *__restrict__ primes, u64 t, u64 t_rlo, u64 t_rhi, u64 gamma,
                                                                   u64 g_rlo, u64 g_rhi, u64 neg_inv_q_t, u64 neg_inv_q_g, u64 inv_gamma_t,
                                                                   int logn, int L, long long total)
    {
        long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over B*n
        if (e >= total)
            return;
        const long long b = e >> logn;
        const int idx = static_cast<int>(e & ((1 << logn) - 1));
        u64 tl = 0, th = 0, gl = 0, gh = 0;
        for (int i = 0; i < L; i++)
        {
            const PrimeDev P = primes[i];
            const long long off = (static_cast<long long>(i) << logn) + idx;
            const u64 x = csub(T[((b * L) << logn) + off] + c0[b * c0_bs + off], P.q);
            const u64 u = mul_shoup(x, dc[i].c, P.q);
            mac128(tl, th, u, dc[i].m_t);
            mac128(gl, gh, u, dc[i].m_g);
        }
        u64 yt = csub(barrett128(tl, th, t, t_rlo, t_rhi), t), yg = csub(barrett128(gl, gh, gamma, g_rlo, g_rhi), gamma);
        yt = mulmod_any(yt, neg_inv_q_t, t, t_rlo, t_rhi);
        yg = mulmod_any(yg, neg_inv_q_g, gamma, g_rlo, g_rhi);
        u64 r;
        if (yg > (gamma >> 1))
            r = csub(yt + csub(barrett128(gamma - yg, 0, t, t_rlo, t_rhi), t), t);
        else
        {
            const u64 s = csub(barrett128(yg, 0, t, t_rlo, t_rhi), t);
            r = csub(yt + t - s, t);
        }
        plain[e] = mulmod_any(r, inv_gamma_t, t, t_rlo, t_rhi);
    }

    // BGV: BaseConverter::exact_convert_array (rns.cpp:466-539) on phase = T (already INTT'd), then the inverse correction factor
    __global__ void __launch_bounds__(128) bgv_modt_kernel(const u64 *__restrict__ T, u64 *__restrict__ plain, const DecConst *__restrict__ dc,
                                                            const PrimeDev *__restrict__ primes, const u64 *__restrict__ fix, u64 t, u64 t_rlo,
                                                            u64 t_rhi, u64 q_mod_t, int logn, int L, long long total)
    {
        long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over B*n
        if (e >= total)
            return;
        const long long b = e >> logn;
        const int idx = static_cast<int>(e & ((1 << logn) - 1));
        double v = 0.0;
        u64 lo = 0, hi = 0;
        for (int i = 0; i < L; i++)
        {
            const PrimeDev P = primes[i];
            const u64 x = mul_shoup(T[(((b * L) + i) << logn) + idx], dc[i].c, P.q);
            v = __dadd_rn(v, __ddiv_rn(__ull2double_rn(x), __ull2double_rn(P.q))); // IEEE doubles in index order, as the reference sums them
            mac128(lo, hi, x, dc[i].m_t);
        }
        const u64 rounded = __double2ull_rz(__dadd_rn(v, 0.5));
        const u64 sum = csub(barrett128(lo, hi, t, t_rlo, t_rhi), t);
        const u64 vq = mulmod_any(csub(barrett128(rounded, 0, t, t_rlo, t_rhi), t), q_mod_t, t, t_rlo, t_rhi);
        u64 r = csub(sum + t - vq, t);
        if (fix)
            r = mulmod_any(r, fix[b], t, t_rlo, t_rhi);
        plain[e] = r;
    }

    // Decryptor::invariant_noise_budget (decryptor.cpp:409-486), per coefficient: the coefficient-form phase (BFV: T + c_0 times t mod
    // q_i, multiply_poly_scalar_coeffmod; BGV: T), composed modulo Q (compose_array), centred against (Q + 1) / 2 (Q - v above it,
    // poly_infty_norm_coeffmod at :22-51) and its significant bit count.  The bit count of the maximum is the maximum of the bit counts,
    // so the norm reduces to one int per ciphertext: warp max, CTA max, one atomicMax per CTA into bits[b] (zeroed by the caller).
    // grid = (B, ceil(n / 128)): a CTA never spans two ciphertexts.  big / invp: Context::CrtLevel of the level.
    template <bool BFV>
    __global__ void __launch_bounds__(128) noise_norm_kernel(const u64 *__restrict__ T, const u64 *__restrict__ c0, long long c0_bs,
                                                             const u64 *__restrict__ t_mod_q, const u64 *__restrict__ big, const Tw *__restrict__ invp,
                                                             const PrimeDev *__restrict__ primes, int logn, int L, int *__restrict__ bits)
    {
        const long long b = blockIdx.x;
        const int i = static_cast<int>(blockIdx.y * blockDim.x + threadIdx.x);
        int nb = 0;
        if (i < (1 << logn))
        {
            const u64 *Q = big, *thr = big + L, *punct = big + 2 * L;
            const u64 *src = T + ((b * L) << logn) + i;
            const u64 *s0 = c0 + b * c0_bs + i;
            u64 val[kCrtMaxWords];
            crt_compose(
                [&](int j) {
                    const long long off = static_cast<long long>(j) << logn;
                    u64 x = src[off];
                    if (BFV)
                    {
                        const PrimeDev &P = primes[j];
                        x = mulmod_barrett(csub(x + s0[off], P.q), t_mod_q[j], P);
                    }
                    return x;
                },
                Q, punct, invp, primes, L, val);
            bool upper = true; // is_greater_than_or_equal_uint(value, (Q + 1) / 2)
            for (int w = L - 1; w >= 0; w--)
                if (val[w] != thr[w])
                {
                    upper = val[w] > thr[w];
                    break;
                }
            if (upper) // Q - value
            {
                u64 bw = 0;
                for (int w = 0; w < L; w++)
                {
                    const u64 a = Q[w], s1 = a - val[w], s2 = s1 - bw;
                    bw = (a < val[w]) | (s1 < bw);
                    val[w] = s2;
                }
            }
            for (int w = L - 1; w >= 0; w--) // get_significant_bit_count_uint
                if (val[w])
                {
                    nb = 64 * w + 64 - __clzll(static_cast<long long>(val[w]));
                    break;
                }
        }
        nb = __reduce_max_sync(0xffffffffu, static_cast<unsigned>(nb));
        __shared__ int warp_max[4];
        if ((threadIdx.x & 31) == 0)
            warp_max[threadIdx.x >> 5] = nb;
        __syncthreads();
        if (threadIdx.x == 0)
        {
            const int m = max(max(warp_max[0], warp_max[1]), max(warp_max[2], warp_max[3]));
            if (m)
                atomicMax(bits + b, m);
        }
    }

    // bits of the largest centred noise coefficient -> max(0, total_bits - bits - 1), in place
    __global__ void __launch_bounds__(256) noise_budget_kernel(int *__restrict__ budgets, int total_bits, long long B)
    {
        const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
        if (e >= B)
            return;
        budgets[e] = max(0, total_bits - budgets[e] - 1);
    }

    static u64 mulmod_host(u64 a, u64 b, u64 m) { return static_cast<u64>(static_cast<unsigned __int128>(a) * b % m); }

    Context::CrtLevel &crt_level(Context &c, size_t L)
    {
        auto it = c.crt_levels.find(L);
        if (it != c.crt_levels.end())
            return it->second;
        const sbh::CkksLevelHost h = sbh::ckks_level(c.q.data(), L);
        Context::CrtLevel lv;
        lv.total_bits = h.total_bits;
        std::vector<u64> big;
        big.insert(big.end(), h.Q.begin(), h.Q.end());
        big.insert(big.end(), h.threshold.begin(), h.threshold.end());
        big.insert(big.end(), h.punctured.begin(), h.punctured.end());
        std::vector<Tw> invp(L);
        for (size_t j = 0; j < L; j++)
            invp[j] = Tw{ h.inv_punctured[j].w, h.inv_punctured[j].wq };
        lv.d_big = upload<u64>(c, big);
        lv.d_invp = upload<Tw>(c, invp);
        return c.crt_levels.emplace(L, std::move(lv)).first->second;
    }
    static const Context::DecryptLevel &decrypt_level(Context &c, size_t L)
    {
        plain_level(c, L); // t Barrett ratio, scheme check
        auto it = c.decrypt_levels.find(L);
        if (it != c.decrypt_levels.end())
            return it->second;
        if (L > 60)
            throw std::invalid_argument("decryption supports at most 60 primes per level");
        const bool bfv = c.scheme == 1;
        const u64 t = c.t, gamma = bfv ? c.aux[1] : 1;
        Context::DecryptLevel dl;
        std::vector<DecConst> h(L);
        u64 q_t = 1 % t, q_g = 1 % gamma;
        for (size_t i = 0; i < L; i++)
            q_t = mulmod_host(q_t, c.q[i] % t, t), q_g = mulmod_host(q_g, c.q[i] % gamma, gamma);
        for (size_t i = 0; i < L; i++)
        {
            u64 punc_q = 1, punc_t = 1 % t, punc_g = 1 % gamma, inv = 0;
            for (size_t j = 0; j < L; j++)
                if (j != i)
                {
                    punc_q = mulmod_host(punc_q, c.q[j] % c.q[i], c.q[i]);
                    punc_t = mulmod_host(punc_t, c.q[j] % t, t);
                    punc_g = mulmod_host(punc_g, c.q[j] % gamma, gamma);
                }
            if (!sbh::invmod(punc_q, c.q[i], inv))
                throw std::logic_error("invalid rns bases");
            u64 cst = inv;
            if (bfv)
                cst = mulmod_host(mulmod_host(t % c.q[i], gamma % c.q[i], c.q[i]), inv, c.q[i]);
            h[i] = DecConst{ Tw{ cst, sbh::shoup(cst, c.q[i]) }, punc_t, punc_g, 0 };
        }
        u64 inv_t = 0, inv_g = 0;
        if (bfv)
        {
            if (!sbh::invmod(q_t, t, inv_t) || !sbh::invmod(q_g, gamma, inv_g))
                throw std::logic_error("invalid rns bases");
            dl.neg_inv_q_mod_t = inv_t ? t - inv_t : 0, dl.neg_inv_q_mod_g = inv_g ? gamma - inv_g : 0;
        }
        dl.q_mod_t = q_t;
        dl.d_consts = upload<DecConst>(c, h);
        return c.decrypt_levels.emplace(L, std::move(dl)).first->second;
    }

    // The coefficient-form phase of ciphertexts ct [batch][size][L][n] (BFV / BGV), in chunks of the batch that fit the scratch arena:
    // per chunk of B ciphertexts from b0, T [B][L][n] = BFV: INTT(sum_{p>=1} NTT(c_p) s^p) (decryptor.cpp:348-379; c_0 is left to the
    // consumer, which adds it in its own pass), BGV: INTT(c_0 + sum_{p>=1} c_p s^p) (:159-197, :409-486).  Then
    // consume(b0, B, T, in, extra): in = the chunk's ciphertexts, extra = B words of scratch the consumer may use.  The key powers
    // s^1 .. s^(size-1) must be in place (ensure_key_powers).
    template <class Consume>
    static void decrypt_phases(Context &c, const SecretKey &sk, size_t L, size_t size, size_t batch, const u64 *ct, cudaStream_t st,
                               const Consume &consume)
    {
        const bool bfv = c.scheme == 1;
        const int n = static_cast<int>(c.n), npow = static_cast<int>(size - 1);
        const long long poly = static_cast<long long>(L) * n, ct_bs = static_cast<long long>(size) * poly, sk_ps = static_cast<long long>(c.k) * n;
        // scratch per ciphertext: T [L][n] (+ the transformed copy of c_1.. for BFV) (+ 1 word for the consumer)
        const size_t per = (L * c.n * (bfv ? size : 1) + 1) * sizeof(u64);
        size_t chunk = std::min(batch, std::max<size_t>(1, c.scratch_budget / per));
        chunk = std::min<size_t>(chunk, std::max<size_t>(1, (size_t(1) << 30) / (size * L * c.n)));
        for (size_t b0 = 0; b0 < batch; b0 += chunk)
        {
            const size_t B = std::min(chunk, batch - b0);
            u64 *T = static_cast<u64 *>(c.ensure_scratch(per * B));
            u64 *extra = T + B * L * c.n;
            const u64 *in = ct + b0 * ct_bs;
            const long long total = static_cast<long long>(B) * poly;
            if (bfv)
            {
                // coefficient-form ciphertext: transform c_1.., accumulate, transform back
                u64 *X = extra; // [B][size-1][L][n]
                cuda_check(cudaMemcpy2DAsync(X, (size - 1) * poly * sizeof(u64), in + poly, ct_bs * sizeof(u64), (size - 1) * poly * sizeof(u64), B,
                                             cudaMemcpyDeviceToDevice, st),
                           "copy");
                op_ntt(c, false, L, size - 1, B, X, st);
                c.stats.begin("decrypt_phase", 0, 8.0 * total * size, st);
                phase_kernel<false><<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(X, static_cast<long long>(size - 1) * poly, nullptr, 0,
                                                                                                sk.d_pow.get(), sk_ps, T, c.d_primes.get(), c.logn,
                                                                                                static_cast<int>(L), npow, total);
                c.stats.end(st);
                cuda_check(cudaGetLastError(), "phase_kernel");
            }
            else
            {
                c.stats.begin("decrypt_phase", 0, 8.0 * total * (size + 1), st);
                phase_kernel<true><<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(in + poly, ct_bs, in, ct_bs, sk.d_pow.get(), sk_ps, T,
                                                                                               c.d_primes.get(), c.logn, static_cast<int>(L), npow, total);
                c.stats.end(st);
                cuda_check(cudaGetLastError(), "phase_kernel");
            }
            op_ntt(c, true, L, 1, B, T, st);
            consume(b0, B, T, in, extra);
        }
    }

    void op_decrypt(Context &c, SecretKey &sk, size_t L, size_t size, size_t batch, const u64 *ct, const u64 *h_cf, u64 *plain, cudaStream_t st)
    {
        if (sk.ctx != &c)
            throw std::invalid_argument("secret key is not valid for encryption parameters");
        if (size < 2 || size > 16)
            throw std::invalid_argument("encrypted is not valid for encryption parameters");
        ensure_key_powers(c, sk, size - 1, st);
        const int n = static_cast<int>(c.n), npow = static_cast<int>(size - 1);
        const long long poly = static_cast<long long>(L) * n, ct_bs = static_cast<long long>(size) * poly, sk_ps = static_cast<long long>(c.k) * n;
        if (c.scheme == 2)
        {
            // ckks_decrypt (decryptor.cpp:137-157): the phase in NTT form is the plaintext
            const size_t step = std::max<size_t>(1, (size_t(1) << 31) / (L * c.n));
            for (size_t b0 = 0; b0 < batch; b0 += step)
            {
                const size_t B = std::min(step, batch - b0);
                const long long total = static_cast<long long>(B) * poly;
                const u64 *in = ct + b0 * ct_bs;
                c.stats.begin("decrypt_phase", 0, 8.0 * total * (size + 1), st);
                phase_kernel<true><<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(in + poly, ct_bs, in, ct_bs, sk.d_pow.get(), sk_ps,
                                                                                               plain + b0 * poly, c.d_primes.get(), c.logn,
                                                                                               static_cast<int>(L), npow, total);
                c.stats.end(st);
                cuda_check(cudaGetLastError(), "phase_kernel");
            }
            return;
        }
        const Context::DecryptLevel &dl = decrypt_level(c, L);
        if (c.scheme == 1)
        {
            const u64 gamma = c.aux[1];
            const unsigned __int128 ratio = ~static_cast<unsigned __int128>(0) / gamma;
            const u64 g_rlo = static_cast<u64>(ratio), g_rhi = static_cast<u64>(ratio >> 64);
            u64 inv_gamma_t = 0;
            if (!sbh::invmod(gamma % c.t, c.t, inv_gamma_t))
                throw std::logic_error("invalid rns bases");
            decrypt_phases(c, sk, L, size, batch, ct, st, [&](size_t b0, size_t B, const u64 *T, const u64 *in, u64 *) {
                const long long tn = static_cast<long long>(B) * n;
                c.stats.begin("bfv_scale_round", 0, 8.0 * tn * (2 * L + 1), st);
                bfv_scale_round_kernel<<<static_cast<unsigned>((tn + 127) / 128), 128, 0, st>>>(
                    T, in, ct_bs, plain + b0 * c.n, dl.d_consts.get(), c.d_primes.get(), c.t, c.t_ratio_lo, c.t_ratio_hi, gamma,
                    g_rlo, g_rhi, dl.neg_inv_q_mod_t, dl.neg_inv_q_mod_g, inv_gamma_t, c.logn, static_cast<int>(L), tn);
                c.stats.end(st);
                cuda_check(cudaGetLastError(), "bfv_scale_round_kernel");
            });
            return;
        }
        // bgv_decrypt (decryptor.cpp:159-197)
        decrypt_phases(c, sk, L, size, batch, ct, st, [&](size_t b0, size_t B, const u64 *T, const u64 *, u64 *extra) {
            const long long tn = static_cast<long long>(B) * n;
            const u64 *d_fix = nullptr;
            std::vector<u64> fix;
            if (h_cf)
            {
                fix.resize(B);
                for (size_t i = 0; i < B; i++)
                {
                    fix[i] = 1;
                    if (h_cf[b0 + i] != 1 && !sbh::invmod(h_cf[b0 + i] % c.t, c.t, fix[i]))
                        throw std::logic_error("invalid correction factor");
                }
                cuda_check(cudaMemcpyAsync(extra, fix.data(), B * sizeof(u64), cudaMemcpyHostToDevice, st), "upload factors");
                cuda_check(cudaStreamSynchronize(st), "synchronize"); // fix lives on this stack frame
                d_fix = extra;
            }
            c.stats.begin("bgv_modt", 0, 8.0 * tn * (L + 1), st);
            bgv_modt_kernel<<<static_cast<unsigned>((tn + 127) / 128), 128, 0, st>>>(T, plain + b0 * c.n, dl.d_consts.get(),
                                                                                     c.d_primes.get(), d_fix, c.t, c.t_ratio_lo, c.t_ratio_hi, dl.q_mod_t,
                                                                                     c.logn, static_cast<int>(L), tn);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "bgv_modt_kernel");
        });
    }

    void check_noise_budget(const Context &c, const SecretKey &sk, size_t L, size_t size)
    {
        if (sk.ctx != &c)
            throw std::invalid_argument("secret key is not valid for encryption parameters");
        if (size < 2 || size > 16)
            throw std::invalid_argument("encrypted is not valid for encryption parameters");
        if (c.scheme != 1 && c.scheme != 3) // the reference has no noise budget for CKKS (decryptor.cpp:424-428)
            throw std::logic_error("unsupported scheme");
        if (L > 60) // the decryption limit (decrypt_level); the composition itself would take up to 64 primes
            throw std::invalid_argument("decryption supports at most 60 primes per level");
    }

    void op_invariant_noise_budget(Context &c, SecretKey &sk, size_t L, size_t size, size_t batch, const u64 *ct, int *budgets, cudaStream_t st)
    {
        check_noise_budget(c, sk, L, size);
        if (!batch)
            return;
        const Context::CrtLevel &lv = crt_level(c, L);
        if (!c.d_t_mod_q)
            plain_level(c, L); // t mod q_i (BFV multiplies the phase by t)
        ensure_key_powers(c, sk, size - 1, st);
        const bool bfv = c.scheme == 1;
        const long long ct_bs = static_cast<long long>(size) * L * c.n;
        cuda_check(cudaMemsetAsync(budgets, 0, batch * sizeof(int), st), "memset");
        decrypt_phases(c, sk, L, size, batch, ct, st, [&](size_t b0, size_t B, const u64 *T, const u64 *in, u64 *) {
            const dim3 grid(static_cast<unsigned>(B), static_cast<unsigned>((c.n + 127) / 128));
            c.stats.begin("noise_norm", 0, 8.0 * B * c.n * (bfv ? 2 * L : L), st);
            if (bfv)
                noise_norm_kernel<true><<<grid, 128, 0, st>>>(T, in, ct_bs, c.d_t_mod_q.get(), lv.d_big.get(), lv.d_invp.get(), c.d_primes.get(), c.logn, static_cast<int>(L),
                                                              budgets + b0);
            else
                noise_norm_kernel<false><<<grid, 128, 0, st>>>(T, in, ct_bs, c.d_t_mod_q.get(), lv.d_big.get(), lv.d_invp.get(), c.d_primes.get(), c.logn, static_cast<int>(L),
                                                               budgets + b0);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "noise_norm_kernel");
        });
        c.stats.begin("noise_budget", 0, 8.0 * batch, st);
        noise_budget_kernel<<<static_cast<unsigned>((batch + 255) / 256), 256, 0, st>>>(budgets, lv.total_bits, static_cast<long long>(batch));
        c.stats.end(st);
        cuda_check(cudaGetLastError(), "noise_budget_kernel");
    }

    // ------------------------------------------------------------------------------------- key switching ----
    // (1) target -> coefficient form: OpKsIntt (sb_src.cuh)

    // (2) digit J re-reduced modulo output prime I and transformed: rows (b, I, J); evaluator.cpp:2682-2702
    struct OpKsDigit
    {
        Src dsrc; // coefficient-form digits: D (CKKS) or the target itself (BFV)
        u64 *E;   // [B][L+1][L][n]
        const PrimeDev *primes;
        int logn, L, k, ntt_in, reduce; // reduce == 0: every digit prime < 4 * every output prime, loads are in range as is
        __device__ __forceinline__ bool skip(int row) const { return ntt_in && ((row / L) % (L + 1)) == (row % L); }
        __device__ __forceinline__ int pid(int row) const
        {
            int I = (row / L) % (L + 1);
            return I == L ? k - 1 : I;
        }
        __device__ __forceinline__ const u64 *direct(int row, const PrimeDev &P) const
        {
            const int J = row % L;
            if (!dsrc.plain() || (reduce && primes[J].q > P.q))
                return nullptr;
            return dsrc.row(row / (L * (L + 1)), J);
        }
        __device__ __forceinline__ u64 load1(int row, int idx, const PrimeDev &P) const
        {
            int J = row % L, b = row / (L * (L + 1));
            u64 qJ = primes[J].q;
            u64 v = dsrc.get(b, J, idx, qJ);
            return (reduce && qJ > P.q) ? barrett64(v, P.q, P.ratio_hi) : v; // evaluator.cpp:2690-2698
        }
        __device__ __forceinline__ void load8(int, int, u64 (&)[8], const PrimeDev &) const {}
        __device__ __forceinline__ u64 *mid(int row) const { return E + (static_cast<long long>(row) << logn); }
        __device__ __forceinline__ void store1(int row, int idx, u64 v, const PrimeDev &P) const
        {
            mid(row)[idx] = csub(csub(v, P.q2), P.q);
        }
        __device__ __forceinline__ void store8(int row, int idx0, u64 (&a)[8], const PrimeDev &P) const
        {
            ulonglong2 *p = reinterpret_cast<ulonglong2 *>(mid(row) + idx0);
#pragma unroll
            for (int j = 0; j < 4; j++)
                p[j] = make_ulonglong2(csub(csub(a[2 * j], P.q2), P.q), csub(csub(a[2 * j + 1], P.q2), P.q));
        }
    };

    // The digit sums of (3) add L products of canonical words, each below (q_I - 1)^2: without a reduction they fit 128 bits as long
    // as L (q_max - 1)^2 < 2^128 at the largest output prime of the level: at every level of primes up to 60 bits (L <= 255), but only
    // up to 64 digits of the largest 61-bit primes.  Deeper levels take the WINDOW instantiations, which reduce the sums after every
    // kKsSumWindow digits: a carried residue plus 64 products, (q - 1) + 64 (q - 1)^2, stays below 2^128 at every prime below 2^61
    // (the context's bound), and 65 products of the largest 61-bit primes do not (DESIGN 3.2b).
    constexpr int kKsSumWindow = 64;
    static bool ks_sum_needs_window(const Context &c, size_t L)
    {
        u64 qmax = c.q[c.k - 1];
        for (size_t i = 0; i < L; i++)
            qmax = std::max(qmax, c.q[i]);
        const unsigned __int128 sq = static_cast<unsigned __int128>(qmax - 1) * (qmax - 1);
        return sq > ~static_cast<unsigned __int128>(0) / L; // L (q_max - 1)^2 >= 2^128
    }

    // (3) multiply-accumulate with the key, 128-bit lazy sums, one Barrett at the end; evaluator.cpp:2705-2755
    //     grid = (B, n/256, L+1): consecutive CTAs share the key tile of (I, coefficient range) through L2.
    //     WINDOW: the sums are also reduced after every kKsSumWindow digits (ks_sum_needs_window).
    template <bool WINDOW>
    __global__ void __launch_bounds__(256) ks_mac_kernel(const u64 *__restrict__ E, Src tgt, int ntt_in, const u64 *__restrict__ key,
                                                          u64 *__restrict__ Pp, const PrimeDev *__restrict__ primes, int logn, int L, int k)
    {
        const int n = 1 << logn;
        const int b = blockIdx.x, I = blockIdx.z;
        const int idx = blockIdx.y * blockDim.x + threadIdx.x;
        if (idx >= n)
            return;
        const int ki = (I == L) ? k - 1 : I;
        const PrimeDev P = primes[ki];
        u64 lo0 = 0, hi0 = 0, lo1 = 0, hi1 = 0;
        const u64 *e = E + ((static_cast<long long>(b) * (L + 1) + I) * L << logn) + idx;
        for (int J = 0, since = 0; J < L; J++)
        {
            u64 x = (ntt_in && I == J) ? tgt.get(b, J, idx, P.q) : e[static_cast<long long>(J) << logn];
            const u64 *kr = key + ((static_cast<long long>(J) * 2 * k + ki) << logn) + idx;
            mac128(lo0, hi0, x, __ldg(kr));
            mac128(lo1, hi1, x, __ldg(kr + (static_cast<long long>(k) << logn)));
            if (WINDOW && ++since == kKsSumWindow)
            {
                since = 0;
                lo0 = barrett128(lo0, hi0, P.q, P.ratio_lo, P.ratio_hi), hi0 = 0;
                lo1 = barrett128(lo1, hi1, P.q, P.ratio_lo, P.ratio_hi), hi1 = 0;
            }
        }
        u64 *o = Pp + (((static_cast<long long>(b) * 2) * (L + 1) + I) << logn) + idx;
        o[0] = barrett128(lo0, hi0, P.q, P.ratio_lo, P.ratio_hi);
        o[static_cast<long long>(L + 1) << logn] = barrett128(lo1, hi1, P.q, P.ratio_lo, P.ratio_hi);
    }

    // (2a) column pass of ALL digits of one (ciphertext b, output prime I) in one CTA: the twiddles of prime I are staged once
    //      by TMA and reused for the L digit rows (the generic ntt_fwd_col pays the staging + row decoding per row).
    //      grid = (column tiles, B*(L+1)); same arithmetic as ntt_fwd_col<LOGNA, FAST, OpKsDigit>.
    //      PLAIN: every digit row is a plain in-range array (no Galois view, no re-reduction) -- the CKKS / BGV case with
    //      primes of one size; the loop then is loads with immediate offsets + the butterflies + stores.
    template <int LOGNA, bool FAST, bool PLAIN>
    __global__ void __launch_bounds__(kColThreads, SB_COL_MIN_BLOCKS) ks_digit_col_kernel(OpKsDigit op, const PrimeDev *__restrict__ primes)
    {
        constexpr int NA = 1 << LOGNA;
        constexpr int C = kTile / NA;
        __shared__ __align__(16) u64 tile[kTile];
        __shared__ __align__(16) Tw tw_s[NA];
        __shared__ __align__(8) u64 bar;
        const int L = op.L, bi = blockIdx.y, I = bi % (L + 1), b = bi / (L + 1), col0 = blockIdx.x * C;
        const int tid = threadIdx.x, c = tid % C, ridx = tid / C;
        const PrimeDev P = primes[I == L ? op.k - 1 : I];
        if (tid == 0)
            mbar_init(&bar, 1);
        __syncthreads();
        if (tid == 0)
        {
            mbar_expect_tx(&bar, NA * sizeof(Tw));
            tma_load_1d(tw_s, P.fwd, NA * sizeof(Tw), &bar);
        }
        mbar_wait(&bar, 0);
        constexpr int g = NA >> 3;
        const int off = (ridx << kLocalLog) + col0 + c;
        const long long n = 1LL << op.logn;
        if (PLAIN)
        {
            const u64 *src = op.dsrc.p + b * op.dsrc.bstride + off;
            u64 *dst = op.E + ((static_cast<long long>(bi) * L) << op.logn) + ((8 * ridx) << kLocalLog) + col0 + c;
            const int skipJ = op.ntt_in ? I : -1;
            for (int J = 0; J < L; J++, src += n, dst += n)
            {
                if (J == skipJ)
                    continue;
                u64 a[8];
#pragma unroll
                for (int j = 0; j < 8; j++)
                    a[j] = src[(j * g) << kLocalLog];
                fwd_col_passes<LOGNA, FAST>(a, tile, tw_s, ridx, c, P);
#pragma unroll
                for (int j = 0; j < 8; j++)
                    dst[j << kLocalLog] = a[j];
            }
            return;
        }
        for (int J = 0; J < L; J++)
        {
            if (op.ntt_in && J == I)
                continue;
            const int row = bi * L + J;
            u64 a[8];
            // same decision as OpKsDigit::direct(), without its per-row index divisions
            const u64 *dp = (op.dsrc.plain() && !(op.reduce && primes[J].q > P.q)) ? op.dsrc.row(b, J) : nullptr;
            if (dp)
            {
#pragma unroll
                for (int j = 0; j < 8; j++)
                    a[j] = dp[off + ((j * g) << kLocalLog)];
            }
            else
            {
#pragma unroll
                for (int j = 0; j < 8; j++)
                    a[j] = op.load1(row, off + ((j * g) << kLocalLog), P);
            }
            fwd_col_passes<LOGNA, FAST>(a, tile, tw_s, ridx, c, P);
            u64 *mid = op.mid(row);
#pragma unroll
            for (int j = 0; j < 8; j++)
                mid[((8 * ridx + j) << kLocalLog) + col0 + c] = a[j];
        }
    }

    template <int LOGNA>
    static void launch_ks_digit_col(const OpKsDigit &op, int B, bool fast, bool plain, const PrimeDev *primes, cudaStream_t st)
    {
        dim3 grid((1 << kLocalLog) / (kTile >> LOGNA), static_cast<unsigned>(B * (op.L + 1)));
        if (fast && plain)
            ks_digit_col_kernel<LOGNA, true, true><<<grid, kColThreads, 0, st>>>(op, primes);
        else if (fast)
            ks_digit_col_kernel<LOGNA, true, false><<<grid, kColThreads, 0, st>>>(op, primes);
        else if (plain)
            ks_digit_col_kernel<LOGNA, false, true><<<grid, kColThreads, 0, st>>>(op, primes);
        else
            ks_digit_col_kernel<LOGNA, false, false><<<grid, kColThreads, 0, st>>>(op, primes);
    }

    // (2b)+(3) fused: the 8 in-block stages of every digit transform + the multiply-accumulate with the key, looping
    //     over the digits J inside the kernel so the transformed digits never reach memory and the 128-bit sums live in
    //     registers.  One warp owns one 256-coefficient block of one (ciphertext b, output prime I); a CTA = 8 adjacent
    //     blocks.  blockIdx.x = b + B * block_group: consecutive CTAs share the key tile of (I, block group) through L2.
    // Component 0 accumulates in registers, component 1 in shared memory (128-bit carry-chain sums).
    struct KsMacSmem
    {
        static constexpr size_t xs = 8 * 256 * sizeof(u64);
        static constexpr size_t acc = 8 * 256 * sizeof(ulonglong2);
        static constexpr size_t tw = (8 * 255 + 1) * sizeof(Tw);
        static constexpr size_t total = xs + acc + tw + 16;
    };
    // PLAIN: the target is a plain slab (relinearize / multiply_relinearize); rotations read it through a Galois view.
    // WINDOW (guarded primes only): the sums are also reduced after every kKsSumWindow digits, as in ks_mac_kernel.
    template <bool FAST, bool PLAIN, bool WINDOW>
    __global__ void __launch_bounds__(256, SB_MAC_MIN_BLOCKS) ks_local_mac_kernel(const u64 *__restrict__ E, Src tgt, int ntt_in, const u64 *__restrict__ key,
                                                                   u64 *__restrict__ Pp, const PrimeDev *__restrict__ primes, int logn, int L, int k,
                                                                   int B)
    {
        // dynamic shared memory: [xs 8x256 u64 | component-1 sums 8x256 x 16 B | twiddles 8*255 x 16 B | mbarrier]
        extern __shared__ __align__(16) unsigned char ks_smem[];
        using SM = KsMacSmem;
        u64(*xs)[256] = reinterpret_cast<u64(*)[256]>(ks_smem);
        // 128-bit sums of key component 1 live in shared memory ([j][thread], conflict-free 16-byte accesses); component 0
        // stays in registers
        ulonglong2(*acc1)[256] = reinterpret_cast<ulonglong2(*)[256]>(ks_smem + SM::xs);
        // the twiddles of this CTA's 8 blocks are the same for every digit J: staged once with 8 TMA bulk copies
        // (stage s of 8 adjacent blocks is one contiguous run of 8*2^s table entries)
        Tw *tws = reinterpret_cast<Tw *>(ks_smem + SM::xs + SM::acc);
        u64 *bar = reinterpret_cast<u64 *>(tws + 8 * 255 + 1);
        const int warp = threadIdx.x >> 5, l = threadIdx.x & 31;
        const int b = blockIdx.x % B, bg = blockIdx.x / B, I = blockIdx.y;
        const int na = 1 << (logn - kLocalLog), blk = bg * 8 + warp;
        const int ki = (I == L) ? k - 1 : I;
        const PrimeDev P = primes[ki];
        const int e0 = (blk << kLocalLog) + 8 * l; // first of this lane's 8 consecutive output coefficients
        if (threadIdx.x == 0)
            mbar_init(bar, 1);
        __syncthreads();
        if (threadIdx.x == 0)
        {
            mbar_expect_tx(bar, 8 * 255 * sizeof(Tw));
#pragma unroll
            for (int st = 0; st < 8; st++)
                tma_load_1d(tws + 8 * ((1 << st) - 1), P.fwd + ((na + bg * 8) << st), (8u << st) * sizeof(Tw), bar);
        }
        u64 s0l[8], s0h[8];
#pragma unroll
        for (int j = 0; j < 8; j++)
        {
            s0l[j] = s0h[j] = 0;
            acc1[j][threadIdx.x] = make_ulonglong2(0, 0);
        }
        mbar_wait(bar, 0);
        auto twf = [&](int st, int i) { return tws[8 * ((1 << st) - 1) + (warp << st) + i]; };
        const u64 *erow = E + ((static_cast<long long>(b) * (L + 1) + I) * L << logn) + (blk << kLocalLog);
        // key rows of output prime I: component c of digit J at key + ((J*2 + c)*k + ki) * n
        const long long kstep = (2LL * k) << logn, kcomp = static_cast<long long>(k) << logn;
        const u64 *krow = key + (static_cast<long long>(ki) << logn) + e0;
        for (int J = 0, since = 0; J < L; J++, krow += kstep)
        {
            u64 a[8];
            if (ntt_in && J == I)
            {
                // the input already is digit J in NTT form modulo q_J (evaluator.cpp:2682-2685)
                if (PLAIN || tgt.plain())
                {
                    const ulonglong2 *tp = reinterpret_cast<const ulonglong2 *>(tgt.p + b * tgt.bstride + (static_cast<long long>(J) << logn) + e0);
#pragma unroll
                    for (int h = 0; h < 4; h++)
                    {
                        ulonglong2 v = tp[h];
                        a[2 * h] = v.x, a[2 * h + 1] = v.y;
                    }
                }
                else
                {
#pragma unroll
                    for (int j = 0; j < 8; j++)
                        a[j] = tgt.get(b, J, e0 + j, P.q);
                }
            }
            else
            {
                const u64 *src = erow + (static_cast<long long>(J) << logn);
#pragma unroll
                for (int j = 0; j < 8; j++)
                    a[j] = src[l + 32 * j];
                fwd_local_block_tw<FAST>(a, xs[warp], twf, l, P);
                if (!FAST)
                {
#pragma unroll
                    for (int j = 0; j < 8; j++)
                        a[j] = csub(csub(csub(a[j], P.q4), P.q2), P.q); // canonical: 256 summands fit 128 bits at 60 bits, 64 at 61 (WINDOW)
                }
                else if (L > 200)
                {
                    // guard-free values reach 72q < 2^63.2: more than 227 products with a 57-bit key word would overflow 128 bits
#pragma unroll
                    for (int j = 0; j < 8; j++)
                        a[j] = barrett_lazy4(a[j], P.ratio_hi, P.nq);
                }
            }
            const ulonglong2 *k0 = reinterpret_cast<const ulonglong2 *>(krow);
            const ulonglong2 *k1 = reinterpret_cast<const ulonglong2 *>(krow + kcomp);
#pragma unroll
            for (int h = 0; h < 4; h++)
            {
                ulonglong2 v = __ldg(k0 + h);
                mac128_4(s0l[2 * h], s0h[2 * h], a[2 * h], v.x);
                mac128_4(s0l[2 * h + 1], s0h[2 * h + 1], a[2 * h + 1], v.y);
            }
#pragma unroll
            for (int h = 0; h < 4; h++)
            {
                ulonglong2 v = __ldg(k1 + h);
                ulonglong2 t0 = acc1[2 * h][threadIdx.x], t1 = acc1[2 * h + 1][threadIdx.x];
                mac128_4(t0.x, t0.y, a[2 * h], v.x);
                mac128_4(t1.x, t1.y, a[2 * h + 1], v.y);
                acc1[2 * h][threadIdx.x] = t0;
                acc1[2 * h + 1][threadIdx.x] = t1;
            }
            if (WINDOW && ++since == kKsSumWindow)
            {
                since = 0;
#pragma unroll
                for (int j = 0; j < 8; j++)
                {
                    s0l[j] = barrett128(s0l[j], s0h[j], P.q, P.ratio_lo, P.ratio_hi), s0h[j] = 0;
                    const ulonglong2 t = acc1[j][threadIdx.x];
                    acc1[j][threadIdx.x] = make_ulonglong2(barrett128(t.x, t.y, P.q, P.ratio_lo, P.ratio_hi), 0);
                }
            }
        }
        ulonglong2 *o0 = reinterpret_cast<ulonglong2 *>(Pp + (((static_cast<long long>(b) * 2) * (L + 1) + I) << logn) + e0);
        ulonglong2 *o1 = reinterpret_cast<ulonglong2 *>(Pp + (((static_cast<long long>(b) * 2 + 1) * (L + 1) + I) << logn) + e0);
#pragma unroll
        for (int h = 0; h < 4; h++)
        {
            o0[h] = make_ulonglong2(barrett128(s0l[2 * h], s0h[2 * h], P.q, P.ratio_lo, P.ratio_hi),
                                    barrett128(s0l[2 * h + 1], s0h[2 * h + 1], P.q, P.ratio_lo, P.ratio_hi));
            ulonglong2 t0 = acc1[2 * h][threadIdx.x], t1 = acc1[2 * h + 1][threadIdx.x];
            o1[h] = make_ulonglong2(barrett128(t0.x, t0.y, P.q, P.ratio_lo, P.ratio_hi), barrett128(t1.x, t1.y, P.q, P.ratio_lo, P.ratio_hi));
        }
    }

    // (4a) special-prime component back to coefficients, + floor(q_sp/2) for rounding; evaluator.cpp:2809-2817.
    //      Also used by rescale with the last data prime (rns.cpp:855-860).  rows = (b, c)
    struct OpTopIntt
    {
        const u64 *src;          // row (b,c) at src + b*bstride + c*pstride
        long long bstride, pstride;
        u64 *U;                  // [B][2][n]
        int logn, pid_top;
        // BGV (evaluator.cpp:2770-2779, rns.cpp:1202-1213): U = the canonical top component, K = -U * q_top^-1 mod t
        u64 *K = nullptr;
        u64 t = 0, t_ratio = 0;
        Tw inv_top_mod_t = { 0, 0 };
        __device__ __forceinline__ bool skip(int) const { return false; }
        __device__ __forceinline__ int pid(int) const { return pid_top; }
        __device__ __forceinline__ const u64 *rowp(int row) const { return src + (row >> 1) * bstride + (row & 1) * pstride; }
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
        __device__ __forceinline__ u64 *mid(int row) const { return U + (static_cast<long long>(row) << logn); }
        __device__ __forceinline__ void store1(int row, int idx, u64 v, const PrimeDev &P) const
        {
            if (K)
            {
                const u64 u = csub(v, P.q), r = barrett64(u, t, t_ratio);
                mid(row)[idx] = u;
                K[(static_cast<long long>(row) << logn) + idx] = mul_shoup(r ? t - r : 0, inv_top_mod_t, t);
                return;
            }
            mid(row)[idx] = csub(csub(v, P.q) + (P.q >> 1), P.q);
        }
        __device__ __forceinline__ void store8(int row, int idx0, u64 (&a)[8], const PrimeDev &P) const
        {
#pragma unroll
            for (int j = 0; j < 8; j++)
                store1(row, idx0 + j, a[j], P);
        }
    };

    // in-place INTT of rows (b, c, i<L) of the accumulated products (BFV branch, evaluator.cpp:2854)
    struct OpProdIntt
    {
        u64 *Pp; // [B][2][L+1][n]
        int logn, L;
        __device__ __forceinline__ bool skip(int) const { return false; }
        __device__ __forceinline__ int pid(int row) const { return row % L; }
        __device__ __forceinline__ u64 *rowp(int row) const
        {
            return Pp + ((static_cast<long long>(row / L) * (L + 1) + row % L) << logn);
        }
        __device__ __forceinline__ const u64 *direct(int row, const PrimeDev &) const { return rowp(row); }
        __device__ __forceinline__ u64 load1(int row, int idx, const PrimeDev &) const { return rowp(row)[idx]; }
        __device__ __forceinline__ void load8(int row, int idx0, u64 (&a)[8], const PrimeDev &) const
        {
#pragma unroll
            for (int j = 0; j < 8; j++)
                a[j] = rowp(row)[idx0 + j];
        }
        __device__ __forceinline__ u64 *mid(int row) const { return rowp(row); }
        __device__ __forceinline__ void store1(int row, int idx, u64 v, const PrimeDev &P) const { rowp(row)[idx] = csub(v, P.q); }
        __device__ __forceinline__ void store8(int row, int idx0, u64 (&a)[8], const PrimeDev &P) const
        {
#pragma unroll
            for (int j = 0; j < 8; j++)
                store1(row, idx0 + j, a[j], P);
        }
    };

    // (4b) per data prime: NTT((u mod q_i) - (half mod q_i)), subtract from the accumulated component, scale by
    //      q_top^-1 and add into the ciphertext; evaluator.cpp:2819-2864 (CKKS branch), rns.cpp:863-900 (rescale).
    //      rows = (b, c, i), i < Lout
    template <class Base = BaseSrc>
    struct OpModDownFwd
    {
        const u64 *U;            // [B][2][n]: (INTT(top component) + half) mod q_top
        const u64 *X;            // component being corrected: X + b*x_bs + c*x_ps + i*n
        long long x_bs, x_ps;
        u64 *T;                  // intermediate rows [B][2][Lout][n]
        u64 *out;                // out + b*o_bs + c*o_ps + i*n
        long long o_bs, o_ps;
        const Tw *inv_top;       // q_top^-1 mod q_i, i < Lout
        Base base;
        u64 q_top;
        int logn, Lout;
        __device__ __forceinline__ bool skip(int) const { return false; }
        __device__ __forceinline__ int pid(int row) const { return row % Lout; }
        __device__ __forceinline__ const u64 *direct(int, const PrimeDev &) const { return nullptr; }
        __device__ __forceinline__ u64 load1(int row, int idx, const PrimeDev &P) const
        {
            u64 u = U[(static_cast<long long>(row / Lout) << logn) + idx];
            if (q_top > P.q)
                u = barrett64(u, P.q, P.ratio_hi);
            u64 half_mod = barrett64(q_top >> 1, P.q, P.ratio_hi);
            return u + (P.q - half_mod); // < 2q (or < q_top + q <= 2q when no reduction was needed)
        }
        __device__ __forceinline__ void load8(int, int, u64 (&)[8], const PrimeDev &) const {}
        __device__ __forceinline__ u64 *mid(int row) const { return T + (static_cast<long long>(row) << logn); }
        __device__ __forceinline__ void store1(int row, int idx, u64 v, const PrimeDev &P) const
        {
            const int i = row % Lout, bc = row / Lout, b = bc >> 1, c = bc & 1;
            u64 t = csub(csub(v, P.q2), P.q);
            u64 x = X[b * x_bs + c * x_ps + (static_cast<long long>(i) << logn) + idx];
            u64 r = mul_shoup(x + P.q - t, inv_top[i], P.q);
            r = csub(r + base.get(b, c, i, idx, P.q), P.q);
            out[b * o_bs + c * o_ps + (static_cast<long long>(i) << logn) + idx] = finish(base, b, c, i, logn, idx, r, P);
        }
        __device__ __forceinline__ void store8(int row, int idx0, u64 (&a)[8], const PrimeDev &P) const
        {
            // 8 consecutive coefficients: 16-byte loads of the accumulated component and of the base ciphertext, 16-byte stores
            const int i = row % Lout, bc = row / Lout, b = bc >> 1, c = bc & 1;
            const ulonglong2 *xp = reinterpret_cast<const ulonglong2 *>(X + b * x_bs + c * x_ps + (static_cast<long long>(i) << logn) + idx0);
            ulonglong2 *op_ = reinterpret_cast<ulonglong2 *>(out + b * o_bs + c * o_ps + (static_cast<long long>(i) << logn) + idx0);
            const bool has_base = base.present && !(c == 1 && base.c1_zero);
            const bool base_plain = has_base && base.s.plain();
            const ulonglong2 *bp = base_plain ? reinterpret_cast<const ulonglong2 *>(base.s.row(b, i) + c * base.pstride + idx0) : nullptr;
            const Tw inv = inv_top[i];
#pragma unroll
            for (int h = 0; h < 4; h++)
            {
                ulonglong2 x = xp[h];
                u64 t0 = csub(csub(a[2 * h], P.q2), P.q), t1 = csub(csub(a[2 * h + 1], P.q2), P.q);
                u64 r0 = mul_shoup(x.x + P.q - t0, inv, P.q), r1 = mul_shoup(x.y + P.q - t1, inv, P.q);
                if (base_plain)
                {
                    ulonglong2 bv = bp[h];
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

    // BGV: the correction polynomial is delta = (U mod q_i) + (K mod q_i) * (q_top mod q_i) instead of (u mod q_i) - half
    // (evaluator.cpp:2762-2805, rns.cpp:1216-1235); the transform and the epilogue are the ones above.
    template <class Base = BaseSrc>
    struct OpModDownFwdBgv : OpModDownFwd<Base>
    {
        const u64 *K;            // [B][2][n]: -U * q_top^-1 mod t
        const Tw *qtop_mod;      // q_top mod q_i, i < Lout
        u64 t;
        __device__ __forceinline__ u64 load1(int row, int idx, const PrimeDev &P) const
        {
            const long long e = (static_cast<long long>(row / this->Lout) << this->logn) + idx;
            u64 u = this->U[e], kk = K[e];
            if (this->q_top > P.q)
                u = barrett64(u, P.q, P.ratio_hi);
            if (t > P.q)
                kk = barrett64(kk, P.q, P.ratio_hi);
            return u + mul_shoup(kk, qtop_mod[row % this->Lout], P.q); // < 2q
        }
    };

    // coefficient-form mod-down (BFV): evaluator.cpp:2819-2864 (bfv branch) and rns.cpp:789-828 (mod_switch).
    // ADD_HALF: U holds the raw top component (mod_switch); otherwise U already includes + half (key switch).
    template <bool ADD_HALF, class Base = BaseSrc>
    __global__ void __launch_bounds__(256) moddown_coeff_kernel(const u64 *__restrict__ U, long long u_bs, long long u_ps, const u64 *X,
                                                                 long long x_bs, long long x_ps, u64 *out, long long o_bs, long long o_ps,
                                                                 const Tw *__restrict__ inv_top, Base base, u64 q_top,
                                                                 const PrimeDev *__restrict__ primes, int logn, int Lout, long long total)
    {
        long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over B*2*Lout*n
        if (e >= total)
            return;
        const int idx = static_cast<int>(e & ((1 << logn) - 1));
        const long long row = e >> logn;
        const int i = static_cast<int>(row % Lout), bc = static_cast<int>(row / Lout), b = bc >> 1, c = bc & 1;
        const PrimeDev P = primes[i];
        u64 u = U[b * u_bs + c * u_ps + idx];
        if (ADD_HALF)
            u = csub(u + (q_top >> 1), q_top);
        if (q_top > P.q)
            u = barrett64(u, P.q, P.ratio_hi);
        else
            u = csub(u, P.q);
        u64 t = u + P.q - barrett64(q_top >> 1, P.q, P.ratio_hi); // in (0, 2q)
        u64 x = X[b * x_bs + c * x_ps + (static_cast<long long>(i) << logn) + idx];
        u64 r = mul_shoup(x + P.q2 - t, inv_top[i], P.q);
        r = csub(r + base.get(b, c, i, idx, P.q), P.q);
        out[b * o_bs + c * o_ps + (static_cast<long long>(i) << logn) + idx] = finish(base, b, c, i, logn, idx, r, P);
    }

    struct KsScratch
    {
        u64 *D, *E, *Pp, *U, *K, *T, *C2;
        KsIntScratch I;
    };
    static size_t ks_words_per_ct(const Context &c, size_t L, bool need_c2)
    {
        if (c.ksint_on(L)) // digits + (the key-multiplied tensor component) + the integer path's own buffers
            return c.n * (L + (need_c2 ? L : 0)) + ksint_bytes_per_ct(c, L) / sizeof(u64);
        return c.n * (L + (L + 1) * L + 2 * (L + 1) + 4 + 2 * L + (need_c2 ? L : 0));
    }
    static KsScratch ks_carve(Context &c, size_t L, size_t B, bool need_c2)
    {
        u64 *p = static_cast<u64 *>(c.ensure_scratch(ks_words_per_ct(c, L, need_c2) * B * sizeof(u64) + (c.ksint_on(L) ? ksint_bytes_fixed(c, L) : 0)));
        KsScratch s{};
        s.D = p, p += B * L * c.n;
        if (c.ksint_on(L))
        {
            s.C2 = need_c2 ? p : nullptr;
            p += need_c2 ? B * L * c.n : 0;
            s.I = ksint_carve(c, L, B, p);
            return s;
        }
        s.E = p, p += B * (L + 1) * L * c.n;
        s.Pp = p, p += B * 2 * (L + 1) * c.n;
        s.U = p, p += B * 2 * c.n;
        s.K = p, p += B * 2 * c.n;
        s.T = p, p += B * 2 * L * c.n;
        s.C2 = need_c2 ? p : nullptr;
        return s;
    }
    static size_t ks_chunk(const Context &c, size_t L, size_t batch, bool need_c2)
    {
        size_t per = ks_words_per_ct(c, L, need_c2) * sizeof(u64);
        size_t chunk = std::max<size_t>(1, c.scratch_budget / per);
        if (c.ksint_on(L) && c.scratch_budget > 2 * ksint_bytes_fixed(c, L))
            chunk = std::max<size_t>(1, (c.scratch_budget - ksint_bytes_fixed(c, L)) / per);
        // keep the row counts of a launch (B * (L+1) * L digit rows) far inside int range; element offsets are 64-bit everywhere
        chunk = std::min(chunk, std::max<size_t>(1, (size_t(1) << 22) / ((L + 1) * L)));
        chunk = std::min<size_t>(chunk, 32768);
        chunk = std::min<size_t>(chunk, 65535 / (L + 1)); // (b, I) pairs ride in gridDim.y of the key-switch kernels
        if (c.ks_chunk_max)
            chunk = std::min(chunk, c.ks_chunk_max);
        return std::min(chunk, batch);
    }

    // ---- in-process measurement of the arithmetic ceilings (SURVEY 8d: "two ceilings must be reported") -------------------
    // The path's butterflies and key multiply-accumulates, on registers only (no memory traffic in the loop), at the launch
    // shapes of the two dominant kernels.  Returns warp-level operations per second of the whole device.
    template <int KIND, int THREADS, int MINB>
    __global__ void __launch_bounds__(THREADS, MINB) selftest_bfly_kernel(u64 *d, const PrimeDev *__restrict__ primes, int rounds, int nmask)
    {
        __shared__ Tw ts[256];
        const PrimeDev P = primes[0];
        for (int i = threadIdx.x; i < 256; i += THREADS)
            ts[i] = ldg_tw(P.fwd + ((1 + i) & nmask)); // any table entries will do
        __syncthreads();
        u64 a[8];
#pragma unroll
        for (int j = 0; j < 8; j++)
            a[j] = d[(static_cast<long long>(blockIdx.x) * 8 + j) * THREADS + threadIdx.x];
        const int lane = threadIdx.x & 31;
        for (int r = 0; r < rounds; r++)
        {
            const Tw *t = ts + ((r * 7 + lane) & 127); // per-lane twiddles from shared memory, as the transform kernels read them
            auto tw = [&](int lvl, int kk) { return t[(1 << lvl) - 1 + kk]; };
            if (KIND == 0)
                fwd_regs<3, true>(a, tw, P);
            else if (KIND == 1)
                fwd_regs<3, false>(a, tw, P);
            else
                inv_regs<0, false>(a, tw, P);
            if (KIND == 0 && (r & 3) == 3)
            {
#pragma unroll
                for (int j = 0; j < 8; j++)
                    a[j] = barrett_lazy4(a[j], P.ratio_hi, P.nq); // the guard-free mode reduces once per 16 stages; here once per 12
            }
        }
#pragma unroll
        for (int j = 0; j < 8; j++)
            d[(static_cast<long long>(blockIdx.x) * 8 + j) * THREADS + threadIdx.x] = a[j];
    }
    __global__ void __launch_bounds__(256, 2) selftest_mac_kernel(u64 *d, const PrimeDev *__restrict__ primes, int rounds)
    {
        const PrimeDev P = primes[0];
        u64 a[8], kw[8], lo[8], hi[8];
#pragma unroll
        for (int j = 0; j < 8; j++)
        {
            a[j] = d[(static_cast<long long>(blockIdx.x) * 8 + j) * 256 + threadIdx.x];
            kw[j] = a[j] % P.q;
            lo[j] = hi[j] = 0;
        }
        for (int r = 0; r < rounds; r++)
        {
#pragma unroll
            for (int j = 0; j < 8; j++)
            {
                const u64 x = a[j] + r; // operands change every round so that nothing is hoisted
                mac128_4(lo[j], hi[j], x >> 1, kw[j]); // the kernel's bound: transform outputs below 2^63.25
                mac128_4(lo[(j + 1) & 7], hi[(j + 1) & 7], x >> 1, kw[(j + 3) & 7]);
            }
        }
#pragma unroll
        for (int j = 0; j < 8; j++)
            d[(static_cast<long long>(blockIdx.x) * 8 + j) * 256 + threadIdx.x] = lo[j] ^ hi[j];
    }
    double selftest_rate(Context &c, int kind, cudaStream_t st)
    {
        int sms = 0;
        cuda_check(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c.device), "device attribute");
        const int rounds = 512, nmask = static_cast<int>(c.n - 1);
        const size_t words = static_cast<size_t>(sms) * 3 * 8 * 512;
        u64 *d = static_cast<u64 *>(c.ensure_scratch(words * sizeof(u64)));
        cuda_check(cudaMemsetAsync(d, 0x5a, words * sizeof(u64), st), "memset");
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
        case 0: // forward butterflies at the column-pass launch shape (512 threads x 3 CTAs per SM)
            ops = static_cast<double>(sms) * 3 * 16 * rounds * 12.0;
            if (c.fast_q)
                run([&] { selftest_bfly_kernel<0, 512, 3><<<sms * 3, 512, 0, st>>>(d, c.d_primes.get(), rounds, nmask); });
            else
                run([&] { selftest_bfly_kernel<1, 512, 3><<<sms * 3, 512, 0, st>>>(d, c.d_primes.get(), rounds, nmask); });
            break;
        case 1: // forward butterflies at the fused kernel's launch shape (256 threads x 2 CTAs per SM)
            ops = static_cast<double>(sms) * 2 * 8 * rounds * 12.0;
            if (c.fast_q)
                run([&] { selftest_bfly_kernel<0, 256, 2><<<sms * 2, 256, 0, st>>>(d, c.d_primes.get(), rounds, nmask); });
            else
                run([&] { selftest_bfly_kernel<1, 256, 2><<<sms * 2, 256, 0, st>>>(d, c.d_primes.get(), rounds, nmask); });
            break;
        case 2: // inverse butterflies
            ops = static_cast<double>(sms) * 3 * 16 * rounds * 12.0;
            run([&] { selftest_bfly_kernel<2, 512, 3><<<sms * 3, 512, 0, st>>>(d, c.d_primes.get(), rounds, nmask); });
            break;
        case 3: // key multiply-accumulates of the fused kernel
            ops = static_cast<double>(sms) * 2 * 8 * rounds * 16.0;
            run([&] { selftest_mac_kernel<<<sms * 2, 256, 0, st>>>(d, c.d_primes.get(), rounds); });
            break;
        default: throw std::invalid_argument("unknown selftest");
        }
        float ms = 0;
        cuda_check(cudaEventElapsedTime(&ms, e0, e1), "cudaEventElapsedTime");
        c.stats.pool.push_back(e0);
        c.stats.pool.push_back(e1);
        return ops / (ms * 1e-3);
    }

    size_t keyswitch_chunk(const Context &c, size_t L, size_t batch, bool fused)
    {
        if (c.scheme == 1)
            fused = false; // BFV multiply_relinearize = BEHZ multiply + relinearize
        return ks_chunk(c, L, batch, fused);
    }

    static void check_ks_args(const Context &c, size_t L, const KSwitchKey &key)
    {
        if (c.k < 2)
            throw std::logic_error("keyswitching is not supported by the context"); // evaluator.cpp:2581-2584
        if (L < 1 || L > c.k - 1)
            throw std::invalid_argument("encrypted is not valid for encryption parameters");
        if (key.ctx != &c)
            throw std::invalid_argument("parameter mismatch"); // evaluator.cpp:2587-2590
        if (key.digits < L)
            throw std::invalid_argument("kswitch_keys inner dimension is too small"); // evaluator.cpp:2635-2638
    }

    // BGV: make the top-component INTT also emit K = -U * q_top^-1 mod t
    static void bgv_top(const Context &c, OpTopIntt &op, u64 *K, size_t top)
    {
        op.K = K, op.t = c.t, op.t_ratio = c.t_ratio;
        op.inv_top_mod_t = Tw{ c.inv_q_mod_t[top], sbh::shoup(c.inv_q_mod_t[top], c.t) };
    }

    // ct[b] (= base) += key-switch(target[b]) for a chunk of B ciphertexts; writes out[b][2][L][n].
    //   out_bs = words between consecutive ciphertexts of out (0: the dense [B][2][L][n] slab)
    template <class Base>
    static void key_switch_chunk(Context &c, size_t L, size_t B, const KsScratch &s, Src target, const KSwitchKey &key, Base base,
                                 u64 *out, cudaStream_t st, long long out_bs = 0)
    {
        const int n = static_cast<int>(c.n), Li = static_cast<int>(L), ki = static_cast<int>(c.k);
        const bool ntt_in = (c.scheme != 1), bgv = (c.scheme == 3);
        if (c.ksint_on(L))
        {
            ksint_core(c, L, B, s.I, target, s.D, key, base, out, out_bs, st);
            return;
        }
        Src dsrc = target;
        if (ntt_in)
        {
            OpKsIntt op{ target, s.D, c.logn, Li };
            cuda_check(launch_ntt_inv(op, static_cast<int>(B * L), c.logn, c.d_primes.get(), st, c.stats, "ks_target_intt"), "ks intt");
            dsrc = Src{ s.D, static_cast<long long>(L) * n, nullptr, 0, c.logn };
        }
        const bool fused = c.logn >= 12; // two-pass transforms: fuse the in-block stages with the key multiply-accumulate
        double active_rows = 0;
        {
            // the transforms accept inputs below 4q: skip the digit re-reduction when no digit prime reaches 4x an output prime
            u64 qmax = 0, qmin = ~0ull;
            for (size_t i = 0; i < L; i++)
                qmax = std::max(qmax, c.q[i]), qmin = std::min(qmin, c.q[i]);
            qmin = std::min(qmin, c.q[c.k - 1]);
            const int reduce = (qmax >> 2) >= qmin ? 1 : 0;
            OpKsDigit op{ dsrc, s.E, c.d_primes.get(), c.logn, Li, ki, ntt_in ? 1 : 0, reduce };
            const int active = static_cast<int>(B * (ntt_in ? L * L : (L + 1) * L));
            active_rows = active;
            const bool plain_rows = !reduce && dsrc.perm == nullptr && dsrc.ginv == 0;
            if (fused)
            {
                c.stats.begin("ks_digit_ntt", 1, 16.0 * active * n, st, 0.5 * active * n * (c.logn - kLocalLog));
                switch (c.logn - kLocalLog)
                {
                case 4: launch_ks_digit_col<4>(op, static_cast<int>(B), c.fast_q, plain_rows, c.d_primes.get(), st); break;
                case 5: launch_ks_digit_col<5>(op, static_cast<int>(B), c.fast_q, plain_rows, c.d_primes.get(), st); break;
                case 6: launch_ks_digit_col<6>(op, static_cast<int>(B), c.fast_q, plain_rows, c.d_primes.get(), st); break;
                case 7: launch_ks_digit_col<7>(op, static_cast<int>(B), c.fast_q, plain_rows, c.d_primes.get(), st); break;
                case 8: launch_ks_digit_col<8>(op, static_cast<int>(B), c.fast_q, plain_rows, c.d_primes.get(), st); break;
                case 9: launch_ks_digit_col<9>(op, static_cast<int>(B), c.fast_q, plain_rows, c.d_primes.get(), st); break;
                default: throw std::logic_error("unsupported transform size");
                }
                c.stats.end(st);
                cuda_check(cudaGetLastError(), "ks_digit_col_kernel");
            }
            else
                cuda_check(launch_ntt_fwd(op, static_cast<int>(B * (L + 1) * L), c.logn, c.d_primes.get(), st, c.stats, "ks_digit_ntt", active, c.fast_q),
                           "ks digit ntt");
        }
        // digits in + 2 accumulated components out per (b, I), plus one pass over the key
        const double mac_bytes = 8.0 * n * (static_cast<double>(B) * (L + 1) * (L + 2) + 2.0 * L * (L + 1));
        const bool window = ks_sum_needs_window(c, L);
        if (fused)
        {
            const int na = n >> kLocalLog;
            dim3 grid(static_cast<unsigned>(B * (na / 8)), static_cast<unsigned>(L + 1));
            const bool plain_tgt = target.perm == nullptr && target.ginv == 0;
            auto launch = [&](auto kern) {
                constexpr size_t smem = KsMacSmem::total;
                cuda_check(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)), "smem attr");
                c.stats.begin("ks_local_mac", 0, mac_bytes, st, 0.5 * active_rows * n * kLocalLog, 2.0 * B * (L + 1) * L * n);
                kern<<<grid, 256, smem, st>>>(s.E, target, ntt_in ? 1 : 0, key.d_key.get(), s.Pp, c.d_primes.get(), c.logn, Li, ki, static_cast<int>(B));
            };
            if (c.fast_q) // primes below 2^57: 255 products of lazy operands (below 4q past 200 digits) stay below 2^128
                plain_tgt ? launch(ks_local_mac_kernel<true, true, false>) : launch(ks_local_mac_kernel<true, false, false>);
            else if (window)
                plain_tgt ? launch(ks_local_mac_kernel<false, true, true>) : launch(ks_local_mac_kernel<false, false, true>);
            else
                plain_tgt ? launch(ks_local_mac_kernel<false, true, false>) : launch(ks_local_mac_kernel<false, false, false>);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "ks_local_mac_kernel");
        }
        else
        {
            int threads = std::min(n, 256);
            dim3 grid(static_cast<unsigned>(B), (n + threads - 1) / threads, static_cast<unsigned>(L + 1));
            c.stats.begin("ks_mac", 0, mac_bytes, st, 0, 2.0 * B * (L + 1) * L * n);
            if (window)
                ks_mac_kernel<true><<<grid, threads, 0, st>>>(s.E, target, ntt_in ? 1 : 0, key.d_key.get(), s.Pp, c.d_primes.get(), c.logn, Li, ki);
            else
                ks_mac_kernel<false><<<grid, threads, 0, st>>>(s.E, target, ntt_in ? 1 : 0, key.d_key.get(), s.Pp, c.d_primes.get(), c.logn, Li, ki);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "ks_mac_kernel");
        }
        const long long pp_ps = static_cast<long long>(L + 1) * n, pp_bs = 2 * pp_ps;
        {
            OpTopIntt op{ s.Pp + static_cast<long long>(L) * n, pp_bs, pp_ps, s.U, c.logn, ki - 1 };
            if (bgv)
                bgv_top(c, op, s.K, c.k - 1);
            cuda_check(launch_ntt_inv(op, static_cast<int>(B * 2), c.logn, c.d_primes.get(), st, c.stats, "ks_top_intt"), "ks top intt");
        }
        const Tw *inv_top = c.d_invq.get() + (c.k - 1) * c.k;
        const long long o_ps = static_cast<long long>(L) * n, o_bs = out_bs ? out_bs : 2 * o_ps;
        if (bgv)
        {
            OpModDownFwdBgv<Base> op{ { s.U, s.Pp, pp_bs, pp_ps, s.T, out, o_bs, o_ps, inv_top, base, c.q[c.k - 1], c.logn, Li },
                                      s.K, c.d_qmod.get() + (c.k - 1) * c.k, c.t };
            cuda_check(launch_ntt_fwd(op, static_cast<int>(B * 2 * L), c.logn, c.d_primes.get(), st, c.stats, "ks_moddown_ntt", -1, c.fast_q), "ks moddown ntt");
        }
        else if (ntt_in)
        {
            OpModDownFwd<Base> op{ s.U, s.Pp, pp_bs, pp_ps, s.T, out, o_bs, o_ps, inv_top, base, c.q[c.k - 1], c.logn, Li };
            cuda_check(launch_ntt_fwd(op, static_cast<int>(B * 2 * L), c.logn, c.d_primes.get(), st, c.stats, "ks_moddown_ntt", -1, c.fast_q), "ks moddown ntt");
        }
        else if constexpr (Base::kPlain) // BFV's result is in coefficient form: a plaintext product there is a convolution
            throw std::logic_error("the key switch's plaintext product needs an NTT-form result (CKKS / BGV)");
        else
        {
            OpProdIntt op{ s.Pp, c.logn, Li };
            cuda_check(launch_ntt_inv(op, static_cast<int>(B * 2 * L), c.logn, c.d_primes.get(), st, c.stats, "ks_prod_intt"), "ks prod intt");
            long long total = static_cast<long long>(B) * 2 * L * n;
            c.stats.begin("moddown_coeff", 0, 32.0 * total, st);
            moddown_coeff_kernel<false, Base><<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(
                s.U, 2LL * n, n, s.Pp, pp_bs, pp_ps, out, o_bs, o_ps, inv_top, base, c.q[c.k - 1], c.d_primes.get(), c.logn, Li, total);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "moddown_coeff_kernel");
        }
    }

    void op_relinearize(Context &c, size_t L, size_t batch, const u64 *in3, const KSwitchKey &key, u64 *out2, cudaStream_t st)
    {
        check_ks_args(c, L, key);
        const size_t poly = L * c.n, chunk = ks_chunk(c, L, batch, false);
        for (size_t b0 = 0; b0 < batch; b0 += chunk)
        {
            size_t B = std::min(chunk, batch - b0);
            KsScratch s = ks_carve(c, L, B, false);
            const u64 *in = in3 + b0 * 3 * poly;
            Src target{ in + 2 * poly, static_cast<long long>(3 * poly), nullptr, 0, c.logn };
            BaseSrc base;
            base.s = Src{ in, static_cast<long long>(3 * poly), nullptr, 0, c.logn };
            base.pstride = static_cast<long long>(poly);
            base.present = 1;
            key_switch_chunk(c, L, B, s, target, key, base, out2 + b0 * 2 * poly, st);
        }
    }

    // one step of relinearize_internal's loop (evaluator.cpp:1179-1187) on ciphertexts of any size >= 3:
    // out = in with (c_0, c_1) += key_switch(c_{size-1}); all other polynomials are copied.  out [B][size][L][n], no aliasing.
    void op_relinearize_sized(Context &c, size_t L, size_t size, size_t batch, const u64 *in, const KSwitchKey &key, u64 *out, cudaStream_t st)
    {
        check_ks_args(c, L, key);
        if (size < 3 || size > 16)
            throw std::invalid_argument("invalid ciphertext size");
        const size_t poly = L * c.n, chunk = ks_chunk(c, L, batch, false);
        // polynomials 2 .. size-1 are carried over unchanged
        cuda_check(cudaMemcpy2DAsync(out + 2 * poly, size * poly * sizeof(u64), in + 2 * poly, size * poly * sizeof(u64), (size - 2) * poly * sizeof(u64),
                                     batch, cudaMemcpyDeviceToDevice, st),
                   "relinearize copy");
        for (size_t b0 = 0; b0 < batch; b0 += chunk)
        {
            size_t B = std::min(chunk, batch - b0);
            KsScratch s = ks_carve(c, L, B, false);
            const u64 *src = in + b0 * size * poly;
            Src target{ src + (size - 1) * poly, static_cast<long long>(size * poly), nullptr, 0, c.logn };
            BaseSrc base;
            base.s = Src{ src, static_cast<long long>(size * poly), nullptr, 0, c.logn };
            base.pstride = static_cast<long long>(poly);
            base.present = 1;
            key_switch_chunk(c, L, B, s, target, key, base, out + b0 * size * poly, st, static_cast<long long>(size * poly));
        }
    }

    void op_multiply_relinearize(Context &c, size_t L, size_t batch, const u64 *a, const u64 *b, const KSwitchKey &key, u64 *out2,
                                 cudaStream_t st)
    {
        check_ks_args(c, L, key);
        const size_t poly = L * c.n;
        if (c.scheme == 1)
        {
            // BFV: BEHZ multiply into a size-3 scratch, then relinearize (no fusion across the base conversion)
            const size_t chunk = std::min(batch, std::max<size_t>(1, (size_t(1) << 30) / (3 * poly * sizeof(u64))));
            u64 *tmp = static_cast<u64 *>(c.ensure_aux(chunk * 3 * poly * sizeof(u64)));
            for (size_t b0 = 0; b0 < batch; b0 += chunk)
            {
                size_t B = std::min(chunk, batch - b0);
                op_bfv_multiply(c, L, B, a + b0 * 2 * poly, b + b0 * 2 * poly, tmp, st);
                op_relinearize(c, L, B, tmp, key, out2 + b0 * 2 * poly, st);
            }
            return;
        }
        const size_t chunk = ks_chunk(c, L, batch, true);
        for (size_t b0 = 0; b0 < batch; b0 += chunk)
        {
            size_t B = std::min(chunk, batch - b0);
            KsScratch s = ks_carve(c, L, B, true);
            u64 *o = out2 + b0 * 2 * poly;
            launch_tensor(c, true, L, B, a + b0 * 2 * poly, b + b0 * 2 * poly, o, s.C2, st);
            Src target{ s.C2, static_cast<long long>(poly), nullptr, 0, c.logn };
            BaseSrc base;
            base.s = Src{ o, static_cast<long long>(2 * poly), nullptr, 0, c.logn }; // read-modify-write of (c0, c1)
            base.pstride = static_cast<long long>(poly);
            base.present = 1;
            key_switch_chunk(c, L, B, s, target, key, base, o, st);
        }
    }

    static void check_galois_args(const Context &c, size_t L, uint32_t elt, const KSwitchKey &key)
    {
        check_ks_args(c, L, key);
        if (!(elt & 1) || elt >= 2 * c.n)
            throw std::invalid_argument("Galois element is not valid"); // evaluator.cpp:2424-2427
    }

    // out = apply_galois(in) (Base = BaseSrc), addend + apply_galois(in) (BaseAddSrc) or [addend +] plain * apply_galois(in)
    // (BasePlainSrc, NTT-form plaintexts [P][L][n] with plain_bs words between members: 0 for one plaintext), in chunks of the
    // key-switching scratch
    template <class Base>
    static void galois_chunks(Context &c, size_t L, size_t batch, const u64 *in2, uint32_t elt, const KSwitchKey &key, const u64 *addend2,
                              u64 *out2, cudaStream_t st, const u64 *plain = nullptr, long long plain_bs = 0)
    {
        const size_t poly = L * c.n, chunk = ks_chunk(c, L, batch, false);
        const uint32_t *perm = nullptr;
        uint32_t ginv = 0;
        if (c.scheme == 1)
        {
            u64 gi = 0;
            sbh::invmod(elt, 2 * c.n, gi);
            ginv = static_cast<uint32_t>(gi);
            if (ginv == 1)
                ginv = 0;
        }
        else
            perm = c.galois_table(elt);
        for (size_t b0 = 0; b0 < batch; b0 += chunk)
        {
            size_t B = std::min(chunk, batch - b0);
            KsScratch s = ks_carve(c, L, B, false);
            const u64 *in = in2 + b0 * 2 * poly;
            Src target{ in + poly, static_cast<long long>(2 * poly), perm, ginv, c.logn };
            Base base;
            base.s = Src{ in, static_cast<long long>(2 * poly), perm, ginv, c.logn };
            base.pstride = static_cast<long long>(poly);
            base.c1_zero = 1;
            base.present = 1;
            if constexpr (Base::kAddend)
            {
                base.a = addend2 + b0 * 2 * poly;
                base.a_bs = static_cast<long long>(2 * poly);
                base.a_ps = static_cast<long long>(poly);
            }
            if constexpr (Base::kPlain)
            {
                base.pl = plain + b0 * plain_bs;
                base.p_bs = plain_bs;
            }
            key_switch_chunk(c, L, B, s, target, key, base, out2 + b0 * 2 * poly, st);
        }
    }

    void op_apply_galois(Context &c, size_t L, size_t batch, const u64 *in2, uint32_t elt, const KSwitchKey &key, u64 *out2,
                         cudaStream_t st)
    {
        check_galois_args(c, L, elt, key);
        if (in2 == out2)
            throw std::invalid_argument("apply_galois: in and out must not alias");
        galois_chunks<BaseSrc>(c, L, batch, in2, elt, key, nullptr, out2, st);
    }

    void op_apply_galois_add(Context &c, size_t L, size_t batch, const u64 *in2, uint32_t elt, const KSwitchKey &key, const u64 *addend2,
                             u64 *out2, cudaStream_t st)
    {
        check_galois_args(c, L, elt, key);
        if (in2 == out2)
            throw std::invalid_argument("apply_galois_add: in and out must not alias");
        galois_chunks<BaseAddSrc>(c, L, batch, in2, elt, key, addend2, out2, st);
    }

    void check_rotate_sum_args(const Context &c, size_t L, size_t steps, const uint32_t *elts, const KSwitchKey *const *keys)
    {
        for (size_t j = 0; j < steps; j++)
            check_galois_args(c, L, elts[j], *keys[j]);
    }

    // Each chunk of the key-switching scratch runs every step before the next chunk starts: the temporary is one chunk, not the
    // batch, and every key is read once per chunk and step, as the chained apply_galois calls read it.
    void op_rotate_sum(Context &c, size_t L, size_t batch, const u64 *in2, size_t steps, const uint32_t *elts, const KSwitchKey *const *keys,
                       u64 *out2, cudaStream_t st)
    {
        check_rotate_sum_args(c, L, steps, elts, keys);
        const size_t poly = L * c.n, bytes = 2 * poly * sizeof(u64);
        if (steps == 0)
        {
            if (in2 != out2)
                cuda_check(cudaMemcpyAsync(out2, in2, batch * bytes, cudaMemcpyDeviceToDevice, st), "rotate_sum copy");
            return;
        }
        const size_t chunk = ks_chunk(c, L, batch, false);
        u64 *tmp = static_cast<u64 *>(c.ensure_aux(chunk * bytes));
        for (size_t b0 = 0; b0 < batch; b0 += chunk)
        {
            const size_t B = std::min(chunk, batch - b0);
            const u64 *y = in2 + b0 * 2 * poly;
            u64 *o = out2 + b0 * 2 * poly;
            // y_j goes to o when steps - j is even and to tmp otherwise, so that y_steps ends in o; an input that is o itself
            // and an odd step count start from a copy in tmp
            if (y == o && (steps & 1))
            {
                cuda_check(cudaMemcpyAsync(tmp, y, B * bytes, cudaMemcpyDeviceToDevice, st), "rotate_sum copy");
                y = tmp;
            }
            for (size_t j = 0; j < steps; j++)
            {
                u64 *dst = ((steps - j - 1) & 1) ? tmp : o;
                galois_chunks<BaseAddSrc>(c, L, B, y, elts[j], *keys[j], y, dst, st);
                y = dst;
            }
        }
    }

    // One rotated term of a diagonal sum on a chunk of B ciphertexts (at most one key-switching chunk): out = [addend +] plain *
    // apply_galois(in), with out == addend allowed.  CKKS / BGV (NTT-form plaintexts): one key switch, the product and the addition in
    // its last pass.  BFV: the chain itself through tmp ([B][2][L][n]): apply_galois, then multiply_plain as the reference multiplies
    // a coefficient-form ciphertext (an NTT-form plaintext: to NTT form, dyadic product, back, evaluator.cpp:2005-2010; a
    // coefficient-form one: multiply_plain_normal), then add_many's two-operand fold.
    static void galois_plain_term(Context &c, size_t L, size_t B, const u64 *in2, uint32_t elt, const KSwitchKey &key, bool shared, const u64 *plain,
                                  bool plain_ntt, const u64 *addend2, u64 *out2, u64 *tmp, cudaStream_t st)
    {
        if (c.scheme != 1)
        {
            if (!plain_ntt)
                throw std::logic_error("the key switch's plaintext product takes NTT-form plaintexts");
            const long long pbs = shared ? 0 : static_cast<long long>(L * c.n);
            if (addend2)
                galois_chunks<BasePlainSrc<true>>(c, L, B, in2, elt, key, addend2, out2, st, plain, pbs);
            else
                galois_chunks<BasePlainSrc<false>>(c, L, B, in2, elt, key, nullptr, out2, st, plain, pbs);
            return;
        }
        galois_chunks<BaseSrc>(c, L, B, in2, elt, key, nullptr, tmp, st);
        u64 *dst = addend2 ? tmp : out2;
        if (plain_ntt)
        {
            op_ntt(c, false, L, 2, B, tmp, st);
            op_multiply_plain(c, L, 2, B, shared, tmp, plain, dst, st);
            op_ntt(c, true, L, 2, B, dst, st);
        }
        else
            op_multiply_plain_coeff(c, L, 2, B, shared, false, tmp, plain, dst, st);
        if (addend2)
        {
            const size_t sizes[2] = { 2, 2 };
            const u64 *ops[2] = { addend2, tmp };
            const int modes[1] = { SB200_FOLD_ADD };
            op_add_many(c, L, B, 2, sizes, ops, modes, nullptr, out2, st);
        }
    }

    void op_apply_galois_multiply_plain_add(Context &c, size_t L, size_t batch, const u64 *in2, uint32_t elt, const KSwitchKey &key, bool shared,
                                            const u64 *plain, const u64 *addend2, u64 *out2, cudaStream_t st)
    {
        check_galois_args(c, L, elt, key);
        if (in2 == out2)
            throw std::invalid_argument("apply_galois_multiply_plain_add: in and out must not alias");
        const size_t poly = L * c.n;
        if (c.scheme != 1)
        {
            galois_chunks<BasePlainSrc<true>>(c, L, batch, in2, elt, key, addend2, out2, st, plain, shared ? 0 : static_cast<long long>(poly));
            return;
        }
        const size_t chunk = ks_chunk(c, L, batch, false);
        u64 *tmp = static_cast<u64 *>(c.ensure_aux(chunk * 2 * poly * sizeof(u64)));
        for (size_t b0 = 0; b0 < batch; b0 += chunk)
        {
            const size_t B = std::min(chunk, batch - b0);
            galois_plain_term(c, L, B, in2 + b0 * 2 * poly, elt, key, shared, shared ? plain : plain + b0 * poly, true, addend2 + b0 * 2 * poly,
                              out2 + b0 * 2 * poly, tmp, st);
        }
    }

    void check_diagonal_sum_args(const Context &c, size_t L, size_t count, const uint32_t *elts, const KSwitchKey *const *keys)
    {
        for (size_t t = 0; t < count; t++)
            if (elts[t] != 1)
                check_galois_args(c, L, elts[t], *keys[t]);
    }

    // Identity terms (element 1) first, all in one multiply_plain_sum pass that initialises out; then each rotated term accumulates
    // into out through galois_plain_term (the first one writes out when there is no identity term).  Each chunk of the key-switching
    // scratch runs every term before the next chunk starts, so every key is read once per chunk and term, as the chain reads it.
    // Temporaries: none for CKKS and for BGV with NTT-form plaintexts.  BGV's coefficient-form plaintexts are lifted and transformed
    // once into the aux arena (the reference's transform_to_ntt_inplace of each plaintext): the shared ones before the first chunk,
    // the per-member ones of each chunk with it.  BFV's chain goes through one chunk-sized ciphertext there.
    void op_diagonal_sum(Context &c, size_t L, size_t batch, const u64 *in2, size_t count, const uint32_t *elts, const KSwitchKey *const *keys,
                         const size_t *plain_counts, const u64 *const *plains, bool plain_ntt, u64 *out2, cudaStream_t st)
    {
        check_diagonal_sum_args(c, L, count, elts, keys);
        if (in2 == out2)
            throw std::invalid_argument("diagonal_sum: in and out must not alias");
        const size_t poly = L * c.n, pw = plain_ntt ? poly : c.n, chunk = ks_chunk(c, L, batch, false);
        const bool bfv = c.scheme == 1, lift = c.scheme == 3 && !plain_ntt;
        std::vector<size_t> ident, rot;
        for (size_t t = 0; t < count; t++)
            (elts[t] == 1 ? ident : rot).push_back(t);
        // aux: [BFV's chunk of ciphertexts][the lifted shared plaintexts][the lifted per-member plaintexts of one chunk]
        const size_t tmp_words = bfv && !rot.empty() ? chunk * 2 * poly : 0;
        size_t shared_words = 0, member_words = 0;
        for (size_t t = 0; t < count && lift; t++)
            (plain_counts[t] == 1 ? shared_words : member_words) += (plain_counts[t] == 1 ? 1 : chunk) * poly;
        const size_t aux_words = tmp_words + shared_words + member_words;
        u64 *aux = aux_words ? static_cast<u64 *>(c.ensure_aux(aux_words * sizeof(u64))) : nullptr;
        std::vector<const u64 *> p(count), id_cts(ident.size()), id_plains(ident.size());
        std::vector<size_t> id_sizes(ident.size(), 2), id_counts(ident.size());
        if (lift)
        {
            u64 *w = aux + tmp_words;
            for (size_t t = 0; t < count; t++)
                if (plain_counts[t] == 1)
                {
                    op_plain_to_ntt(c, L, 1, plains[t], nullptr, w, st);
                    p[t] = w, w += poly;
                }
        }
        for (size_t b0 = 0; b0 < batch; b0 += chunk)
        {
            const size_t B = std::min(chunk, batch - b0);
            const u64 *x = in2 + b0 * 2 * poly;
            u64 *o = out2 + b0 * 2 * poly;
            u64 *w = aux ? aux + tmp_words + shared_words : nullptr;
            for (size_t t = 0; t < count; t++)
            {
                if (plain_counts[t] == 1)
                {
                    if (!lift)
                        p[t] = plains[t];
                    continue;
                }
                p[t] = plains[t] + b0 * pw;
                if (lift)
                {
                    op_plain_to_ntt(c, L, B, p[t], nullptr, w, st);
                    p[t] = w, w += B * poly;
                }
            }
            const bool pn = plain_ntt || lift;
            for (size_t u = 0; u < ident.size(); u++)
            {
                id_cts[u] = x;
                id_plains[u] = p[ident[u]];
                id_counts[u] = plain_counts[ident[u]] == 1 ? 1 : B;
            }
            if (!ident.empty())
                op_multiply_plain_sum(c, L, B, ident.size(), 1, id_sizes.data(), id_cts.data(), id_counts.data(), id_plains.data(), !bfv, pn,
                                      nullptr, nullptr, &o, st);
            bool first = ident.empty();
            for (size_t t : rot)
            {
                galois_plain_term(c, L, B, x, elts[t], *keys[t], plain_counts[t] == 1, p[t], pn, first ? nullptr : o, o, aux, st);
                first = false;
            }
        }
    }

    // ---- is_data_valid_for (valcheck.cpp: every coefficient below its modulus), for the checked wire-format load ----
    __global__ void __launch_bounds__(256) range_check_kernel(const u64 *__restrict__ d, const PrimeDev *__restrict__ primes, int logn, int L,
                                                               long long total, int *flag)
    {
        long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
        if (e < total && d[e] >= primes[static_cast<int>((e >> logn) % L)].q)
            atomicOr(flag, 1);
    }
    bool op_residues_in_range(Context &c, size_t L, size_t rows, const u64 *d, cudaStream_t st)
    {
        if (!c.d_flag)
        {
            c.d_flag = DevBuf<int>(1);
            c.table_bytes += c.d_flag.bytes();
        }
        int *flag = c.d_flag.get(); // a word of its own: the aux arena may be in use by an operation in flight on another stream
        cuda_check(cudaMemsetAsync(flag, 0, sizeof(int), st), "memset");
        const size_t step = std::max<size_t>(1, (size_t(1) << 31) / c.n);
        for (size_t r0 = 0; r0 < rows; r0 += step * L)
        {
            const long long total = static_cast<long long>(std::min(step * L, rows - r0) * c.n);
            range_check_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(d + r0 * c.n, c.d_primes.get(), c.logn, static_cast<int>(L),
                                                                                            total, flag);
            cuda_check(cudaGetLastError(), "range_check_kernel");
            c.stats.launches++;
        }
        int h = 0;
        cuda_check(cudaMemcpyAsync(&h, flag, sizeof(int), cudaMemcpyDeviceToHost, st), "flag D2H");
        cuda_check(cudaStreamSynchronize(st), "synchronize");
        return h == 0;
    }

    // ------------------------------------------------------------------------- rescale / modulus switching ----
    // `polys` = batch * size polynomials, each [L][n], contiguous: every polynomial of a ciphertext is treated alike
    // (rns.cpp:830-901 is applied per polynomial, evaluator.cpp:1263-1280), so any ciphertext size works.  The kernels decode a
    // row as (pair, component) with pair stride = 2 * polynomial stride, i.e. plain polynomial index * stride.
    void op_rescale(Context &c, size_t L, size_t polys, const u64 *in, u64 *out, cudaStream_t st)
    {
        if (c.scheme != 2)
            throw std::invalid_argument("unsupported operation for scheme type"); // evaluator.cpp:1533
        if (L < 2 || L > c.k)
            throw std::invalid_argument("end of modulus switching chain reached"); // evaluator.cpp:1521
        const int n = static_cast<int>(c.n);
        const size_t Lout = L - 1;
        const size_t per = (1 + Lout) * c.n * sizeof(u64);
        size_t chunk = std::min(polys, std::max<size_t>(1, c.scratch_budget / per));
        chunk = std::min<size_t>(chunk, std::max<size_t>(1, (size_t(1) << 30) / (L * c.n)));
        for (size_t p0 = 0; p0 < polys; p0 += chunk)
        {
            size_t P = std::min(chunk, polys - p0);
            u64 *U = static_cast<u64 *>(c.ensure_scratch(per * P));
            u64 *T = U + P * c.n;
            const u64 *src = in + p0 * L * c.n;
            const long long i_ps = static_cast<long long>(L) * n, i_bs = 2 * i_ps;
            OpTopIntt top{ src + (L - 1) * c.n, i_bs, i_ps, U, c.logn, static_cast<int>(L - 1) };
            cuda_check(launch_ntt_inv(top, static_cast<int>(P), c.logn, c.d_primes.get(), st, c.stats, "rescale_top_intt"), "rescale intt");
            BaseSrc none;
            const long long o_ps = static_cast<long long>(Lout) * n, o_bs = 2 * o_ps;
            OpModDownFwd<> op{ U, src, i_bs, i_ps, T, out + p0 * Lout * c.n, o_bs, o_ps, c.d_invq.get() + (L - 1) * c.k, none, c.q[L - 1],
                             c.logn, static_cast<int>(Lout) };
            cuda_check(launch_ntt_fwd(op, static_cast<int>(P * Lout), c.logn, c.d_primes.get(), st, c.stats, "rescale_ntt", -1, c.fast_q), "rescale ntt");
        }
    }

    void op_mod_switch(Context &c, size_t L, size_t polys, const u64 *in, u64 *out, cudaStream_t st)
    {
        if (L < 2 || L > c.k)
            throw std::invalid_argument("end of modulus switching chain reached");
        const size_t Lout = L - 1;
        if (c.scheme == 2)
        {
            // CKKS mod_switch_drop_to_next: drop the last RNS component (evaluator.cpp:1296-1358)
            cuda_check(cudaMemcpy2DAsync(out, Lout * c.n * sizeof(u64), in, L * c.n * sizeof(u64), Lout * c.n * sizeof(u64), polys,
                                         cudaMemcpyDeviceToDevice, st),
                       "mod_switch copy");
            return;
        }
        const int n = static_cast<int>(c.n);
        if (c.scheme == 3)
        {
            // BGV: mod_t_and_divide_q_last_ntt_inplace on every polynomial (evaluator.cpp:1263-1267, rns.cpp:1193-1236)
            const size_t per = (2 + Lout) * c.n * sizeof(u64);
            size_t chunk = std::min(polys, std::max<size_t>(1, c.scratch_budget / per));
            chunk = std::min<size_t>(chunk, std::max<size_t>(1, (size_t(1) << 30) / (L * c.n)));
            for (size_t p0 = 0; p0 < polys; p0 += chunk)
            {
                size_t P = std::min(chunk, polys - p0);
                u64 *U = static_cast<u64 *>(c.ensure_scratch(per * P));
                u64 *K = U + P * c.n, *T = K + P * c.n;
                const u64 *src = in + p0 * L * c.n;
                const long long i_ps = static_cast<long long>(L) * n, i_bs = 2 * i_ps;
                OpTopIntt top{ src + (L - 1) * c.n, i_bs, i_ps, U, c.logn, static_cast<int>(L - 1) };
                bgv_top(c, top, K, L - 1);
                cuda_check(launch_ntt_inv(top, static_cast<int>(P), c.logn, c.d_primes.get(), st, c.stats, "modswitch_top_intt"), "mod switch intt");
                BaseSrc none;
                const long long o_ps = static_cast<long long>(Lout) * n, o_bs = 2 * o_ps;
                OpModDownFwdBgv<> op{ { U, src, i_bs, i_ps, T, out + p0 * Lout * c.n, o_bs, o_ps, c.d_invq.get() + (L - 1) * c.k, none, c.q[L - 1],
                                      c.logn, static_cast<int>(Lout) },
                                    K, c.d_qmod.get() + (L - 1) * c.k, c.t };
                cuda_check(launch_ntt_fwd(op, static_cast<int>(P * Lout), c.logn, c.d_primes.get(), st, c.stats, "modswitch_ntt", -1, c.fast_q),
                           "mod switch ntt");
            }
            return;
        }
        const long long i_ps = static_cast<long long>(L) * n, o_ps = static_cast<long long>(Lout) * n;
        const size_t step = std::max<size_t>(1, (size_t(1) << 31) / (L * c.n));
        BaseSrc none;
        for (size_t p0 = 0; p0 < polys; p0 += step)
        {
            size_t P = std::min(step, polys - p0);
            const u64 *src = in + p0 * L * c.n;
            long long total = static_cast<long long>(P) * Lout * n;
            c.stats.begin("moddown_coeff", 0, 24.0 * total, st);
            moddown_coeff_kernel<true><<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(
                src + (L - 1) * c.n, 2 * i_ps, i_ps, src, 2 * i_ps, i_ps, out + p0 * Lout * c.n, 2 * o_ps, o_ps,
                c.d_invq.get() + (L - 1) * c.k, none, c.q[L - 1], c.d_primes.get(), c.logn, static_cast<int>(Lout), total);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "moddown_coeff_kernel");
        }
    }
} // namespace sb
