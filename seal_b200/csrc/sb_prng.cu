// seal_b200/csrc/sb_prng.cu -- the PRNG-driven pieces on the device: seed-compressed ciphertexts expanded at load time (SURVEY 8f
// rank 3) and symmetric-key encryption of zero (the producer of those ciphertexts; second half of this file).
//
// A ciphertext that comes out of a symmetric-key encryption is saved with its first polynomial only; the second one is
// uniformly random and is carried as the 64-byte seed of the PRNG that produced it (Serializable<Ciphertext>,
// ciphertext.cpp:325-352).  Ciphertext::load re-creates it with Ciphertext::expand_seed (ciphertext.cpp:118-150) ->
// sample_poly_uniform (util/rlwe.cpp:104-132) on a Blake2xbPRNG (randomgen.cpp:204-214).  Doing that here halves the bytes a
// fresh ciphertext moves over PCIe.  What is reproduced, bit for bit:
//   * the PRNG stream: buffer b (4096 bytes) = BLAKE2Xb(out 4096, in = 64-bit counter b, key = seed)  -- RFC 7693 BLAKE2b with
//     the BLAKE2X parameter block: a keyed root hash over the counter, then 64 output blocks B_i = BLAKE2b(root) whose
//     parameter block carries node_offset = i and xof_length = 4096 (util/blake2xb.c); or, when the stream names prng_type
//     shake256, buffer b = SHAKE256(seed || b, 4096 bytes) (Shake256PRNG, randomgen.cpp:216-227; FIPS 202);
//   * sample_poly_uniform: the first L*n words of the stream fill the polynomial; every word >= max_multiple of its prime
//     (rejection sampling for uniformity) is replaced, in coefficient order, by the next words of the stream; the survivors are
//     reduced modulo the prime.
// Parallel schedule: one thread per 64-byte output block generates a BLAKE2Xb stream (root hash recomputed per thread: 3
// compressions per block), one thread per 4096-byte buffer a SHAKE256 stream (31 permutations in sequence; prng_stream picks), one CTA per ciphertext lists the rejected coefficients in order (two passes with a block-wide scan), one thread per
// ciphertext consumes the replacement words (a few thousand sequential steps at n = 65536, 31 primes), one streaming kernel reduces.
#include "sb_engine.cuh"

namespace sb
{
    namespace
    {
        __constant__ u64 c_iv[8] = { 0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                                     0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull };
        __constant__ unsigned char c_sigma[12][16] = {
            { 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15 }, { 14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3 },
            { 11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4 }, { 7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8 },
            { 9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13 }, { 2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9 },
            { 12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11 }, { 13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10 },
            { 6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5 }, { 10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0 },
            { 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15 }, { 14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3 }
        };
        __device__ __forceinline__ u64 rotr64(u64 v, int s)
        {
            return (v >> s) | (v << (64 - s));
        }
        // BLAKE2b compression function F (RFC 7693 3.2): h updated with one 128-byte block m, byte counter t, last-block flag
        __device__ void blake2b_compress(u64 (&h)[8], const u64 (&m)[16], u64 t, bool last)
        {
            u64 v[16];
#pragma unroll
            for (int i = 0; i < 8; i++)
                v[i] = h[i], v[i + 8] = c_iv[i];
            v[12] ^= t;
            if (last)
                v[14] = ~v[14];
#define SB_G(a, b, c, d, x, y)                        \
    v[a] += v[b] + (x), v[d] = rotr64(v[d] ^ v[a], 32); \
    v[c] += v[d], v[b] = rotr64(v[b] ^ v[c], 24);       \
    v[a] += v[b] + (y), v[d] = rotr64(v[d] ^ v[a], 16); \
    v[c] += v[d], v[b] = rotr64(v[b] ^ v[c], 63);
            for (int r = 0; r < 12; r++)
            {
                const unsigned char *s = c_sigma[r];
                SB_G(0, 4, 8, 12, m[s[0]], m[s[1]])
                SB_G(1, 5, 9, 13, m[s[2]], m[s[3]])
                SB_G(2, 6, 10, 14, m[s[4]], m[s[5]])
                SB_G(3, 7, 11, 15, m[s[6]], m[s[7]])
                SB_G(0, 5, 10, 15, m[s[8]], m[s[9]])
                SB_G(1, 6, 11, 12, m[s[10]], m[s[11]])
                SB_G(2, 7, 8, 13, m[s[12]], m[s[13]])
                SB_G(3, 4, 9, 14, m[s[14]], m[s[15]])
            }
#undef SB_G
#pragma unroll
            for (int i = 0; i < 8; i++)
                h[i] ^= v[i] ^ v[i + 8];
        }

        constexpr unsigned kXof = 4096;       // UniformRandomGenerator::buffer_size_ (randomgen.h:391)
        constexpr int kWordsPerBuffer = kXof / 8;

        // thread = one 64-byte output block of one PRNG buffer of one ciphertext: W[b][buffer*512 + block*8 .. +8)
        __global__ void __launch_bounds__(128) blake2xb_stream_kernel(const u64 *__restrict__ seeds, u64 *__restrict__ W, long long words_per_ct,
                                                                       long long blocks_per_ct, long long total_blocks)
        {
            const long long g = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
            if (g >= total_blocks)
                return;
            const long long b = g / blocks_per_ct, blk = g % blocks_per_ct;
            const u64 counter = static_cast<u64>(blk >> 6); // buffer index = Blake2xbPRNG::counter_ at its refill
            const unsigned node = static_cast<unsigned>(blk & 63);
            u64 h[8], m[16];
            // root: keyed BLAKE2b, digest 64, key length 64, fanout 1, depth 1, xof_length 4096 (blake2xb_init_key)
#pragma unroll
            for (int i = 0; i < 8; i++)
                h[i] = c_iv[i];
            h[0] ^= 64ull | (64ull << 8) | (1ull << 16) | (1ull << 24);
            h[1] ^= static_cast<u64>(kXof) << 32; // bytes 8..11 node_offset = 0, bytes 12..15 xof_length
#pragma unroll
            for (int i = 0; i < 8; i++)
                m[i] = seeds[b * 8 + i], m[i + 8] = 0; // the key, padded to one block
            blake2b_compress(h, m, 128, false);
#pragma unroll
            for (int i = 0; i < 16; i++)
                m[i] = 0;
            m[0] = counter; // the message: the 8-byte counter
            blake2b_compress(h, m, 128 + 8, true);
            // output block `node`: unkeyed BLAKE2b over the 64-byte root with digest 64, fanout 0, depth 0, leaf_length 64,
            // node_offset = node, xof_length 4096, node_depth 0, inner_length 64 (blake2xb_final)
            u64 o[8];
#pragma unroll
            for (int i = 0; i < 8; i++)
                o[i] = c_iv[i], m[i] = h[i], m[i + 8] = 0;
            o[0] ^= 64ull | (64ull << 32);
            o[1] ^= static_cast<u64>(node) | (static_cast<u64>(kXof) << 32);
            o[2] ^= 64ull << 8; // byte 16 node_depth = 0, byte 17 inner_length = 64
            blake2b_compress(o, m, 64, true);
            u64 *dst = W + b * words_per_ct + blk * 8;
#pragma unroll
            for (int i = 0; i < 8; i++)
                dst[i] = o[i];
        }

        // Keccak-f[1600] (FIPS 202 section 3), lanes a[x + 5 y].  Every 64-bit rotation is two funnel shifts of the 32-bit halves
        // (the shift amounts are constants once the round body is unrolled); chi's a ^ (~b & c) is one three-input logic op per half.
        __constant__ u64 c_keccak_rc[24] = {
            0x0000000000000001ull, 0x0000000000008082ull, 0x800000000000808Aull, 0x8000000080008000ull, 0x000000000000808Bull,
            0x0000000080000001ull, 0x8000000080008081ull, 0x8000000000008009ull, 0x000000000000008Aull, 0x0000000000000088ull,
            0x0000000080008009ull, 0x000000008000000Aull, 0x000000008000808Bull, 0x800000000000008Bull, 0x8000000000008089ull,
            0x8000000000008003ull, 0x8000000000008002ull, 0x8000000000000080ull, 0x000000000000800Aull, 0x800000008000000Aull,
            0x8000000080008081ull, 0x8000000000008080ull, 0x0000000080000001ull, 0x8000000080008008ull
        };
        __device__ __forceinline__ u64 rotl64(u64 v, int s)
        {
            const unsigned lo = static_cast<unsigned>(v), hi = static_cast<unsigned>(v >> 32);
            unsigned rl, rh;
            if (s == 0)
                return v;
            if (s < 32)
                rh = __funnelshift_l(lo, hi, s), rl = __funnelshift_l(hi, lo, s);
            else
                rh = __funnelshift_l(hi, lo, s - 32), rl = __funnelshift_l(lo, hi, s - 32);
            return (static_cast<u64>(rh) << 32) | rl;
        }
        __device__ __forceinline__ void keccak_f1600(u64 (&a)[25])
        {
            // rho offsets r[x + 5 y] (FIPS 202 table 2)
            constexpr int rho[25] = { 0, 1, 62, 28, 27, 36, 44, 6, 55, 20, 3, 10, 43, 25, 39, 41, 45, 15, 21, 8, 18, 2, 61, 56, 14 };
#pragma unroll 1
            for (int r = 0; r < 24; r++)
            {
                u64 c[5], d[5], t[25];
#pragma unroll
                for (int x = 0; x < 5; x++) // theta
                    c[x] = a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20];
#pragma unroll
                for (int x = 0; x < 5; x++)
                    d[x] = c[(x + 4) % 5] ^ rotl64(c[(x + 1) % 5], 1);
#pragma unroll
                for (int y = 0; y < 5; y++) // rho and pi: lane (x, y) moves to (y, 2x + 3y)
#pragma unroll
                    for (int x = 0; x < 5; x++)
                        t[y + 5 * ((2 * x + 3 * y) % 5)] = rotl64(a[x + 5 * y] ^ d[x], rho[x + 5 * y]);
#pragma unroll
                for (int y = 0; y < 5; y++) // chi
#pragma unroll
                    for (int x = 0; x < 5; x++)
                        a[x + 5 * y] = t[x + 5 * y] ^ (~t[(x + 1) % 5 + 5 * y] & t[(x + 2) % 5 + 5 * y]);
                a[0] ^= c_keccak_rc[r]; // iota
            }
        }

        // thread = one PRNG buffer of one ciphertext, Shake256PRNG::refill_buffer (randomgen.cpp:216-227): W[b][buffer*512 .. +512) =
        // SHAKE256(seed (64 bytes) || buffer index (8 bytes, little-endian), 4096 bytes).  The 72-byte message fits the 136-byte rate
        // block: padding 0x1F at byte 72 and 0x80 at byte 135.  4096 bytes = 30 full squeezes of 17 lanes + 2 lanes of the 31st.
        __global__ void __launch_bounds__(128) shake256_stream_kernel(const u64 *__restrict__ seeds, u64 *__restrict__ W, long long words_per_ct,
                                                                       long long buffers_per_ct, long long total_buffers)
        {
            const long long g = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
            if (g >= total_buffers)
                return;
            const long long b = g / buffers_per_ct, buf = g % buffers_per_ct;
            u64 a[25];
#pragma unroll
            for (int i = 0; i < 8; i++)
                a[i] = seeds[b * 8 + i];
            a[8] = static_cast<u64>(buf);
            a[9] = 0x1Full;
#pragma unroll
            for (int i = 10; i < 25; i++)
                a[i] = 0;
            a[16] = 0x80ull << 56;
            u64 *dst = W + b * words_per_ct + buf * kWordsPerBuffer;
#pragma unroll 1
            for (int s = 0; s < 30; s++, dst += 17)
            {
                keccak_f1600(a);
#pragma unroll
                for (int i = 0; i < 17; i++)
                    dst[i] = a[i];
            }
            keccak_f1600(a);
            dst[0] = a[0], dst[1] = a[1];
        }

        // one CTA per ciphertext: list the rejected coefficients in order, then let one thread walk the replacement words
        __global__ void __launch_bounds__(1024) seed_reject_kernel(u64 *__restrict__ W, long long words_per_ct, const u64 *__restrict__ max_mult,
                                                                   unsigned *__restrict__ list, long long list_cap, int logn, int L, int *overflow)
        {
            __shared__ unsigned cnt[1024];
            __shared__ unsigned total;
            const int b = blockIdx.x, t = threadIdx.x;
            u64 *w = W + b * words_per_ct;
            unsigned *mine = list + b * list_cap;
            const long long need = static_cast<long long>(L) << logn;
            const long long seg = (need + 1023) / 1024, lo = t * seg, hi = lo + seg < need ? lo + seg : need;
            unsigned c = 0;
            for (long long i = lo; i < hi; i++)
                c += w[i] >= max_mult[i >> logn];
            cnt[t] = c;
            __syncthreads();
            if (t == 0)
            {
                unsigned run = 0;
                for (int i = 0; i < 1024; i++)
                {
                    const unsigned v = cnt[i];
                    cnt[i] = run;
                    run += v;
                }
                total = run;
            }
            __syncthreads();
            unsigned at = cnt[t];
            if (total > list_cap)
            {
                if (t == 0)
                    atomicOr(overflow, 1);
                return;
            }
            for (long long i = lo; i < hi; i++)
                if (w[i] >= max_mult[i >> logn])
                    mine[at++] = static_cast<unsigned>(i);
            __syncthreads();
            if (t != 0)
                return;
            // util/rlwe.cpp:121-128: while (rand >= max_multiple) take the next word of the stream
            long long r = need;
            for (unsigned k = 0; k < total; k++)
            {
                const unsigned idx = mine[k];
                const u64 mm = max_mult[idx >> logn];
                u64 v;
                do
                {
                    if (r >= words_per_ct)
                    {
                        atomicOr(overflow, 1);
                        return;
                    }
                    v = w[r++];
                } while (v >= mm);
                w[idx] = v;
            }
        }

        // barrett_reduce_64 of the accepted words into the second polynomial of each ciphertext
        __global__ void __launch_bounds__(256) seed_reduce_kernel(const u64 *__restrict__ W, long long words_per_ct, u64 *__restrict__ out,
                                                                  const long long *__restrict__ dst_off, const PrimeDev *__restrict__ primes,
                                                                  int logn, int L, long long total)
        {
            const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
            if (e >= total)
                return;
            const long long need = static_cast<long long>(L) << logn, b = e / need, i = e % need;
            const PrimeDev P = primes[static_cast<int>(i >> logn)];
            out[dst_off[b] + i] = barrett64(W[b * words_per_ct + i], P.q, P.ratio_hi);
        }
    } // namespace

    void check_prng_type(int type)
    {
        if (type != kPrngBlake2xb && type != kPrngShake256)
            throw std::invalid_argument("prng_type is invalid"); // randomgen.h:29-36: unknown (0) makes no PRNG
    }

    // The one place that knows the PRNG formats: W[b][0, words_per_ct) = the output stream of ciphertext b's PRNG, whose type
    // types[b] (host) is SEAL's prng_type and whose seed is d_seeds[b] (device, 8 words); words_per_ct is a whole number of 4096-byte
    // buffers.  Every consumer reads the stream as one sequence of bytes, whichever PRNG made it.  A run of equal types is one
    // launch; its profile entry is names[0] for blake2xb and names[1] for shake256 (string literals: the profile keeps the pointers).
    static void prng_stream(Context &c, const char *const (&names)[2], const int *types, size_t B, const u64 *d_seeds, u64 *W, long long words_per_ct,
                            cudaStream_t st)
    {
        const long long buffers_per_ct = words_per_ct / kWordsPerBuffer;
        for (size_t b0 = 0, b1; b0 < B; b0 = b1)
        {
            check_prng_type(types[b0]);
            for (b1 = b0 + 1; b1 < B && types[b1] == types[b0];)
                b1++;
            const long long nb = static_cast<long long>(b1 - b0);
            const u64 *seeds = d_seeds + b0 * 8;
            u64 *w = W + b0 * words_per_ct;
            if (types[b0] == kPrngBlake2xb)
            {
                const long long blocks_per_ct = words_per_ct / 8, total_blocks = blocks_per_ct * nb;
                c.stats.begin(names[0], 0, 8.0 * nb * words_per_ct, st);
                blake2xb_stream_kernel<<<static_cast<unsigned>((total_blocks + 127) / 128), 128, 0, st>>>(seeds, w, words_per_ct, blocks_per_ct,
                                                                                                         total_blocks);
                c.stats.end(st);
                cuda_check(cudaGetLastError(), "blake2xb_stream_kernel");
            }
            else
            {
                const long long total_buffers = buffers_per_ct * nb;
                c.stats.begin(names[1], 0, 8.0 * nb * words_per_ct, st);
                shake256_stream_kernel<<<static_cast<unsigned>((total_buffers + 127) / 128), 128, 0, st>>>(seeds, w, words_per_ct, buffers_per_ct,
                                                                                                          total_buffers);
                c.stats.end(st);
                cuda_check(cudaGetLastError(), "shake256_stream_kernel");
            }
        }
    }

    // seeds: [B][8] words (prng_seed_type), on the host or (seeds_on_device) already on the device; types: [B] host prng_type of each
    // seed; dst_off: [B] host word offsets into d_out of the polynomial to fill ([L][n])
    static void expand_impl(Context &c, size_t L, size_t B, const u64 *seeds, bool seeds_on_device, const int *types, const long long *h_dst_off,
                            u64 *d_out, cudaStream_t st)
    {
        if (!B)
            return;
        if (L < 1 || L > c.k)
            throw std::invalid_argument("encrypted is not valid for encryption parameters");
        for (size_t b = 0; b < B; b++)
            check_prng_type(types[b]);
        const long long need = static_cast<long long>(L) * c.n;
        // rejection probability of prime j = (2^64 - max_multiple_j) / 2^64; spare stream words: twice the expectation + a margin
        std::vector<u64> mm(L);
        double expect = 0;
        for (size_t j = 0; j < L; j++)
        {
            const u64 max_random = ~0ull;
            mm[j] = max_random - (max_random % c.q[j]) - 1;
            expect += static_cast<double>(c.n) * (static_cast<double>(max_random - mm[j]) / 18446744073709551616.0);
        }
        for (int attempt = 0; attempt < 4; attempt++)
        {
            const long long spare = static_cast<long long>((2.0 * expect + 2048.0) * (1 << attempt));
            const long long buffers = (need + spare + kWordsPerBuffer - 1) / kWordsPerBuffer, words_per_ct = buffers * kWordsPerBuffer;
            const long long list_cap = spare;
            // scratch: stream words, rejection lists, per-ciphertext seeds / offsets / thresholds, overflow flag
            const size_t bytes = B * words_per_ct * sizeof(u64) + B * list_cap * sizeof(unsigned) + (B * 8 + B + L) * sizeof(u64) + 64;
            u64 *W = static_cast<u64 *>(c.ensure_scratch(bytes));
            unsigned *list = reinterpret_cast<unsigned *>(W + B * words_per_ct);
            u64 *d_seeds = reinterpret_cast<u64 *>(reinterpret_cast<unsigned char *>(list) + ((B * list_cap * sizeof(unsigned) + 15) / 16) * 16);
            long long *d_off = reinterpret_cast<long long *>(d_seeds + B * 8);
            u64 *d_mm = reinterpret_cast<u64 *>(d_off + B);
            int *d_flag = reinterpret_cast<int *>(d_mm + L);
            cuda_check(cudaMemcpyAsync(d_seeds, seeds, B * 8 * sizeof(u64), seeds_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st),
                       "seeds");
            cuda_check(cudaMemcpyAsync(d_off, h_dst_off, B * sizeof(long long), cudaMemcpyHostToDevice, st), "offsets H2D");
            cuda_check(cudaMemcpyAsync(d_mm, mm.data(), L * sizeof(u64), cudaMemcpyHostToDevice, st), "thresholds H2D");
            cuda_check(cudaMemsetAsync(d_flag, 0, sizeof(int), st), "memset");
            prng_stream(c, { "seed_stream", "seed_stream:shake256" }, types, B, d_seeds, W, words_per_ct, st);
            c.stats.begin("seed_reject", 0, 16.0 * B * need, st);
            seed_reject_kernel<<<static_cast<unsigned>(B), 1024, 0, st>>>(W, words_per_ct, d_mm, list, list_cap, c.logn, static_cast<int>(L), d_flag);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "seed_reject_kernel");
            int flag = 0;
            cuda_check(cudaMemcpyAsync(&flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st), "flag D2H");
            cuda_check(cudaStreamSynchronize(st), "synchronize"); // also: the host arrays above may now go out of scope
            if (flag)
                continue; // more rejections than spare words (probability far below 2^-40 at the first attempt): take more
            const long long total = need * static_cast<long long>(B);
            c.stats.begin("seed_reduce", 0, 16.0 * total, st);
            seed_reduce_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(W, words_per_ct, d_out, d_off, c.d_primes.get(), c.logn,
                                                                                           static_cast<int>(L), total);
            c.stats.end(st);
            cuda_check(cudaGetLastError(), "seed_reduce_kernel");
            return;
        }
        throw std::logic_error("seed expansion ran out of random words");
    }

    void op_expand_seeded(Context &c, size_t L, size_t B, const u64 *h_seeds, const int *h_types, const long long *h_dst_off, u64 *d_out,
                          cudaStream_t st)
    {
        expand_impl(c, L, B, h_seeds, false, h_types, h_dst_off, d_out, st);
    }

    // ------------------------------------------------------------------------------------------------------------------------------
    // Encryptor::encrypt_zero_symmetric (encryptor.cpp:168-173 -> util/rlwe.cpp:264-408) for a batch of ciphertexts.
    // Per ciphertext, from ONE bootstrap PRNG (Blake2xb of a fresh 64-byte seed):
    //   bytes [0, 64)          the public seed P: c_1 = sample_poly_uniform(Blake2xb(P))            (rlwe.cpp:298-324)
    //   bytes [64 + 6i, +6)    the noise coefficient i: hw(x0, x1, x2 & 31) - hw(x3, x4, x5 & 31)    (sample_poly_cbd, rlwe.cpp:73-102)
    //   c_0 = -(c_1 s + e)  [CKKS: everything in NTT form;  BGV: -(c_1 s + t e), NTT form;  BFV: coefficient form, see below]
    // BFV ciphertexts are in coefficient form (rlwe.cpp:314-324, 347-372): when the seed is kept (Serializable<Ciphertext>) the sampled
    // polynomial IS c_1 and a transformed copy is multiplied with the key; otherwise the sample is taken as NTT(c_1).
    // The uniform polynomial reuses the expansion above with the seeds left on the device; the noise costs 6 bytes per coefficient and
    // is re-read per prime from L2; the transforms are the library's own (op_ntt).
    namespace
    {
        // the plaintexts an encryption adds to c_0, one per ciphertext (both pointers null: an encryption of zero)
        struct EncPlain
        {
            const u64 *ntt = nullptr;     // CKKS: [B][L][n], NTT form at the level
            const u64 *coeff = nullptr;   // BFV / BGV: [B][n], words < t
            const Tw *delta = nullptr;    // BFV: [L] floor(q / t) mod q_j
            u64 t = 0, t_ratio_lo = 0, t_ratio_hi = 0, q_mod_t = 0;
        };
        __device__ __forceinline__ int cbd_noise(const unsigned char *boot, long long i)
        {
            const unsigned short *x = reinterpret_cast<const unsigned short *>(boot + 64 + 6 * i); // 64 + 6 i is even
            const unsigned w0 = x[0], w1 = x[1], w2 = x[2];
            const unsigned lo = (w0 | (w1 << 16)) & 0x1FFFFFu, hi = ((w1 >> 8) | (w2 << 8)) & 0x1FFFFFu;
            return __popc(lo) - __popc(hi);
        }
        __device__ __forceinline__ u64 neg_sum(u64 a, u64 b, u64 q) // -(a + b) mod q, operands < q
        {
            u64 v = a + b;
            v -= v >= q ? q : 0;
            return v ? q - v : 0;
        }
        // MODE 0  tmp = m_j e                 (CKKS m = 1 / BGV m = t mod q_j; transformed afterwards)
        //         BGV with a plaintext: tmp = t e - lift(p)  (the transform is linear with canonical outputs, so MODE 1 then
        //         gives -(s c_1 + NTT(t e)) + NTT(lift(p)), the reference's c_0 word for word: encryptor.cpp:245-336)
        // MODE 1  c_0 = -(s c_1 + tmp)        (NTT form schemes); CKKS with a plaintext: + p (add_poly_coeffmod, encryptor.cpp:232-235)
        // MODE 2  tmp = c_1                   (BFV with the seed kept: the copy that gets transformed)
        // MODE 3  tmp = s tmp
        // MODE 4  c_0 = -(tmp + e)
        // MODE 5  c_0 = s c_1                 (BFV without the seed: both polynomials are inverse-transformed afterwards)
        // MODE 6  c_0 = -(c_0 + e)
        //         MODES 4 / 6, BFV with a plaintext: + round(q p / t) (multiply_add_plain_with_scaling_variant, encryptor.cpp:210-213)
        // MODE 7  MODE 1, plus on row j = digit of each digit's c_0: (q_{k-1} mod q_j) s'_j  (a key-switching key, L = k)
        template <int MODE>
        __global__ void __launch_bounds__(256) enc_kernel(u64 *__restrict__ out, u64 *__restrict__ tmp, const u64 *__restrict__ sk,
                                                          const unsigned char *__restrict__ boot, long long boot_bytes, const u64 *__restrict__ mult,
                                                          KsFactor ks, EncPlain pl, const PrimeDev *__restrict__ primes, int logn, int L,
                                                          long long total)
        {
            const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over B * L * n
            if (e >= total)
                return;
            const long long poly = static_cast<long long>(L) << logn, b = e / poly, r = e % poly;
            const int j = static_cast<int>(r >> logn);
            const long long i = r & ((1ll << logn) - 1);
            const PrimeDev P = primes[j];
            u64 *c0 = out + b * 2 * poly + r, *c1 = c0 + poly;
            u64 noise = 0;
            if (MODE == 0 || MODE == 4 || MODE == 6)
            {
                const int v = cbd_noise(boot + b * boot_bytes, i);
                noise = v >= 0 ? static_cast<u64>(v) : P.q - static_cast<u64>(-v);
            }
            if (MODE == 0)
            {
                u64 v = mult ? mulmod_barrett(noise, mult[j], P) : noise;
                if (pl.coeff)
                    v = csub(v + P.q - plain_lift(pl.coeff[(b << logn) + i], pl.t, mult[j], P), P.q); // BGV: mult = t mod q_j
                tmp[e] = v;
            }
            else if (MODE == 1)
            {
                u64 v = neg_sum(mulmod_barrett(sk[r], *c1, P), tmp[e], P.q);
                if (pl.ntt)
                    v = csub(v + pl.ntt[e], P.q);
                *c0 = v;
            }
            else if (MODE == 2)
                tmp[e] = *c1;
            else if (MODE == 3)
                tmp[e] = mulmod_barrett(sk[r], tmp[e], P);
            else if (MODE == 4 || MODE == 6)
            {
                u64 v = neg_sum(MODE == 4 ? tmp[e] : *c0, noise, P.q);
                if (pl.coeff)
                {
                    const u64 m = pl.coeff[(b << logn) + i];
                    v = csub(v + bfv_plain_scaled(m, bfv_plain_fix(m, pl.t, pl.t_ratio_lo, pl.t_ratio_hi, pl.q_mod_t), pl.t, pl.delta[j], P), P.q);
                }
                *c0 = v;
            }
            else if (MODE == 5)
                *c0 = mulmod_barrett(sk[r], *c1, P);
            else
            {
                u64 v = neg_sum(mulmod_barrett(sk[r], *c1, P), tmp[e], P.q);
                if (j == ks.digit0 + b)
                {
                    // keygenerator.cpp:349-356: barrett_reduce_64(q_{k-1}, q_j) s'_j, added mod q_j
                    const u64 factor = barrett64(primes[L - 1].q, P.q, P.ratio_hi);
                    const u64 s_new = ks.new_key[(static_cast<long long>(j) << logn) + (ks.perm ? ks.perm[i] : i)];
                    v = csub(v + mulmod_barrett(factor, s_new, P), P.q);
                }
                *c0 = v;
            }
        }
    } // namespace

    // util::encrypt_zero_symmetric (util/rlwe.cpp:264-408) at the level with L primes (1..k, the key level included), checks done by
    // the callers.  h_boot_seeds [B][8]: the seeds of the bootstrap PRNGs (one per ciphertext); d_out [B][2][L][n]; is_ntt_form: the
    // reference's argument of that name (true: NTT form for every scheme, as KeyGenerator asks; false: BFV's coefficient form);
    // h_public_seeds: nullptr or [B][8], receives the seed c_1 of each ciphertext expands from (what Serializable<Ciphertext> stores);
    // ks: nullptr, or the factor term that turns ciphertext b into digit ks->digit0 + b of a key-switching key (L = k, NTT form);
    // pl: the plaintexts added to c_0 (Encryptor::encrypt_internal, encryptor.cpp:176-340), or none
    static void encrypt_zero_symmetric_impl(Context &c, const SecretKey &sk, size_t L, size_t B, const u64 *h_boot_seeds, int boot_prng,
                                            int ct_prng, bool is_ntt_form, bool save_seed, const KsFactor *ks, const EncPlain &pl, u64 *d_out,
                                            u64 *h_public_seeds, cudaStream_t st)
    {
        const long long poly = static_cast<long long>(L) * c.n, total = poly * static_cast<long long>(B);
        // bootstrap stream: whole PRNG buffers covering 64 + 6 n bytes
        const long long boot_words = ((64 + 6 * static_cast<long long>(c.n) + kXof - 1) / kXof) * kWordsPerBuffer, boot_bytes = boot_words * 8;
        const size_t bytes = B * boot_bytes + static_cast<size_t>(total) * sizeof(u64) + (B * 8 + B * 8 + L) * sizeof(u64);
        u64 *Wb = static_cast<u64 *>(c.ensure_aux(bytes));
        u64 *tmp = Wb + B * boot_words, *d_boot_seeds = tmp + total, *d_pub = d_boot_seeds + B * 8, *d_mult = d_pub + B * 8;
        cuda_check(cudaMemcpyAsync(d_boot_seeds, h_boot_seeds, B * 8 * sizeof(u64), cudaMemcpyHostToDevice, st), "bootstrap seeds H2D");
        const u64 *mult = nullptr;
        std::vector<u64> h_mult;
        if (c.scheme == 3 /* BGV */)
        {
            h_mult.resize(L);
            for (size_t j = 0; j < L; j++)
                h_mult[j] = c.t % c.q[j];
            cuda_check(cudaMemcpyAsync(d_mult, h_mult.data(), L * sizeof(u64), cudaMemcpyHostToDevice, st), "t mod q H2D");
            mult = d_mult;
        }
        const std::vector<int> boot_types(B, boot_prng), ct_types(B, ct_prng);
        prng_stream(c, { "enc_bootstrap_stream", "enc_bootstrap_stream:shake256" }, boot_types.data(), B, d_boot_seeds, Wb, boot_words, st);
        cuda_check(cudaMemcpy2DAsync(d_pub, 64, Wb, boot_bytes, 64, B, cudaMemcpyDeviceToDevice, st), "public seeds");
        std::vector<long long> off(B);
        for (size_t b = 0; b < B; b++)
            off[b] = static_cast<long long>(b) * 2 * poly + poly;
        expand_impl(c, L, B, d_pub, true, ct_types.data(), off.data(), d_out, st); // c_1 (synchronises the stream: the host vectors above are free)
        if (h_public_seeds)
            cuda_check(cudaMemcpyAsync(h_public_seeds, d_pub, B * 8 * sizeof(u64), cudaMemcpyDeviceToHost, st), "public seeds D2H");
        const unsigned grid = static_cast<unsigned>((total + 255) / 256);
        const unsigned char *boot = reinterpret_cast<const unsigned char *>(Wb);
        const u64 *s = sk.d_pow.get(); // s^1, [k][n] at the key level: the first L rows are the level's primes
        const int logn = c.logn, Li = static_cast<int>(L);
        const KsFactor f = ks ? *ks : KsFactor{};
#define SB_ENC(MODE, name)                                                                                           \
    c.stats.begin(name, 0, 24.0 * total, st);                                                                         \
    enc_kernel<MODE><<<grid, 256, 0, st>>>(d_out, tmp, s, boot, boot_bytes, mult, f, pl, c.d_primes.get(), logn, Li, total); \
    c.stats.end(st);                                                                                                  \
    cuda_check(cudaGetLastError(), name);
        if (is_ntt_form)
        {
            SB_ENC(0, "enc_noise")
            op_ntt(c, false, L, 1, B, tmp, st);
            if (ks)
            {
                SB_ENC(7, "enc_combine:kswitch")
            }
            else
            {
                SB_ENC(1, "enc_combine")
            }
        }
        else if (save_seed)
        {
            SB_ENC(2, "enc_copy")
            op_ntt(c, false, L, 1, B, tmp, st);
            SB_ENC(3, "enc_mul_key")
            op_ntt(c, true, L, 1, B, tmp, st);
            SB_ENC(4, "enc_combine")
        }
        else
        {
            SB_ENC(5, "enc_mul_key")
            op_ntt(c, true, L, 2, B, d_out, st);
            SB_ENC(6, "enc_combine")
        }
#undef SB_ENC
        c.wipe_aux(st); // bootstrap stream and noise: with c_0 they give c_1 s (util/rlwe.cpp:292: clear-on-destruction pool)
        if (h_public_seeds)
            cuda_check(cudaStreamSynchronize(st), "synchronize");
    }

    // ciphertexts per chunk of a symmetric encryption at the level with L primes: per ciphertext the noise / product polynomial (aux
    // arena) and the c_1 stream (scratch arena, expand_impl), plus the bootstrap stream, within the scratch budget
    static size_t enc_symmetric_chunk(const Context &c, size_t L, size_t B)
    {
        const size_t per = 2 * L * c.n * sizeof(u64) + 6 * c.n + kXof + 64;
        return std::max<size_t>(1, std::min(B, c.scratch_budget / per));
    }

    static void check_encrypt_symmetric(const Context &c, const SecretKey &sk, size_t L)
    {
        if (L < 1 || L > c.k || (c.k > 1 && L == c.k))
            throw std::invalid_argument("parms_id is not valid for encryption parameters");
        if (!sk.d_pow || sk.ctx != &c)
            throw std::invalid_argument("secret key is not valid for encryption parameters");
    }

    // the batch in chunks: each chunk is one encrypt_zero_symmetric_impl, which wipes its noise and streams.  The words do not depend
    // on the chunk size: every ciphertext has its own bootstrap seed.
    static void encrypt_symmetric_chunked(Context &c, const SecretKey &sk, size_t L, size_t B, const EncPlain &pl, const u64 *h_boot_seeds,
                                          int boot_prng, int ct_prng, bool save_seed, u64 *d_out, u64 *h_public_seeds, cudaStream_t st)
    {
        const size_t chunk = enc_symmetric_chunk(c, L, B), poly = L * c.n;
        for (size_t b0 = 0; b0 < B; b0 += chunk)
        {
            EncPlain p = pl;
            if (p.ntt)
                p.ntt += b0 * poly;
            if (p.coeff)
                p.coeff += b0 * c.n;
            encrypt_zero_symmetric_impl(c, sk, L, std::min(chunk, B - b0), h_boot_seeds + b0 * 8, boot_prng, ct_prng, c.scheme != 1 /* CKKS, BGV */,
                                        save_seed, nullptr, p, d_out + b0 * 2 * poly, h_public_seeds ? h_public_seeds + b0 * 8 : nullptr, st);
        }
    }

    // h_boot_seeds [B][8]: the seeds of the bootstrap PRNGs (one fresh seed per ciphertext); d_out [B][2][L][n];
    // h_public_seeds: nullptr or [B][8], receives the seed c_1 of each ciphertext expands from (what Serializable<Ciphertext> stores)
    void op_encrypt_zero_symmetric(Context &c, const SecretKey &sk, size_t L, size_t B, const u64 *h_boot_seeds, int boot_prng, int ct_prng,
                                   bool save_seed, u64 *d_out, u64 *h_public_seeds, cudaStream_t st)
    {
        check_prng_type(boot_prng);
        check_prng_type(ct_prng);
        if (!B)
            return;
        check_encrypt_symmetric(c, sk, L);
        encrypt_symmetric_chunked(c, sk, L, B, EncPlain{}, h_boot_seeds, boot_prng, ct_prng, save_seed, d_out, h_public_seeds, st);
    }

    // the level check of a plaintext encryption (BFV / BGV encrypt at first_parms_id, encryptor.cpp:209, :241) and its plaintext terms
    static EncPlain encrypt_plain(Context &c, size_t L, const u64 *d_plain)
    {
        EncPlain pl;
        if (c.scheme == 2 /* CKKS */)
        {
            pl.ntt = d_plain;
            return pl;
        }
        if (L != (c.k > 1 ? c.k - 1 : 1))
            throw std::invalid_argument("BFV and BGV encrypt at the first level");
        const Context::PlainLevel &lv = plain_level(c, L);
        pl.coeff = d_plain;
        pl.delta = lv.d_delta.get();
        pl.t = c.t, pl.t_ratio_lo = c.t_ratio_lo, pl.t_ratio_hi = c.t_ratio_hi, pl.q_mod_t = lv.q_mod_t;
        return pl;
    }

    void op_encrypt_symmetric(Context &c, const SecretKey &sk, size_t L, size_t B, const u64 *d_plain, const u64 *h_boot_seeds, int boot_prng,
                              int ct_prng, bool save_seed, u64 *d_out, u64 *h_public_seeds, cudaStream_t st)
    {
        check_prng_type(boot_prng);
        check_prng_type(ct_prng);
        if (!B)
            return;
        check_encrypt_symmetric(c, sk, L);
        const EncPlain pl = encrypt_plain(c, L, d_plain);
        encrypt_symmetric_chunked(c, sk, L, B, pl, h_boot_seeds, boot_prng, ct_prng, save_seed, d_out, h_public_seeds, st);
    }

    // ------------------------------------------------------------------------------------------------------------------------------
    // KeyGenerator (keygenerator.cpp:96-120, 327-360): the public key and every key-switching key are key-level symmetric encryptions
    // of zero in NTT form (is_ntt_form = true for every scheme, BFV included), drawn from one bootstrap PRNG each.
    static void check_key(const Context &c, const SecretKey &sk, int boot_prng, int ct_prng)
    {
        check_prng_type(boot_prng);
        check_prng_type(ct_prng);
        if (!sk.d_pow || sk.ctx != &c)
            throw std::invalid_argument("secret key is not valid for encryption parameters");
    }

    void op_generate_public_key(Context &c, const SecretKey &sk, int boot_prng, int ct_prng, const u64 *h_boot_seed, u64 *d_out, cudaStream_t st,
                                u64 *h_public_seed)
    {
        check_key(c, sk, boot_prng, ct_prng);
        encrypt_zero_symmetric_impl(c, sk, c.k, 1, h_boot_seed, boot_prng, ct_prng, true, false, nullptr, EncPlain{}, d_out, h_public_seed, st);
    }

    // generate_one_kswitch_key: digit j = encrypt_zero_symmetric at the key level + (q_{k-1} mod q_j) s'_j on row j of c_0, with
    // s' = s^2 (relinearization, the key array of compute_secret_key_array) or s seen through the NTT-form Galois permutation
    // (apply_galois_ntt, galois.cpp:148-160), which the combine kernel reads in place: the permuted key is never stored.  The digits
    // are cut into chunks by the scratch budget; each chunk is one batch of encryptions and wipes its noise and streams.  With
    // h_public_seeds, each chunk's public seeds are in place and its digits complete when on_chunk(d0, count) is called.
    void op_generate_kswitch_key(Context &c, SecretKey &sk, uint32_t galois_elt, int boot_prng, int ct_prng, const u64 *h_boot_seeds, u64 *d_out,
                                 cudaStream_t st, u64 *h_public_seeds, const std::function<void(size_t, size_t)> &on_chunk)
    {
        if (galois_elt && (!(galois_elt & 1) || galois_elt >= 2 * c.n))
            throw std::invalid_argument("Galois element is not valid"); // keygenerator.cpp:195-199
        if (c.k < 2)
            throw std::logic_error("keyswitching is not supported by the context"); // keygenerator.cpp:329-332
        check_key(c, sk, boot_prng, ct_prng);
        KsFactor f{};
        if (galois_elt)
            f.new_key = sk.d_pow.get(), f.perm = c.galois_table(galois_elt);
        else
        {
            ensure_key_powers(c, sk, 2, st);
            f.new_key = sk.d_pow.get() + c.k * c.n;
        }
        const size_t digits = c.k - 1, poly = c.k * c.n;
        const size_t chunk = enc_symmetric_chunk(c, c.k, digits);
        for (size_t d0 = 0; d0 < digits; d0 += chunk)
        {
            f.digit0 = static_cast<long long>(d0);
            const size_t cnt = std::min(chunk, digits - d0);
            encrypt_zero_symmetric_impl(c, sk, c.k, cnt, h_boot_seeds + d0 * 8, boot_prng, ct_prng, true, false, &f, EncPlain{},
                                        d_out + d0 * 2 * poly, h_public_seeds ? h_public_seeds + d0 * 8 : nullptr, st);
            if (on_chunk)
                on_chunk(d0, cnt);
        }
    }

    // ------------------------------------------------------------------------------------------------------------------------------
    // Encryptor::encrypt_zero with a public key (encryptor.cpp:88-174 -> util::encrypt_zero_asymmetric, util/rlwe.cpp:184-276).
    // One PRNG per ciphertext yields, in order: the ternary polynomial u -- one 32-bit word r per coefficient mapped to (r * 3) >> 32
    // (std::uniform_int_distribution<uint64_t>(0, 2) over a 32-bit generator in libstdc++ >= 11: Lemire's method, redraw only for
    // r == 0) -- then the noise polynomials e_0, e_1 (6 bytes per coefficient each).  c_j = pk_j u + e_j (BGV: t e_j) is formed one
    // level above the requested one (L + 1 primes, the level's prev_context_data) and divided down by that level's last prime with
    // the evaluator's own kernels (CKKS: op_rescale, BFV / BGV: op_mod_switch); at the key level (L == k) it is returned as sampled.
    // A redraw shifts everything behind it by one word: the parallel kernel only counts zero words, and a one-thread-per-ciphertext
    // kernel re-walks the (probability 2^-32 per coefficient) ciphertexts that had one.
    namespace
    {
        __device__ __forceinline__ void ternary_store(u64 *__restrict__ u, long long b, long long i, unsigned r, const PrimeDev *__restrict__ primes,
                                                      int logn, int Lp)
        {
            const u64 v = (static_cast<u64>(r) * 3u) >> 32;
            u64 *dst = u + ((b * Lp) << logn) + i;
            for (int j = 0; j < Lp; j++)
                dst[static_cast<long long>(j) << logn] = v + (v == 0 ? primes[j].q : 0) - 1; // rlwe.cpp:32-37
        }
        __global__ void __launch_bounds__(256) enc_ternary_kernel(const u64 *__restrict__ W, long long words_per_ct, u64 *__restrict__ u,
                                                                  unsigned *__restrict__ pos, const PrimeDev *__restrict__ primes, int logn, int Lp,
                                                                  long long total)
        {
            const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over B * n
            if (e >= total)
                return;
            const long long b = e >> logn, i = e & ((1ll << logn) - 1);
            const unsigned r = reinterpret_cast<const unsigned *>(W + b * words_per_ct)[i];
            if (r == 0)
                atomicAdd(pos + b, 1u); // pos[b] starts at n: anything else marks the ciphertext for the sequential walk
            ternary_store(u, b, i, r, primes, logn, Lp);
        }
        __global__ void enc_ternary_fix_kernel(const u64 *__restrict__ W, long long words_per_ct, u64 *__restrict__ u, unsigned *__restrict__ pos,
                                               const PrimeDev *__restrict__ primes, int logn, int Lp, int *overflow)
        {
            const long long b = blockIdx.x, n = 1ll << logn;
            if (threadIdx.x != 0 || pos[b] == static_cast<unsigned>(n))
                return;
            const unsigned *w = reinterpret_cast<const unsigned *>(W + b * words_per_ct);
            const long long cap = words_per_ct * 2;
            long long p = 0;
            for (long long i = 0; i < n; i++)
            {
                unsigned r;
                do
                {
                    if (p >= cap)
                    {
                        atomicOr(overflow, 1);
                        return;
                    }
                    r = w[p++];
                } while (r == 0);
                ternary_store(u, b, i, r, primes, logn, Lp);
            }
            pos[b] = static_cast<unsigned>(p);
        }
        // MODE 0  T_p = m_j e_p                  (CKKS / BGV: transformed afterwards)
        // MODE 1  T_p = u pk_p + T_p             (CKKS / BGV)
        // MODE 2  T_p = u pk_p                   (BFV: inverse-transformed afterwards)
        // MODE 3  T_p = T_p + e_p                (BFV)
        template <int MODE>
        __global__ void __launch_bounds__(256) enc_pk_kernel(u64 *__restrict__ T, const u64 *__restrict__ u, const u64 *__restrict__ pk, long long pk_poly,
                                                             const u64 *__restrict__ W, long long words_per_ct, const unsigned *__restrict__ pos,
                                                             const u64 *__restrict__ mult, const PrimeDev *__restrict__ primes, int logn, int Lp,
                                                             long long total)
        {
            const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; // over B * 2 * Lp * n
            if (e >= total)
                return;
            const long long n = 1ll << logn, poly = static_cast<long long>(Lp) << logn;
            const long long b = e / (2 * poly), rem = e % (2 * poly), p = rem / poly, r = rem % poly;
            const int j = static_cast<int>(r >> logn);
            const long long i = r & (n - 1);
            const PrimeDev P = primes[j];
            u64 noise = 0;
            if (MODE == 0 || MODE == 3)
            {
                // the noise bytes start behind the ternary words: byte 4 pos[b]; polynomial p, coefficient i at + 6 (p n + i);
                // cbd_noise reads from its argument + 64 (the symmetric layout), hence the - 64
                const unsigned char *base = reinterpret_cast<const unsigned char *>(W + b * words_per_ct) + 4ll * pos[b] - 64;
                const int v = cbd_noise(base, p * n + i);
                noise = v >= 0 ? static_cast<u64>(v) : P.q - static_cast<u64>(-v);
            }
            if (MODE == 0)
                T[e] = mult ? mulmod_barrett(noise, mult[j], P) : noise;
            else
            {
                u64 v = 0;
                if (MODE == 1 || MODE == 2)
                    v = mulmod_barrett(u[b * poly + r], pk[p * pk_poly + r], P);
                if (MODE == 1)
                    v += T[e];
                if (MODE == 3)
                    v = T[e] + noise;
                T[e] = v >= P.q ? v - P.q : v;
            }
        }
    } // namespace

    void public_key_create(Context &c, const u64 *h_pk, PublicKey &out)
    {
        out.d_key = DevBuf<u64>(2 * c.k * c.n);
        out.ctx = &c;
        cuda_check(cudaMemcpy(out.d_key.get(), h_pk, out.d_key.bytes(), cudaMemcpyHostToDevice), "upload public key");
        if (!op_residues_in_range(c, c.k, 2 * c.k, out.d_key.get(), nullptr))
            throw std::invalid_argument("public key is not valid for encryption parameters");
    }

    // stream words per ciphertext: 4 n bytes of ternary words + 12 n bytes of noise + spare words for redraws, in whole PRNG buffers
    static long long asym_stream_words(const Context &c)
    {
        return ((16 * static_cast<long long>(c.n) + 256 + kXof - 1) / kXof) * kWordsPerBuffer;
    }

    // one chunk of op_encrypt_zero_asymmetric, checks done by the caller
    static void encrypt_zero_asymmetric_impl(Context &c, const PublicKey &pk, size_t L, size_t B, const u64 *h_seeds, int prng, u64 *d_out,
                                             cudaStream_t st)
    {
        const size_t Lp = L < c.k ? L + 1 : L;
        const long long n = static_cast<long long>(c.n), poly = static_cast<long long>(Lp) * n, total1 = static_cast<long long>(B) * poly;
        const long long words = asym_stream_words(c);
        const size_t bytes = (B * words + static_cast<size_t>(total1) * 3 + B * 8 + Lp) * sizeof(u64) + (B + 4) * sizeof(unsigned);
        u64 *W = static_cast<u64 *>(c.ensure_aux(bytes));
        u64 *U = W + B * words, *T = U + total1, *d_seeds = T + 2 * total1, *d_mult = d_seeds + B * 8;
        unsigned *d_pos = reinterpret_cast<unsigned *>(d_mult + Lp);
        int *d_over = reinterpret_cast<int *>(d_pos + B);
        u64 *dst = Lp == L ? d_out : T;
        cuda_check(cudaMemcpyAsync(d_seeds, h_seeds, B * 8 * sizeof(u64), cudaMemcpyHostToDevice, st), "seeds H2D");
        std::vector<unsigned> h_pos(B, static_cast<unsigned>(n));
        cuda_check(cudaMemcpyAsync(d_pos, h_pos.data(), B * sizeof(unsigned), cudaMemcpyHostToDevice, st), "positions H2D");
        cuda_check(cudaMemsetAsync(d_over, 0, sizeof(int), st), "memset");
        const u64 *mult = nullptr;
        std::vector<u64> h_mult;
        if (c.scheme == 3 /* BGV */)
        {
            h_mult.resize(Lp);
            for (size_t j = 0; j < Lp; j++)
                h_mult[j] = c.t % c.q[j];
            cuda_check(cudaMemcpyAsync(d_mult, h_mult.data(), Lp * sizeof(u64), cudaMemcpyHostToDevice, st), "t mod q H2D");
            mult = d_mult;
        }
        const std::vector<int> types(B, prng);
        prng_stream(c, { "enc_stream", "enc_stream:shake256" }, types.data(), B, d_seeds, W, words, st);
        const long long bn = static_cast<long long>(B) * n;
        const int logn = c.logn, Lpi = static_cast<int>(Lp);
        c.stats.begin("enc_ternary", 0, (4.0 + 8.0 * Lp) * bn, st);
        enc_ternary_kernel<<<static_cast<unsigned>((bn + 255) / 256), 256, 0, st>>>(W, words, U, d_pos, c.d_primes.get(), logn, Lpi, bn);
        enc_ternary_fix_kernel<<<static_cast<unsigned>(B), 32, 0, st>>>(W, words, U, d_pos, c.d_primes.get(), logn, Lpi, d_over);
        c.stats.end(st);
        cuda_check(cudaGetLastError(), "enc_ternary_kernel");
        op_ntt(c, false, Lp, 1, B, U, st);
        const long long total2 = 2 * total1, pk_poly = static_cast<long long>(c.k) * n;
        const unsigned grid = static_cast<unsigned>((total2 + 255) / 256);
#define SB_ENC(MODE, name)                                                                                                          \
    c.stats.begin(name, 0, 24.0 * total2, st);                                                                                       \
    enc_pk_kernel<MODE><<<grid, 256, 0, st>>>(dst, U, pk.d_key.get(), pk_poly, W, words, d_pos, mult, c.d_primes.get(), logn, Lpi, total2);      \
    c.stats.end(st);                                                                                                                 \
    cuda_check(cudaGetLastError(), name);
        if (c.scheme != 1 /* CKKS, BGV */)
        {
            SB_ENC(0, "enc_noise")
            op_ntt(c, false, Lp, 2, B, dst, st);
            SB_ENC(1, "enc_combine")
        }
        else
        {
            SB_ENC(2, "enc_mul_key")
            op_ntt(c, true, Lp, 2, B, dst, st);
            SB_ENC(3, "enc_combine")
        }
#undef SB_ENC
        int over = 0;
        cuda_check(cudaMemcpyAsync(&over, d_over, sizeof(int), cudaMemcpyDeviceToHost, st), "flag D2H");
        cuda_check(cudaStreamSynchronize(st), "synchronize"); // also: the host vectors above may now go out of scope
        if (over)
            throw std::logic_error("ternary sampling ran out of random words");
        if (Lp != L)
        {
            // Encryptor::encrypt_zero_internal (encryptor.cpp:125-161): switch down to the requested level
            if (c.scheme == 2)
                op_rescale(c, Lp, 2 * B, T, d_out, st);
            else
                op_mod_switch(c, Lp, 2 * B, T, d_out, st);
        }
        c.wipe_aux(st); // u, the noise and the PRNG stream (util/rlwe.cpp:195: clear-on-destruction pool)
    }

    static void check_encrypt_asymmetric(const Context &c, const PublicKey &pk, size_t L)
    {
        if (L < 1 || L > c.k)
            throw std::invalid_argument("parms_id is not valid for encryption parameters");
        if (!pk.d_key || pk.ctx != &c)
            throw std::invalid_argument("public key is not valid for encryption parameters");
    }

    // the batch in chunks within the scratch budget (per ciphertext: the PRNG stream, u and the two sampled polynomials, one level
    // above); each chunk wipes its streams.  The words do not depend on the chunk size: every ciphertext has its own seed.
    static void encrypt_zero_asymmetric_chunked(Context &c, const PublicKey &pk, size_t L, size_t B, const u64 *h_seeds, int prng, u64 *d_out,
                                                cudaStream_t st)
    {
        const size_t Lp = L < c.k ? L + 1 : L;
        const size_t per = (static_cast<size_t>(asym_stream_words(c)) + 3 * Lp * c.n + 8) * sizeof(u64) + sizeof(unsigned);
        const size_t chunk = std::max<size_t>(1, std::min(B, c.scratch_budget / per)), poly = L * c.n;
        for (size_t b0 = 0; b0 < B; b0 += chunk)
            encrypt_zero_asymmetric_impl(c, pk, L, std::min(chunk, B - b0), h_seeds + b0 * 8, prng, d_out + b0 * 2 * poly, st);
    }

    // h_seeds [B][8]: the seed of each ciphertext's PRNG; d_out [B][2][L][n] at the level with L primes (L == k: the key level)
    void op_encrypt_zero_asymmetric(Context &c, const PublicKey &pk, size_t L, size_t B, const u64 *h_seeds, int prng, u64 *d_out, cudaStream_t st)
    {
        check_prng_type(prng);
        if (!B)
            return;
        check_encrypt_asymmetric(c, pk, L);
        encrypt_zero_asymmetric_chunked(c, pk, L, B, h_seeds, prng, d_out, st);
    }

    // Encryptor(public key)::encrypt (encryptor.cpp:176-340): the plaintexts are added to c_0 once the sample has been divided down,
    // by the evaluator's add_plain code in one pass over the batch (BGV: its lift-and-transform, then the add)
    void op_encrypt_asymmetric(Context &c, const PublicKey &pk, size_t L, size_t B, const u64 *d_plain, const u64 *h_seeds, int prng, u64 *d_out,
                               cudaStream_t st)
    {
        check_prng_type(prng);
        if (!B)
            return;
        check_encrypt_asymmetric(c, pk, L);
        encrypt_plain(c, L, d_plain); // the level check, before any launch
        encrypt_zero_asymmetric_chunked(c, pk, L, B, h_seeds, prng, d_out, st);
        if (c.scheme == 2)
            op_add_plain_ntt(c, L, 2, B, false, false, d_out, d_plain, d_out, st);
        else
            op_add_plain_coeff(c, L, 2, B, false, false, d_out, d_plain, nullptr, d_out, st);
    }
} // namespace sb
