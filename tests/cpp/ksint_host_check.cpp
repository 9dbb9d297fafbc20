// tests/cpp/ksint_host_check.cpp -- CPU check of the tables sbh::build_ksint produces for the integer key-switching path
// (seal_b200/csrc/sb_ksint.cu): the transforms are re-enacted here with the kernels' own index scheme (outer radix-2^r pass,
// three radix-16 passes per 4096-block with the transposed last-pass twiddles) and must satisfy the round trip and the
// convolution theorem; the CRT constants must reconstruct known integers.  No GPU, no CUDA.
#include "../../seal_b200/csrc/sb_host.hpp"
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <random>
using namespace sbh;
typedef uint32_t u32;

static u32 mulw(u32 y, const u32 *w, u32 p)
{
    u32 q = static_cast<u32>((static_cast<u64>(y) * w[1]) >> 32);
    u32 r = y * w[0] - q * p; // [0, 2p)
    if (r >= 2 * p) { std::printf("lazy product out of range\n"); std::exit(1); }
    return r;
}
static void ct(u32 &x, u32 &y, const u32 *w, u32 p)
{
    u32 u = x >= 2 * p ? x - 2 * p : x, t = mulw(y, w, p);
    x = u + t, y = u - t + 2 * p;
}
static void gs(u32 &x, u32 &y, const u32 *w, u32 p)
{
    u32 u = x + y, v = x - y + 2 * p;
    x = u >= 2 * p ? u - 2 * p : u, y = mulw(v, w, p);
}
template <class TW> static void radix_fwd(int LOG, u32 *a, TW tw, u32 p)
{
    for (int lvl = 0; lvl < LOG; lvl++)
    {
        int gap = (1 << (LOG - 1)) >> lvl;
        for (int g = 0; g < (1 << lvl); g++)
            for (int e = 0; e < gap; e++)
                ct(a[2 * g * gap + e], a[2 * g * gap + e + gap], tw(lvl, g), p);
    }
}
template <class TW> static void radix_inv(int LOG, u32 *a, TW tw, u32 p)
{
    for (int lvl = LOG - 1; lvl >= 0; lvl--)
    {
        int gap = (1 << (LOG - 1)) >> lvl;
        for (int g = 0; g < (1 << lvl); g++)
            for (int e = 0; e < gap; e++)
                gs(a[2 * g * gap + e], a[2 * g * gap + e + gap], tw(lvl, g), p);
    }
}
static void forward(const KsIntHost &h, int t, size_t n, std::vector<u32> &x)
{
    const u32 p = h.p[t];
    const int r = h.r, E = 1 << r;
    const size_t nb = size_t(1) << r;
    for (size_t j = 0; j < 4096; j++)
    {
        u32 a[32];
        for (int e = 0; e < E; e++) a[e] = x[j + 4096 * e];
        const u32 *tw = &h.fwd_outer[(t * nb) * 2];
        radix_fwd(r, a, [&](int lvl, int g) { return tw + 2 * ((1 << lvl) + g); }, p);
        for (int e = 0; e < E; e++) x[j + 4096 * e] = a[e];
    }
    for (size_t g = 0; g < nb; g++)
    {
        u32 *blk = &x[g * 4096];
        const u32 *tws = &h.fwd_local[(t * nb + g) * 4096 * 2];
        for (int tid = 0; tid < 256; tid++)
        {
            u32 a[16];
            for (int e = 0; e < 16; e++) a[e] = blk[tid + 256 * e];
            radix_fwd(4, a, [&](int lvl, int gg) { return tws + 2 * ((1 << lvl) + gg); }, p);
            for (int e = 0; e < 16; e++) blk[tid + 256 * e] = a[e];
        }
        for (int tid = 0; tid < 256; tid++)
        {
            int b = tid >> 4, l = tid & 15;
            u32 a[16];
            for (int e = 0; e < 16; e++) a[e] = blk[(b << 8) + l + 16 * e];
            radix_fwd(4, a, [&](int lvl, int gg) { return tws + 2 * ((16 << lvl) + (b << lvl) + gg); }, p);
            for (int e = 0; e < 16; e++) blk[(b << 8) + l + 16 * e] = a[e];
        }
        for (int tid = 0; tid < 256; tid++)
        {
            u32 a[16];
            for (int e = 0; e < 16; e++) a[e] = blk[16 * tid + e];
            radix_fwd(4, a, [&](int lvl, int gg) { return tws + 2 * (256 + (((1 << lvl) - 1 + gg) << 8) + tid); }, p);
            for (int e = 0; e < 16; e++)
            {
                u32 v = a[e];
                v = v >= 2 * p ? v - 2 * p : v, v = v >= p ? v - p : v;
                blk[16 * tid + e] = v;
            }
        }
    }
}
static void inverse(const KsIntHost &h, int t, size_t n, std::vector<u32> &x)
{
    const u32 p = h.p[t];
    const int r = h.r, E = 1 << r;
    const size_t nb = size_t(1) << r;
    for (size_t g = 0; g < nb; g++)
    {
        u32 *blk = &x[g * 4096];
        const u32 *tws = &h.inv_local[(t * nb + g) * 4096 * 2];
        for (int tid = 0; tid < 256; tid++)
        {
            u32 a[16];
            for (int e = 0; e < 16; e++) a[e] = blk[16 * tid + e];
            radix_inv(4, a, [&](int lvl, int gg) { return tws + 2 * (256 + (((1 << lvl) - 1 + gg) << 8) + tid); }, p);
            for (int e = 0; e < 16; e++) blk[16 * tid + e] = a[e];
        }
        for (int tid = 0; tid < 256; tid++)
        {
            int b = tid >> 4, l = tid & 15;
            u32 a[16];
            for (int e = 0; e < 16; e++) a[e] = blk[(b << 8) + l + 16 * e];
            radix_inv(4, a, [&](int lvl, int gg) { return tws + 2 * ((16 << lvl) + (b << lvl) + gg); }, p);
            for (int e = 0; e < 16; e++) blk[(b << 8) + l + 16 * e] = a[e];
        }
        for (int tid = 0; tid < 256; tid++)
        {
            u32 a[16];
            for (int e = 0; e < 16; e++) a[e] = blk[tid + 256 * e];
            radix_inv(4, a, [&](int lvl, int gg) { return tws + 2 * ((1 << lvl) + gg); }, p);
            for (int e = 0; e < 16; e++) blk[tid + 256 * e] = a[e];
        }
    }
    for (size_t j = 0; j < 4096; j++)
    {
        u32 a[32];
        for (int e = 0; e < E; e++) a[e] = x[j + 4096 * e];
        const u32 *tw = &h.inv_outer[(t * nb) * 2];
        radix_inv(r, a, [&](int lvl, int g) { return tw + 2 * ((1 << lvl) + g); }, p);
        for (int e = 0; e < E; e++) x[j + 4096 * e] = a[e];
    }
}

int main(int argc, char **argv)
{
    const size_t n = argc > 1 ? std::strtoul(argv[1], nullptr, 10) : 8192;
    std::vector<int> bits = { 55, 55, 55, 56 };
    if (argc > 2)
    {
        bits.clear();
        for (int i = 2; i < argc; i++) bits.push_back(std::atoi(argv[i]));
    }
    std::vector<u64> q = coeff_modulus_create(n, bits);
    const size_t k = q.size();
    KsIntHost h = build_ksint(n, q.data(), k);
    if (h.S < 1) { std::printf("no tables\n"); return 1; }
    std::mt19937_64 rng(n);
    int bad = 0;
    // (1) transforms: round trip and convolution theorem, every auxiliary prime
    for (int t = 0; t < h.S; t++)
    {
        const u64 p = h.p[t];
        if (p % (2 * n) != 1 || !is_prime(p) || p >= (u64(1) << 29)) bad++, std::printf("bad prime %llu\n", p);
        std::vector<u32> a(n), b(n);
        for (size_t i = 0; i < n; i++) a[i] = rng() % p, b[i] = rng() % p;
        std::vector<u32> fa = a, fb = b;
        forward(h, t, n, fa), forward(h, t, n, fb);
        std::vector<u32> back = fa;
        inverse(h, t, n, back);
        for (size_t i = 0; i < n; i++)
            if (back[i] % p != mulmod(a[i], n % p, p)) { bad++; std::printf("round trip fails, prime %d index %zu\n", t, i); break; }
        std::vector<u32> prod(n);
        for (size_t i = 0; i < n; i++) prod[i] = static_cast<u32>(mulmod(fa[i], fb[i], p));
        inverse(h, t, n, prod);
        // sparse direct check: 8 output coefficients
        for (int s = 0; s < 8; s++)
        {
            size_t x = rng() % n;
            u64 acc = 0;
            for (size_t i = 0; i < n; i++)
            {
                size_t j = (x + n - i) % n;
                u64 term = mulmod(a[i], b[j], p);
                acc = (i + j == x) ? (acc + term) % p : (acc + p - term) % p;
            }
            if (prod[x] % p != mulmod(acc, n % p, p)) { bad++; std::printf("convolution fails, prime %d index %zu\n", t, x); break; }
        }
    }
    // (2) CRT constants: value v in (-B, B) from its residues, as ks32_crt_kernel evaluates it; the first trials are the exact
    // extremes +-L n (q_J - 1)(q_I - 1) with the largest primes (what all-(q - 1) digits and keys reach), then random magnitudes
    u128 Bound = static_cast<u128>(k - 1) * n;
    const u64 qmax = *std::max_element(q.begin(), q.end());
    for (int trial = 0; trial < 2000 + 2 * static_cast<int>(k); trial++)
    {
        const bool extreme = trial < 2 * static_cast<int>(k);
        // v = +- m1 * m2 * mult, |v| <= L n (max q - 1)^2
        const u64 m1 = extreme ? qmax - 1 : rng() % q[k - 1], m2 = extreme ? qmax - 1 : rng() % q[0];
        const bool neg = extreme ? (trial & 1) : (rng() & 1);
        const u64 mult = extreme ? static_cast<u64>(Bound) : rng() % static_cast<u64>(Bound);
        const size_t i = extreme ? static_cast<size_t>(trial >> 1) : rng() % k;
        const u64 qi = q[i];
        u64 vq = mulmod(mulmod(m1 % qi, m2 % qi, qi), mult % qi, qi);
        if (neg) vq = (qi - vq) % qi;
        u64 f = 0; // the kernels' estimate of alpha: sum y_t floor(2^60 / p_t) >> 60
        u128 acc = 0; // 96 bits suffice
        for (int t = 0; t < h.S; t++)
        {
            const u64 p = h.p[t];
            u64 r = mulmod(mulmod(m1 % p, m2 % p, p), mult % p, p);
            if (neg) r = (p - r) % p;
            const u64 x = mulmod(r, n % p, p);              // what the unscaled inverse transform returns
            u64 y = (mulmod(x, h.c1[2 * t], p) + h.c2[t]) % p;
            f += y * ((u64(1) << 60) / p);
            acc += static_cast<u128>(y) * h.punct_mod_q[i * h.S + t];
        }
        const int alpha = static_cast<int>(f >> 60);
        if (alpha < 0 || alpha >= h.S) { bad++; std::printf("alpha out of range\n"); break; }
        acc += h.neg_mod_q[i * h.S + alpha];
        if (static_cast<u64>(acc % qi) != vq) { bad++; std::printf("CRT reconstruction fails (trial %d%s)\n", trial, extreme ? ", extreme" : ""); break; }
    }
    // (3) the product kernels' 64-bit sums: max_digits products of (max p - 1)^2 fit, one more does not
    {
        const u64 pm1 = *std::max_element(h.p.begin(), h.p.end()) - 1;
        const u128 sq = static_cast<u128>(pm1) * pm1, lim = static_cast<u128>(1) << 64;
        if (h.max_digits < 1 || static_cast<u128>(h.max_digits) * sq >= lim || static_cast<u128>(h.max_digits + 1) * sq < lim)
            bad++, std::printf("max_digits %zu is not the largest L with L (p - 1)^2 < 2^64\n", h.max_digits);
    }
    std::printf("auxiliary primes:");
    for (int t = 0; t < h.S; t++)
        std::printf(" %u", h.p[t]);
    std::printf("\nmax_digits %zu\n", h.max_digits);
    std::printf("ksint host check n=%zu S=%d r=%d: %s\n", n, h.S, h.r, bad ? "FAILED" : "ok");
    return bad ? 1 : 0;
}
