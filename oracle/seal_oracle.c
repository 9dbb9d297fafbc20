/* oracle/seal_oracle.c -- TEST INFRASTRUCTURE ONLY (see seal_oracle.h for the contract and how it is pinned).
 *
 * Plain restatement of the reference hot path with `unsigned __int128 %` arithmetic.  Paths in comments are relative
 * to /root/reference/native/src/seal/.  Nothing here is tuned; clarity over speed.
 */
#include "seal_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

typedef uint64_t u64;
typedef unsigned __int128 u128;

/* ------------------------------------------------------------------ scalar helpers (util/uintarithsmallmod.h) -- */
static u64 mulmod(u64 a, u64 b, u64 q) { return (u64)(((u128)a * b) % q); }
static u64 addmod(u64 a, u64 b, u64 q) { return (u64)(((u128)a + b) % q); }
static u64 submod(u64 a, u64 b, u64 q) { return (u64)(((u128)(a % q) + q - (b % q)) % q); }
/* the reference's words for add_poly_coeffmod / sub_poly_coeffmod / negate_poly_coeffmod on ANY 64-bit operands (release build,
 * polyarithsmallmod.cpp:93-128, polyarithsmallmod.h:95-105): the sum wraps mod 2^64 and sheds q once; the difference is the
 * 64-bit one plus q on a borrow, not reduced further; the negation is q - x mod 2^64 for x != 0.  On words below q they equal
 * addmod / submod; on other words they are what a caller of the reference gets back. */
static u64 add_word(u64 a, u64 b, u64 q)
{
    u64 s = a + b;
    return s >= q ? s - q : s;
}
static u64 sub_word(u64 a, u64 b, u64 q) { return a - b + (a < b ? q : 0); }
static u64 neg_word(u64 a, u64 q) { return a ? q - a : 0; }
static u64 powmod(u64 a, u64 e, u64 q)
{
    u64 r = 1 % q;
    a %= q;
    while (e)
    {
        if (e & 1)
            r = mulmod(r, a, q);
        a = mulmod(a, a, q);
        e >>= 1;
    }
    return r;
}
/* modular inverse for any modulus coprime to a (extended Euclid; needed for m_tilde = 2^32 and 2n) */
static int invmod(u64 a, u64 m, u64 *out)
{
    __int128 t = 0, nt = 1, r = m, nr = a % m;
    while (nr)
    {
        __int128 qq = r / nr, tmp = t - qq * nt;
        t = nt, nt = tmp;
        tmp = r - qq * nr;
        r = nr, nr = tmp;
    }
    if (r != 1)
        return 0;
    if (t < 0)
        t += m;
    *out = (u64)t;
    return 1;
}
static u64 reverse_bits(u64 x, int bits)
{
    u64 r = 0;
    for (int i = 0; i < bits; i++)
        r |= ((x >> i) & 1) << (bits - 1 - i);
    return r;
}
static int ilog2(size_t n)
{
    int l = 0;
    while (((size_t)1 << l) < n)
        l++;
    return l;
}

/* ------------------------------------------------------------------------------- number theory (util/numth.cpp) -- */
/* numth.cpp:180-277 is a probabilistic Miller-Rabin; primality is a fact, so we use the deterministic base set that
 * is exact for all 64-bit integers. */
int orc_is_prime(u64 v)
{
    static const u64 small[] = { 2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37 };
    if (v < 2)
        return 0;
    for (size_t i = 0; i < 12; i++)
    {
        if (v == small[i])
            return 1;
        if (v % small[i] == 0)
            return 0;
    }
    u64 d = v - 1;
    int r = 0;
    while (!(d & 1))
        d >>= 1, r++;
    for (size_t i = 0; i < 12; i++)
    {
        u64 x = powmod(small[i], d, v);
        if (x == 1 || x == v - 1)
            continue;
        int ok = 0;
        for (int j = 1; j < r; j++)
        {
            x = mulmod(x, x, v);
            if (x == v - 1)
            {
                ok = 1;
                break;
            }
        }
        if (!ok)
            return 0;
    }
    return 1;
}

/* numth.cpp:278-311: primes = 1 mod factor, scanning down from 2^bit_size */
int orc_get_primes(u64 factor, int bit_size, size_t count, u64 *out)
{
    u64 value = (((u64)1 << bit_size) - 1) / factor * factor + 1;
    u64 lower = (u64)1 << (bit_size - 1);
    size_t found = 0;
    while (found < count && value > lower)
    {
        if (orc_is_prime(value))
            out[found++] = value;
        value -= factor;
    }
    return found == count ? 0 : -1;
}

/* modulus.cpp:144-184: per distinct bit size take the `count` largest primes; hand them out smallest-first */
int orc_coeff_modulus_create(size_t n, const int *bits, size_t k, u64 *out)
{
    int used[ORC_MAX_PRIMES] = { 0 };
    if (k > ORC_MAX_PRIMES)
        return -1;
    for (size_t i = 0; i < k; i++)
    {
        if (used[i])
            continue;
        size_t cnt = 0, idx[ORC_MAX_PRIMES];
        for (size_t j = i; j < k; j++)
            if (bits[j] == bits[i])
                idx[cnt++] = j, used[j] = 1;
        u64 primes[ORC_MAX_PRIMES];
        if (orc_get_primes(2 * (u64)n, bits[i], cnt, primes))
            return -1;
        for (size_t j = 0; j < cnt; j++)
            out[idx[j]] = primes[cnt - 1 - j];
    }
    return 0;
}

/* numth.cpp:340-412: the reference draws a random primitive root and then walks all odd powers keeping the minimum;
 * the minimum over the full set of primitive degree-th roots does not depend on the starting point, so we start from
 * the first small generator candidate that works. */
int orc_minimal_primitive_root(u64 degree, u64 q, u64 *root)
{
    if ((q - 1) % degree)
        return -1;
    u64 quot = (q - 1) / degree, r = 0;
    for (u64 g = 2; g < 1000; g++)
    {
        r = powmod(g, quot, q);
        if (powmod(r, degree >> 1, q) == q - 1)
            break;
        r = 0;
    }
    if (!r)
        return -1;
    u64 gsq = mulmod(r, r, q), cur = r, best = r;
    for (u64 i = 0; i < degree; i += 2)
    {
        if (cur < best)
            best = cur;
        cur = mulmod(cur, gsq, q);
    }
    *root = best;
    return 0;
}

/* ------------------------------------------------------------------------------------------------- NTT tables -- */
typedef struct
{
    u64 q, root, inv_n;
    u64 *rp;  /* root_powers[bitrev(i)] = psi^i            ntt.cpp:269-278 */
    u64 *irp; /* inv_root_powers[bitrev(i-1)+1] = psi^-i   ntt.cpp:280-288 */
} orc_tab;

static int tab_init(orc_tab *t, size_t n, u64 q)
{
    int logn = ilog2(n);
    t->q = q;
    if (orc_minimal_primitive_root(2 * (u64)n, q, &t->root)) /* ntt.cpp:254 */
        return -1;
    u64 inv_root = 0;
    if (!invmod(t->root, q, &inv_root))
        return -1;
    t->rp = (u64 *)malloc(n * sizeof(u64));
    t->irp = (u64 *)malloc(n * sizeof(u64));
    u64 p = t->root;
    for (size_t i = 1; i < n; i++)
    {
        t->rp[reverse_bits(i, logn)] = p;
        p = mulmod(p, t->root, q);
    }
    t->rp[0] = 1;
    p = inv_root;
    for (size_t i = 1; i < n; i++)
    {
        t->irp[reverse_bits(i - 1, logn) + 1] = p;
        p = mulmod(p, inv_root, q);
    }
    t->irp[0] = 1;
    if (!invmod((u64)n % q, q, &t->inv_n)) /* ntt.cpp:290-296 */
        return -1;
    return 0;
}
static void tab_free(orc_tab *t)
{
    free(t->rp);
    free(t->irp);
    t->rp = t->irp = NULL;
}

/* dwthandler.h:94-191 (Cooley-Tukey, natural in -> bit-reversed out, roots consumed sequentially from index 1) */
static void ntt_fwd(const orc_tab *t, size_t n, u64 *x)
{
    u64 q = t->q;
    size_t gap = n >> 1, m = 1, ridx = 0;
    for (; m < n; m <<= 1, gap >>= 1)
    {
        size_t off = 0;
        for (size_t i = 0; i < m; i++, off += 2 * gap)
        {
            u64 r = t->rp[++ridx];
            for (size_t j = 0; j < gap; j++)
            {
                u64 u = x[off + j] % q, v = mulmod(x[off + j + gap], r, q);
                x[off + j] = addmod(u, v, q);
                x[off + j + gap] = submod(u, v, q);
            }
        }
    }
}
/* dwthandler.h:202-356 (Gentleman-Sande, bit-reversed in -> natural out, 1/n folded into the last stage) */
static void ntt_inv(const orc_tab *t, size_t n, u64 *x)
{
    u64 q = t->q;
    size_t gap = 1, m = n >> 1, ridx = 0;
    for (; m >= 1; m >>= 1, gap <<= 1)
    {
        size_t off = 0;
        for (size_t i = 0; i < m; i++, off += 2 * gap)
        {
            u64 r = t->irp[++ridx];
            for (size_t j = 0; j < gap; j++)
            {
                u64 u = x[off + j] % q, v = x[off + j + gap] % q;
                x[off + j] = addmod(u, v, q);
                x[off + j + gap] = mulmod(submod(u, v, q), r, q);
            }
        }
        if (m == 1)
            break;
    }
    for (size_t i = 0; i < n; i++)
        x[i] = mulmod(x[i], t->inv_n, q);
}

/* ---------------------------------------------------------------------------------------------------- context -- */
struct orc_ctx
{
    int scheme;
    size_t n, k;
    int logn;
    u64 q[ORC_MAX_PRIMES], t;
    orc_tab tab[ORC_MAX_PRIMES];
};

orc_ctx *orc_create(int scheme, size_t n, const u64 *moduli, size_t k, u64 t)
{
    if (k == 0 || k > ORC_MAX_PRIMES || n < 2 || (n & (n - 1)))
        return NULL;
    orc_ctx *c = (orc_ctx *)calloc(1, sizeof(orc_ctx));
    c->scheme = scheme, c->n = n, c->k = k, c->t = t, c->logn = ilog2(n);
    for (size_t i = 0; i < k; i++)
    {
        c->q[i] = moduli[i];
        if (tab_init(&c->tab[i], n, moduli[i]))
        {
            orc_destroy(c);
            return NULL;
        }
    }
    return c;
}
void orc_destroy(orc_ctx *c)
{
    if (!c)
        return;
    for (size_t i = 0; i < c->k; i++)
        tab_free(&c->tab[i]);
    free(c);
}
int orc_ntt_tables(const orc_ctx *c, size_t i, u64 *root, u64 *rp, u64 *irp, u64 *inv_n)
{
    if (i >= c->k)
        return -1;
    *root = c->tab[i].root;
    *inv_n = c->tab[i].inv_n;
    memcpy(rp, c->tab[i].rp, c->n * sizeof(u64));
    memcpy(irp, c->tab[i].irp, c->n * sizeof(u64));
    return 0;
}

void orc_ntt_row(const orc_ctx *c, size_t i, u64 *row) { ntt_fwd(&c->tab[i], c->n, row); }
void orc_intt_row(const orc_ctx *c, size_t i, u64 *row) { ntt_inv(&c->tab[i], c->n, row); }

void orc_ntt_forward(const orc_ctx *c, size_t L, size_t size, u64 *d)
{
    for (size_t p = 0; p < size; p++)
        for (size_t i = 0; i < L; i++)
            ntt_fwd(&c->tab[i], c->n, d + (p * L + i) * c->n);
}
void orc_ntt_inverse(const orc_ctx *c, size_t L, size_t size, u64 *d)
{
    for (size_t p = 0; p < size; p++)
        for (size_t i = 0; i < L; i++)
            ntt_inv(&c->tab[i], c->n, d + (p * L + i) * c->n);
}

/* ---------------------------------------------------------------------- CKKS multiply (evaluator.cpp:634-662) -- */
void orc_ckks_multiply(const orc_ctx *c, size_t L, const u64 *a, const u64 *b, u64 *o)
{
    orc_ckks_multiply_sized(c, L, 2, 2, a, b, o);
}

/* out[k] = sum_{i+j=k} x_i * y_j over rows of nb primes (the general-size loop, evaluator.cpp:664-700; 2x2 is :600-662) */
static void tensor_rows(const u64 *x, size_t s1, const u64 *y, size_t s2, size_t nb, size_t n, const u64 *mods, u64 *o)
{
    size_t P = nb * n;
    for (size_t k = 0; k < s1 + s2 - 1; k++)
        for (size_t i = 0; i < nb; i++)
            for (size_t j = 0; j < n; j++)
            {
                size_t e = i * n + j;
                u64 acc = 0;
                for (size_t p = 0; p < s1; p++)
                    if (k >= p && k - p < s2)
                        acc = addmod(acc, mulmod(x[p * P + e], y[(k - p) * P + e], mods[i]), mods[i]);
                o[k * P + e] = acc;
            }
}
void orc_ckks_multiply_sized(const orc_ctx *c, size_t L, size_t s1, size_t s2, const u64 *a, const u64 *b, u64 *o)
{
    tensor_rows(a, s1, b, s2, L, c->n, c->q, o);
}

/* add / sub / negate (evaluator.cpp:130-350; polyarithsmallmod.cpp:43-195) */
void orc_linear(const orc_ctx *c, int mode, size_t L, size_t size, const u64 *a, const u64 *b, u64 *out)
{
    size_t n = c->n;
    for (size_t p = 0; p < size; p++)
        for (size_t i = 0; i < L; i++)
            for (size_t j = 0; j < n; j++)
            {
                size_t e = (p * L + i) * n + j;
                u64 q = c->q[i];
                out[e] = mode == 0 ? add_word(a[e], b[e], q) : mode == 1 ? sub_word(a[e], b[e], q) : neg_word(a[e], q);
            }
}

/* multiply_plain with both operands in NTT form (evaluator.cpp:2157-2195: dyadic_product_coeffmod per polynomial) */
void orc_multiply_plain_ntt(const orc_ctx *c, size_t L, size_t size, const u64 *a, const u64 *plain, u64 *out)
{
    size_t n = c->n;
    for (size_t p = 0; p < size; p++)
        for (size_t i = 0; i < L; i++)
            for (size_t j = 0; j < n; j++)
                out[(p * L + i) * n + j] = mulmod(a[(p * L + i) * n + j], plain[i * n + j], c->q[i]);
}

/* ---- BatchEncoder (batchencoder.cpp:54-76 index map, :84-130 encode, :229-275 decode) ------------------------------------ */
int orc_batch_codec(const orc_ctx *c, int decode, const u64 *in, u64 *out)
{
    size_t n = c->n, row = n >> 1;
    int logn = ilog2(n);
    orc_tab tt; /* plain_ntt_tables: transform tables modulo t (context.cpp:374-394) */
    if (tab_init(&tt, n, c->t))
        return -1;
    size_t *map = (size_t *)malloc(n * sizeof(size_t));
    u64 m = (u64)n << 1, pos = 1;
    for (size_t i = 0; i < row; i++)
    {
        map[i] = (size_t)reverse_bits((pos - 1) >> 1, logn);
        map[row | i] = (size_t)reverse_bits((m - pos - 1) >> 1, logn);
        pos = (pos * 3) & (m - 1);
    }
    if (!decode)
    {
        for (size_t i = 0; i < n; i++)
            out[map[i]] = in[i];
        ntt_inv(&tt, n, out);
    }
    else
    {
        u64 *tmp = (u64 *)malloc(n * sizeof(u64));
        memcpy(tmp, in, n * sizeof(u64));
        ntt_fwd(&tt, n, tmp);
        for (size_t i = 0; i < n; i++)
            out[i] = tmp[map[i]];
        free(tmp);
    }
    free(map);
    tab_free(&tt);
    return 0;
}

/* ---- coefficient-form plaintexts (BFV / BGV) -------------------------------------------------------------------------- */
/* the lift of evaluator.cpp:2240-2272 / :2101-2127: words >= (t+1)/2 stand for negative numbers */
static u64 plain_lift(u64 v, u64 t, u64 q)
{
    return v >= ((t + 1) >> 1) ? submod(v % q, t % q, q) : v % q;
}
/* Evaluator::transform_to_ntt_inplace(Plaintext, parms_id) (evaluator.cpp:2197-2287): plain [n] -> out [L][n] */
void orc_plain_to_ntt(const orc_ctx *c, size_t L, const u64 *plain, u64 *out)
{
    size_t n = c->n;
    for (size_t i = 0; i < L; i++)
    {
        for (size_t j = 0; j < n; j++)
            out[i * n + j] = plain_lift(plain[j], c->t, c->q[i]);
        ntt_fwd(&c->tab[i], n, out + i * n);
    }
}
/* Evaluator::multiply_plain with a coefficient-form plaintext: multiply_plain_normal (:2021-2155) when the ciphertext is in
 * coefficient form, transform + multiply_plain_ntt (:1999-2004) when it is in NTT form */
void orc_multiply_plain_coeff(const orc_ctx *c, size_t L, size_t size, int ct_is_ntt, const u64 *a, const u64 *plain, u64 *out)
{
    size_t n = c->n;
    u64 *p = (u64 *)malloc(L * n * sizeof(u64));
    orc_plain_to_ntt(c, L, plain, p);
    memcpy(out, a, size * L * n * sizeof(u64));
    if (!ct_is_ntt)
        orc_ntt_forward(c, L, size, out);
    orc_multiply_plain_ntt(c, L, size, out, p, out);
    if (!ct_is_ntt)
        orc_ntt_inverse(c, L, size, out);
    free(p);
}
/* Evaluator::add_plain / sub_plain with a coefficient-form plaintext; BFV: util/scalingvariant.cpp:70-160 (c_0 +/-
 * floor((q m + (t+1)/2) / t), evaluated as m * floor(q/t) + floor((m (q mod t) + (t+1)/2) / t)); BGV: evaluator.cpp:1838-1849 */
void orc_add_plain_coeff(const orc_ctx *c, size_t L, size_t size, int subtract, u64 correction_factor, const u64 *a, const u64 *plain, u64 *out)
{
    size_t n = c->n;
    u64 t = c->t;
    memcpy(out, a, size * L * n * sizeof(u64));
    if (c->scheme == ORC_BFV)
    {
        u64 q_mod_t = 1;
        for (size_t i = 0; i < L; i++)
            q_mod_t = mulmod(q_mod_t, c->q[i] % t, t);
        for (size_t i = 0; i < L; i++)
        {
            u64 q = c->q[i], inv_t = 0;
            invmod(t % q, q, &inv_t);
            u64 delta = mulmod(submod(0, q_mod_t % q, q), inv_t, q); /* floor(Q / t) mod q_i, Q = 0 mod q_i */
            for (size_t j = 0; j < n; j++)
            {
                u64 m = plain[j];
                u64 fix = (u64)(((u128)m * q_mod_t + ((t + 1) >> 1)) / t);
                u64 scaled = addmod(mulmod(m % q, delta, q), fix % q, q);
                out[i * n + j] = subtract ? sub_word(out[i * n + j], scaled, q) : add_word(out[i * n + j], scaled, q);
            }
        }
        return;
    }
    u64 *m = (u64 *)malloc(n * sizeof(u64)), *p = (u64 *)malloc(L * n * sizeof(u64));
    for (size_t j = 0; j < n; j++)
        m[j] = mulmod(plain[j], correction_factor, t);
    orc_plain_to_ntt(c, L, m, p);
    for (size_t i = 0; i < L; i++)
        for (size_t j = 0; j < n; j++)
            out[i * n + j] = subtract ? sub_word(out[i * n + j], p[i * n + j], c->q[i]) : add_word(out[i * n + j], p[i * n + j], c->q[i]);
    free(m), free(p);
}

/* -------------------------------------------------------------------- key switching (evaluator.cpp:2561-2867) -- */
void orc_switch_key(const orc_ctx *c, size_t L, u64 *ct, const u64 *target, const u64 *key)
{
    size_t n = c->n, K = c->k, sp = K - 1;
    int ntt_in = (c->scheme != ORC_BFV);
    /* :2651-2658  d_J = coefficients of the J-th RNS component */
    u64 *d = (u64 *)malloc(L * n * sizeof(u64));
    memcpy(d, target, L * n * sizeof(u64));
    if (ntt_in)
        for (size_t J = 0; J < L; J++)
            ntt_inv(&c->tab[J], n, d + J * n);
    u64 *prod = (u64 *)calloc(2 * (L + 1) * n, sizeof(u64)); /* t_poly_prod [2][L+1][n] */
    u64 *tmp = (u64 *)malloc(n * sizeof(u64));
    for (size_t I = 0; I <= L; I++)
    {
        size_t ki = (I == L) ? sp : I; /* :2664 */
        u64 q = c->q[ki];
        for (size_t J = 0; J < L; J++)
        {
            /* :2682-2702  digit J seen modulo q_I, in NTT form */
            if (ntt_in && I == J)
                memcpy(tmp, target + J * n, n * sizeof(u64));
            else
            {
                for (size_t j = 0; j < n; j++)
                    tmp[j] = d[J * n + j] % q;
                ntt_fwd(&c->tab[ki], n, tmp);
            }
            /* :2705-2729  multiply-accumulate with key[J][comp][ki] */
            for (size_t comp = 0; comp < 2; comp++)
            {
                const u64 *kr = key + ((J * 2 + comp) * K + ki) * n;
                u64 *acc = prod + (comp * (L + 1) + I) * n;
                for (size_t j = 0; j < n; j++)
                    acc[j] = addmod(acc[j], mulmod(tmp[j] % q, kr[j], q), q);
            }
        }
    }
    /* :2806-2864 mod-down by the special prime, added into ct */
    u64 qk = c->q[sp], half = qk >> 1;
    for (size_t comp = 0; comp < 2 && c->scheme == ORC_BGV; comp++)
    {
        /* :2762-2805 BGV: subtract c + k*qk with k = -c * qk^-1 mod t, so the quotient stays = 0 mod t */
        u64 *last = prod + (comp * (L + 1) + L) * n, t = c->t, inv_t = 0;
        ntt_inv(&c->tab[sp], n, last);
        invmod(qk % t, t, &inv_t); /* RNSTool::inv_q_last_mod_t of the key level, rns.cpp:778-787 */
        for (size_t i = 0; i < L; i++)
        {
            u64 q = c->q[i], inv = 0;
            u64 *acc = prod + (comp * (L + 1) + i) * n;
            for (size_t j = 0; j < n; j++)
            {
                u64 k = mulmod(submod(0, last[j] % t, t), inv_t, t);                /* :2773-2779 */
                tmp[j] = addmod(mulmod(k % q, qk % q, q), last[j] % q, q);          /* :2785-2794 */
            }
            ntt_fwd(&c->tab[i], n, tmp); /* :2795 */
            invmod(qk % q, q, &inv);
            u64 *dst = ct + (comp * L + i) * n;
            for (size_t j = 0; j < n; j++)
                dst[j] = addmod(dst[j], mulmod(submod(acc[j], tmp[j], q), inv, q), q); /* :2796-2802 */
        }
    }
    for (size_t comp = 0; comp < 2 && c->scheme != ORC_BGV; comp++)
    {
        u64 *last = prod + (comp * (L + 1) + L) * n;
        ntt_inv(&c->tab[sp], n, last);
        for (size_t j = 0; j < n; j++)
            last[j] = addmod(last[j], half, qk); /* :2813-2817 */
        for (size_t i = 0; i < L; i++)
        {
            u64 q = c->q[i];
            u64 *acc = prod + (comp * (L + 1) + i) * n;
            for (size_t j = 0; j < n; j++)
                tmp[j] = submod(last[j] % q, half % q, q); /* :2824-2836 */
            if (c->scheme == ORC_CKKS)
                ntt_fwd(&c->tab[i], n, tmp); /* :2842 */
            else
                ntt_inv(&c->tab[i], n, acc); /* :2854 (BFV: accumulated poly back to coefficients) */
            u64 inv = 0;
            invmod(qk % q, q, &inv); /* inv_q_last_mod_q of the key level, rns.cpp:767-776 */
            u64 *dst = ct + (comp * L + i) * n;
            for (size_t j = 0; j < n; j++)
                dst[j] = addmod(dst[j], mulmod(submod(acc[j], tmp[j], q), inv, q), q); /* :2858-2863 */
        }
    }
    free(d), free(prod), free(tmp);
}

/* evaluator.cpp:1144-1199 (size 3 -> 2) */
void orc_relinearize(const orc_ctx *c, size_t L, const u64 *in3, const u64 *key, u64 *out2)
{
    size_t P = L * c->n;
    memcpy(out2, in3, 2 * P * sizeof(u64));
    orc_switch_key(c, L, out2, in3 + 2 * P, key);
}

/* CKKS rescale: rns.cpp:830-901 + evaluator.cpp:1276-1279 (drop last component) */
void orc_rescale(const orc_ctx *c, size_t L, const u64 *in2, u64 *out2)
{
    size_t n = c->n;
    u64 ql = c->q[L - 1], half = ql >> 1;
    u64 *last = (u64 *)malloc(n * sizeof(u64)), *tmp = (u64 *)malloc(n * sizeof(u64));
    for (size_t p = 0; p < 2; p++)
    {
        memcpy(last, in2 + (p * L + L - 1) * n, n * sizeof(u64));
        ntt_inv(&c->tab[L - 1], n, last);
        for (size_t j = 0; j < n; j++)
            last[j] = addmod(last[j], half, ql);
        for (size_t i = 0; i + 1 < L; i++)
        {
            u64 q = c->q[i], inv = 0;
            invmod(ql % q, q, &inv);
            for (size_t j = 0; j < n; j++)
                tmp[j] = submod(last[j] % q, half % q, q);
            ntt_fwd(&c->tab[i], n, tmp);
            const u64 *src = in2 + (p * L + i) * n;
            u64 *dst = out2 + (p * (L - 1) + i) * n;
            for (size_t j = 0; j < n; j++)
                dst[j] = mulmod(submod(src[j], tmp[j], q), inv, q);
        }
    }
    free(last), free(tmp);
}

/* BGV mod_switch_to_next: mod_t_and_divide_q_last_ntt_inplace, rns.cpp:1193-1236 + evaluator.cpp:1263-1279 */
void orc_bgv_mod_switch(const orc_ctx *c, size_t L, const u64 *in2, u64 *out2)
{
    size_t n = c->n;
    u64 ql = c->q[L - 1], t = c->t, inv_t = 0;
    invmod(ql % t, t, &inv_t); /* inv_q_last_mod_t of this level, rns.cpp:778-787 */
    u64 *last = (u64 *)malloc(n * sizeof(u64)), *tmp = (u64 *)malloc(n * sizeof(u64));
    for (size_t p = 0; p < 2; p++)
    {
        memcpy(last, in2 + (p * L + L - 1) * n, n * sizeof(u64));
        ntt_inv(&c->tab[L - 1], n, last);
        for (size_t i = 0; i + 1 < L; i++)
        {
            u64 q = c->q[i], inv = 0;
            invmod(ql % q, q, &inv);
            for (size_t j = 0; j < n; j++)
            {
                u64 k = mulmod(submod(0, last[j] % t, t), inv_t, t);       /* :1205-1213 */
                tmp[j] = addmod(mulmod(k % q, ql % q, q), last[j] % q, q); /* :1219-1228 */
            }
            ntt_fwd(&c->tab[i], n, tmp);
            const u64 *src = in2 + (p * L + i) * n;
            u64 *dst = out2 + (p * (L - 1) + i) * n;
            for (size_t j = 0; j < n; j++)
                dst[j] = mulmod(submod(src[j], tmp[j], q), inv, q); /* :1229-1234 */
        }
    }
    free(last), free(tmp);
}

/* BFV mod_switch_to_next: rns.cpp:789-828 (coefficient form) */
void orc_bfv_mod_switch(const orc_ctx *c, size_t L, const u64 *in2, u64 *out2)
{
    size_t n = c->n;
    u64 ql = c->q[L - 1], half = ql >> 1;
    for (size_t p = 0; p < 2; p++)
        for (size_t i = 0; i + 1 < L; i++)
        {
            u64 q = c->q[i], inv = 0;
            invmod(ql % q, q, &inv);
            const u64 *last = in2 + (p * L + L - 1) * n, *src = in2 + (p * L + i) * n;
            u64 *dst = out2 + (p * (L - 1) + i) * n;
            for (size_t j = 0; j < n; j++)
            {
                u64 l = addmod(last[j], half, ql);
                dst[j] = mulmod(submod(src[j], submod(l % q, half % q, q), q), inv, q);
            }
        }
}

/* ------------------------------------------------------------------------------------- Galois (util/galois.cpp) -- */
uint32_t orc_galois_elt_from_step(size_t n, int step) /* galois.cpp:53-95 */
{
    uint64_t m = 2 * (uint64_t)n;
    if (step == 0)
        return (uint32_t)(m - 1);
    int sign = step < 0;
    uint32_t pos = (uint32_t)(sign ? -step : step);
    if (pos >= (n >> 1))
        return 0;
    int s = sign ? (int)(n >> 1) - (int)pos : (int)pos;
    uint64_t e = 1;
    while (s--)
        e = (e * 3) & (m - 1);
    return (uint32_t)e;
}
void orc_galois_coeff_row(size_t n, u64 q, uint32_t g, const u64 *in, u64 *out) /* galois.cpp:148-190 */
{
    int logn = ilog2(n);
    for (u64 i = 0; i < n; i++)
    {
        u64 raw = i * g, idx = raw & (n - 1), v = in[i];
        if ((raw >> logn) & 1)
            v = v ? q - v : 0;
        out[idx] = v;
    }
}
void orc_galois_ntt_row(size_t n, uint32_t g, const u64 *in, u64 *out) /* galois.cpp:18-51, 192-218 */
{
    int logn = ilog2(n);
    for (size_t i = 0; i < n; i++)
    {
        u64 rev = reverse_bits(i + n, logn + 1);
        u64 raw = ((u64)g * rev) >> 1;
        raw &= (n - 1);
        out[i] = in[reverse_bits(raw, logn)];
    }
}
/* evaluator.cpp:2384-2502 */
void orc_apply_galois(const orc_ctx *c, size_t L, const u64 *in2, uint32_t g, const u64 *key, u64 *out2)
{
    size_t n = c->n, P = L * n;
    u64 *temp = (u64 *)malloc(P * sizeof(u64));
    for (size_t i = 0; i < L; i++)
    {
        if (c->scheme == ORC_BFV)
        {
            orc_galois_coeff_row(n, c->q[i], g, in2 + i * n, out2 + i * n);
            orc_galois_coeff_row(n, c->q[i], g, in2 + P + i * n, temp + i * n);
        }
        else
        {
            orc_galois_ntt_row(n, g, in2 + i * n, out2 + i * n);
            orc_galois_ntt_row(n, g, in2 + P + i * n, temp + i * n);
        }
    }
    memset(out2 + P, 0, P * sizeof(u64));
    orc_switch_key(c, L, out2, temp, key);
    free(temp);
}

/* ------------------------------------------------------------------------------ BEHZ (util/rns.cpp, BFV only) -- */
/* bit length of prod(q[0..L)) via a tiny big-integer (rns.cpp:605) */
static int prod_bit_count(const u64 *q, size_t L)
{
    u64 limbs[ORC_MAX_PRIMES + 1] = { 1 };
    size_t len = 1;
    for (size_t i = 0; i < L; i++)
    {
        u64 carry = 0;
        for (size_t j = 0; j < len; j++)
        {
            u128 v = (u128)limbs[j] * q[i] + carry;
            limbs[j] = (u64)v;
            carry = (u64)(v >> 64);
        }
        if (carry)
            limbs[len++] = carry;
    }
    int bits = 0;
    u64 top = limbs[len - 1];
    while (top)
        bits++, top >>= 1;
    return (int)(len - 1) * 64 + bits;
}
static int bit_count(u64 v)
{
    int b = 0;
    while (v)
        b++, v >>= 1;
    return b;
}
typedef struct
{
    size_t nB, nBsk;
    u64 B[ORC_MAX_PRIMES + 1], msk, Bsk[ORC_MAX_PRIMES + 2];
} behz_base;
/* rns.cpp:598-641; works for ANY pairwise-coprime base q (the reference's RNSTool KATs use q = {3}, {3,5}) */
static int behz_base_init_raw(size_t n, const u64 *q, size_t L, u64 t, behz_base *b)
{
    b->nB = L;
    if (32 + bit_count(t) + prod_bit_count(q, L) >= 61 * (int)L + 61)
        b->nB++;
    b->nBsk = b->nB + 1;
    u64 primes[ORC_MAX_PRIMES + 4];
    if (orc_get_primes(2 * (u64)n, 61, b->nBsk + 1, primes))
        return -1;
    b->msk = primes[0]; /* primes[1] = gamma (decryption only) */
    for (size_t i = 0; i < b->nB; i++)
        b->B[i] = b->Bsk[i] = primes[2 + i];
    b->Bsk[b->nB] = b->msk;
    return 0;
}
static int behz_base_init(const orc_ctx *c, size_t L, behz_base *b) { return behz_base_init_raw(c->n, c->q, L, c->t, b); }
size_t orc_behz_base(size_t n, const u64 *q, size_t L, u64 t, u64 *out)
{
    behz_base b;
    if (behz_base_init_raw(n, q, L, t, &b))
        return 0;
    memcpy(out, b.Bsk, b.nBsk * sizeof(u64));
    return b.nBsk;
}
size_t orc_base_bsk(const orc_ctx *c, size_t L, u64 *out) { return orc_behz_base(c->n, c->q, L, c->t, out); }
/* prod_{j != skip} base[j] mod p  (skip = (size_t)-1 for the full product) */
static u64 prod_mod(const u64 *base, size_t nb, size_t skip, u64 p)
{
    u64 r = 1 % p;
    for (size_t j = 0; j < nb; j++)
        if (j != skip)
            r = mulmod(r, base[j] % p, p);
    return r;
}
/* FastBConv, rns.cpp:418-463: y = sum_i [x_i * (b/b_i)^-1 mod b_i] * ((b/b_i) mod p) mod p   (no correction term) */
static void fastbconv(const u64 *ibase, size_t ni, const u64 *x, size_t xstride, size_t n, u64 p, u64 *out)
{
    u64 inv[ORC_MAX_PRIMES + 2], mat[ORC_MAX_PRIMES + 2];
    for (size_t i = 0; i < ni; i++)
    {
        inv[i] = 0;
        invmod(prod_mod(ibase, ni, i, ibase[i]), ibase[i], &inv[i]);
        mat[i] = prod_mod(ibase, ni, i, p);
    }
    for (size_t j = 0; j < n; j++)
    {
        u128 s = 0;
        for (size_t i = 0; i < ni; i++)
        {
            u64 ti = mulmod(x[i * xstride + j] % ibase[i], inv[i], ibase[i]);
            s = (s + (u128)ti * mat[i]) % p;
        }
        out[j] = (u64)s;
    }
}
/* BaseConverter::fast_convert_array (rns.cpp:418-463): in [ni][n] -> out [no][n] */
void orc_fastbconv_array(const u64 *ibase, size_t ni, const u64 *obase, size_t no, const u64 *in, size_t n, u64 *out)
{
    for (size_t s = 0; s < no; s++)
        fastbconv(ibase, ni, in, n, n, obase[s], out + s * n);
}
#define ORC_MT ((u64)1 << 32) /* m_tilde, rns.cpp:635 */
/* RNSTool::fastbconv_m_tilde (rns.cpp:1086-1131): in [L][n] (base q) -> out [nBsk+1][n] (base Bsk U {m_tilde}) */
int orc_behz_fastbconv_m_tilde(size_t n, const u64 *q, size_t L, u64 t, const u64 *in, u64 *out)
{
    behz_base bb;
    if (behz_base_init_raw(n, q, L, t, &bb))
        return -1;
    u64 *tmp = (u64 *)malloc(L * n * sizeof(u64));
    for (size_t i = 0; i < L; i++)
        for (size_t j = 0; j < n; j++)
            tmp[i * n + j] = mulmod(in[i * n + j] % q[i], ORC_MT % q[i], q[i]); /* :1123-1124 */
    for (size_t s = 0; s < bb.nBsk; s++)
        fastbconv(q, L, tmp, n, n, bb.Bsk[s], out + s * n); /* :1127 */
    fastbconv(q, L, tmp, n, n, ORC_MT, out + bb.nBsk * n);  /* :1130 */
    free(tmp);
    return 0;
}
/* RNSTool::sm_mrq (rns.cpp:979-1039): in [nBsk+1][n] -> out [nBsk][n] */
int orc_behz_sm_mrq(size_t n, const u64 *q, size_t L, u64 t, const u64 *in, u64 *out)
{
    behz_base bb;
    if (behz_base_init_raw(n, q, L, t, &bb))
        return -1;
    u64 qinv_mt = 0;
    invmod(prod_mod(q, L, (size_t)-1, ORC_MT), ORC_MT, &qinv_mt);
    u64 neg_inv_q_mt = (ORC_MT - qinv_mt) % ORC_MT; /* rns.cpp:724-730 */
    const u64 *ymt = in + bb.nBsk * n;
    for (size_t s = 0; s < bb.nBsk; s++)
    {
        u64 P = bb.Bsk[s], inv_mt = 0, qmodP = prod_mod(q, L, (size_t)-1, P);
        invmod(ORC_MT % P, P, &inv_mt);
        for (size_t j = 0; j < n; j++)
        {
            u64 r = (u64)(((u128)(ymt[j] % ORC_MT) * neg_inv_q_mt) % ORC_MT);
            if (r >= (ORC_MT >> 1)) /* :1028 */
                r += P - ORC_MT;
            out[s * n + j] = mulmod(addmod(mulmod(r, qmodP, P), in[s * n + j] % P, P), inv_mt, P);
        }
    }
    return 0;
}
/* RNSTool::fast_floor (rns.cpp:1041-1084): in [L + nBsk][n] (base q then Bsk) -> out [nBsk][n] */
int orc_behz_fast_floor(size_t n, const u64 *q, size_t L, u64 t, const u64 *in, u64 *out)
{
    behz_base bb;
    if (behz_base_init_raw(n, q, L, t, &bb))
        return -1;
    u64 *conv = (u64 *)malloc(n * sizeof(u64));
    for (size_t s = 0; s < bb.nBsk; s++)
    {
        u64 P = bb.Bsk[s], invq = 0;
        invmod(prod_mod(q, L, (size_t)-1, P), P, &invq);
        fastbconv(q, L, in, n, n, P, conv);
        for (size_t j = 0; j < n; j++)
            out[s * n + j] = mulmod(submod(in[(L + s) * n + j], conv[j], P), invq, P);
    }
    free(conv);
    return 0;
}
/* RNSTool::fastbconv_sk (rns.cpp:903-977): in [nBsk][n] -> out [L][n] */
int orc_behz_fastbconv_sk(size_t n, const u64 *q, size_t L, u64 t, const u64 *in, u64 *out)
{
    behz_base bb;
    if (behz_base_init_raw(n, q, L, t, &bb))
        return -1;
    size_t nB = bb.nB;
    u64 *conv = (u64 *)malloc(n * sizeof(u64)), *alpha = (u64 *)malloc(n * sizeof(u64));
    u64 invB = 0;
    invmod(prod_mod(bb.B, nB, (size_t)-1, bb.msk), bb.msk, &invB);
    fastbconv(bb.B, nB, in, n, n, bb.msk, conv);
    for (size_t j = 0; j < n; j++)
        alpha[j] = mulmod(submod(conv[j], in[nB * n + j], bb.msk), invB, bb.msk); /* :946-949 */
    for (size_t i = 0; i < L; i++)
    {
        u64 qi = q[i], prodB = prod_mod(bb.B, nB, (size_t)-1, qi);
        u64 *dst = out + i * n;
        fastbconv(bb.B, nB, in, n, n, qi, dst);
        for (size_t j = 0; j < n; j++)
        {
            if (alpha[j] > (bb.msk >> 1)) /* :964 */
                dst[j] = addmod(dst[j], mulmod((bb.msk - alpha[j]) % qi, prodB, qi), qi);
            else
                dst[j] = addmod(dst[j], mulmod(alpha[j] % qi, (qi - prodB) % qi, qi), qi);
        }
    }
    free(conv), free(alpha);
    return 0;
}
/* RNSTool::divide_and_round_q_last_inplace (rns.cpp:789-828): data [L][n]; the first L-1 rows receive the result */
void orc_divide_and_round_q_last(const u64 *q, size_t L, size_t n, u64 *data)
{
    u64 ql = q[L - 1], half = ql >> 1;
    u64 *last = data + (L - 1) * n;
    for (size_t j = 0; j < n; j++)
        last[j] = addmod(last[j], half, ql);
    for (size_t i = 0; i + 1 < L; i++)
    {
        u64 qi = q[i], inv = 0;
        invmod(ql % qi, qi, &inv);
        for (size_t j = 0; j < n; j++)
            data[i * n + j] = mulmod(submod(data[i * n + j], submod(last[j] % qi, half % qi, qi), qi), inv, qi);
    }
}

int orc_bfv_multiply(const orc_ctx *c, size_t L, const u64 *a, const u64 *b, u64 *out3)
{
    return orc_bfv_multiply_sized(c, L, 2, 2, a, b, out3);
}
int orc_bfv_multiply_sized(const orc_ctx *c, size_t L, size_t s1, size_t s2, const u64 *a, const u64 *b, u64 *out3)
{
    size_t n = c->n, nin = s1 + s2, nout = s1 + s2 - 1;
    behz_base bb;
    if (c->scheme != ORC_BFV || behz_base_init(c, L, &bb))
        return -1;
    size_t nS = bb.nBsk;
    orc_tab *stab = (orc_tab *)calloc(nS, sizeof(orc_tab));
    for (size_t i = 0; i < nS; i++)
        if (tab_init(&stab[i], n, bb.Bsk[i]))
            return -1;
    /* steps (1)-(3), evaluator.cpp:456-474, for every input poly: those of a, then those of b */
    u64 *xq = (u64 *)malloc(nin * L * n * sizeof(u64)), *xs = (u64 *)malloc(nin * nS * n * sizeof(u64));
    u64 *lift = (u64 *)malloc((nS + 1) * n * sizeof(u64));
    for (size_t p = 0; p < nin; p++)
    {
        const u64 *src = p < s1 ? a + p * L * n : b + (p - s1) * L * n;
        for (size_t i = 0; i < L; i++)
        {
            memcpy(xq + (p * L + i) * n, src + i * n, n * sizeof(u64));
            ntt_fwd(&c->tab[i], n, xq + (p * L + i) * n);
        }
        orc_behz_fastbconv_m_tilde(n, c->q, L, c->t, src, lift);
        orc_behz_sm_mrq(n, c->q, L, c->t, lift, xs + p * nS * n);
        for (size_t s = 0; s < nS; s++)
            ntt_fwd(&stab[s], n, xs + (p * nS + s) * n);
    }
    /* step (4) tensor, :497-541; (5) INTT :545-546; (6) times t :554-556 */
    u64 *dq = (u64 *)malloc(nout * L * n * sizeof(u64)), *ds = (u64 *)malloc(nout * nS * n * sizeof(u64));
    for (int base = 0; base < 2; base++)
    {
        size_t nb = base ? nS : L;
        u64 *x = base ? xs : xq, *d = base ? ds : dq;
        tensor_rows(x, s1, x + s1 * nb * n, s2, nb, n, base ? bb.Bsk : c->q, d);
        for (size_t i = 0; i < nb; i++)
        {
            u64 P = base ? bb.Bsk[i] : c->q[i];
            const orc_tab *t = base ? &stab[i] : &c->tab[i];
            for (size_t p = 0; p < nout; p++)
            {
                ntt_inv(t, n, d + (p * nb + i) * n);
                for (size_t j = 0; j < n; j++)
                    d[(p * nb + i) * n + j] = mulmod(d[(p * nb + i) * n + j], c->t % P, P);
            }
        }
    }
    /* steps (7) fast_floor rns.cpp:1041-1084 and (8) fastbconv_sk rns.cpp:903-977 */
    u64 *qs = (u64 *)malloc((L + nS) * n * sizeof(u64)), *f = (u64 *)malloc(nS * n * sizeof(u64));
    for (size_t p = 0; p < nout; p++)
    {
        memcpy(qs, dq + p * L * n, L * n * sizeof(u64));
        memcpy(qs + L * n, ds + p * nS * n, nS * n * sizeof(u64));
        orc_behz_fast_floor(n, c->q, L, c->t, qs, f);
        orc_behz_fastbconv_sk(n, c->q, L, c->t, f, out3 + p * L * n);
    }
    free(qs), free(f), free(dq), free(ds), free(xq), free(xs), free(lift);
    for (size_t i = 0; i < nS; i++)
        tab_free(&stab[i]);
    free(stab);
    return 0;
}

/* ------------------------------------------------------------------------------ decryption (decryptor.cpp) -- */
/* dot_product_ct_sk_array (decryptor.cpp:312-384): phase = c_0 + sum_{p>=1} c_p * s^p, in the ciphertext's own form.
 * sk = the secret key in NTT form at the key level, [k][n]. */
void orc_decrypt_phase(const orc_ctx *c, size_t L, size_t size, int ct_is_ntt, const u64 *ct, const u64 *sk, u64 *out)
{
    size_t n = c->n;
    u64 *pw = (u64 *)malloc(n * sizeof(u64)), *tmp = (u64 *)malloc(n * sizeof(u64)), *acc = (u64 *)malloc(n * sizeof(u64));
    for (size_t i = 0; i < L; i++)
    {
        u64 q = c->q[i];
        memset(acc, 0, n * sizeof(u64));
        for (size_t j = 0; j < n; j++)
            pw[j] = 1;
        for (size_t p = 1; p < size; p++)
        {
            for (size_t j = 0; j < n; j++)
                pw[j] = mulmod(pw[j], sk[i * n + j], q); /* s^p, compute_secret_key_array :245-310 */
            memcpy(tmp, ct + (p * L + i) * n, n * sizeof(u64));
            if (!ct_is_ntt)
                ntt_fwd(&c->tab[i], n, tmp);
            for (size_t j = 0; j < n; j++)
                acc[j] = addmod(acc[j], mulmod(tmp[j], pw[j], q), q);
        }
        if (!ct_is_ntt)
            ntt_inv(&c->tab[i], n, acc);
        for (size_t j = 0; j < n; j++)
            out[i * n + j] = addmod(acc[j], ct[i * n + j], q);
    }
    free(pw), free(tmp), free(acc);
}

/* Decryptor::bfv_decrypt (decryptor.cpp:111-135) = phase + RNSTool::decrypt_scale_and_round (rns.cpp:1133-1191) */
int orc_bfv_decrypt(const orc_ctx *c, size_t L, size_t size, const u64 *ct, const u64 *sk, u64 *plain)
{
    size_t n = c->n;
    u64 t = c->t, primes[2];
    if (orc_get_primes(2 * (u64)n, 61, 2, primes))
        return -1;
    u64 gamma = primes[1], base[2] = { t, gamma };
    u64 *phase = (u64 *)malloc(L * n * sizeof(u64)), *conv = (u64 *)malloc(2 * n * sizeof(u64));
    orc_decrypt_phase(c, L, size, 0, ct, sk, phase);
    for (size_t i = 0; i < L; i++) /* :1155-1158  |gamma * t|_{q_i} * ct(s) */
    {
        u64 f = mulmod(t % c->q[i], gamma % c->q[i], c->q[i]);
        for (size_t j = 0; j < n; j++)
            phase[i * n + j] = mulmod(phase[i * n + j], f, c->q[i]);
    }
    for (int b = 0; b < 2; b++) /* :1164 FastBConv q -> {t, gamma}; :1167-1171 times -q^-1 */
    {
        u64 p = base[b], inv = 0;
        fastbconv(c->q, L, phase, n, n, p, conv + b * n);
        invmod(prod_mod(c->q, L, (size_t)-1, p), p, &inv);
        for (size_t j = 0; j < n; j++)
            conv[b * n + j] = mulmod(conv[b * n + j], submod(0, inv, p), p);
    }
    u64 inv_gamma = 0;
    invmod(gamma % t, t, &inv_gamma);
    for (size_t j = 0; j < n; j++) /* :1175-1190 */
    {
        u64 g = conv[n + j], r;
        if (g > (gamma >> 1))
            r = addmod(conv[j], (gamma - g) % t, t);
        else
            r = submod(conv[j], g % t, t);
        plain[j] = mulmod(r, inv_gamma, t);
    }
    free(phase), free(conv);
    return 0;
}

/* Decryptor::bgv_decrypt (decryptor.cpp:159-197): phase, INTT, BaseConverter::exact_convert_array (rns.cpp:466-539, in
 * IEEE doubles, summed in index order), times the inverse correction factor */
int orc_bgv_decrypt(const orc_ctx *c, size_t L, size_t size, u64 correction_factor, const u64 *ct, const u64 *sk, u64 *plain)
{
    size_t n = c->n;
    u64 t = c->t;
    u64 *phase = (u64 *)malloc(L * n * sizeof(u64));
    orc_decrypt_phase(c, L, size, 1, ct, sk, phase);
    for (size_t i = 0; i < L; i++)
        ntt_inv(&c->tab[i], n, phase + i * n);
    u64 inv[ORC_MAX_PRIMES + 2], mat[ORC_MAX_PRIMES + 2], q_mod_t = prod_mod(c->q, L, (size_t)-1, t), fix = 1;
    for (size_t i = 0; i < L; i++)
    {
        inv[i] = 0;
        invmod(prod_mod(c->q, L, i, c->q[i]), c->q[i], &inv[i]);
        mat[i] = prod_mod(c->q, L, i, t);
    }
    if (correction_factor != 1 && !invmod(correction_factor % t, t, &fix))
        return -1; /* "invalid correction factor", decryptor.cpp:186-189 */
    for (size_t j = 0; j < n; j++)
    {
        volatile double v = 0.0; /* sequential double additions, :519-523 */
        u128 sum = 0;
        for (size_t i = 0; i < L; i++)
        {
            u64 x = mulmod(phase[i * n + j], inv[i], c->q[i]); /* :494-513 (operand 1: the same value) */
            v = v + (double)x / (double)c->q[i];
            sum = (sum + (u128)x * mat[i]) % t;
        }
        v = v + 0.5;
        u64 rounded = (u64)v; /* :524-525 */
        u64 r = submod((u64)sum, mulmod(rounded % t, q_mod_t, t), t); /* :532-537 */
        plain[j] = mulmod(r, fix, t);
    }
    free(phase);
    return 0;
}


/* ---- seed-compressed ciphertexts --------------------------------------------------------------------------------------
 * BLAKE2b / BLAKE2Xb restated from RFC 7693 and the BLAKE2X specification (the reference vendors the BLAKE2 team's
 * reference code as util/blake2b.c, util/blake2xb.c); parameter block layout: digest_length, key_length, fanout, depth,
 * leaf_length (4), node_offset (4), xof_length (4), node_depth, inner_length, reserved (14), salt (16), personal (16). */
static const uint64_t b2_iv[8] = { 0x6a09e667f3bcc908ULL, 0xbb67ae8584caa73bULL, 0x3c6ef372fe94f82bULL, 0xa54ff53a5f1d36f1ULL,
                                   0x510e527fade682d1ULL, 0x9b05688c2b3e6c1fULL, 0x1f83d9abfb41bd6bULL, 0x5be0cd19137e2179ULL };
static const unsigned char b2_sigma[10][16] = {
    { 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15 }, { 14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3 },
    { 11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4 }, { 7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8 },
    { 9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13 }, { 2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9 },
    { 12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11 }, { 13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10 },
    { 6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5 }, { 10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0 }
};
static uint64_t b2_rotr(uint64_t v, int s)
{
    return (v >> s) | (v << (64 - s));
}
static void b2_compress(uint64_t h[8], const uint64_t m[16], uint64_t t, int last)
{
    uint64_t v[16];
    for (int i = 0; i < 8; i++)
        v[i] = h[i], v[i + 8] = b2_iv[i];
    v[12] ^= t;
    if (last)
        v[14] = ~v[14];
    for (int r = 0; r < 12; r++)
    {
        const unsigned char *s = b2_sigma[r % 10];
        static const int idx[8][4] = { { 0, 4, 8, 12 }, { 1, 5, 9, 13 }, { 2, 6, 10, 14 }, { 3, 7, 11, 15 },
                                       { 0, 5, 10, 15 }, { 1, 6, 11, 12 }, { 2, 7, 8, 13 }, { 3, 4, 9, 14 } };
        for (int g = 0; g < 8; g++)
        {
            const int a = idx[g][0], b = idx[g][1], c = idx[g][2], d = idx[g][3];
            v[a] += v[b] + m[s[2 * g]], v[d] = b2_rotr(v[d] ^ v[a], 32);
            v[c] += v[d], v[b] = b2_rotr(v[b] ^ v[c], 24);
            v[a] += v[b] + m[s[2 * g + 1]], v[d] = b2_rotr(v[d] ^ v[a], 16);
            v[c] += v[d], v[b] = b2_rotr(v[b] ^ v[c], 63);
        }
    }
    for (int i = 0; i < 8; i++)
        h[i] ^= v[i] ^ v[i + 8];
}
/* one PRNG buffer: 4096 bytes = BLAKE2Xb(in = counter, key = seed) (randomgen.cpp:204-214, util/blake2xb.c) */
static void b2x_buffer(const uint64_t seed[8], uint64_t counter, uint64_t out[512])
{
    uint64_t h[8], m[16];
    for (int i = 0; i < 8; i++)
        h[i] = b2_iv[i];
    h[0] ^= 64ULL | (64ULL << 8) | (1ULL << 16) | (1ULL << 24); /* digest 64, key 64, fanout 1, depth 1 */
    h[1] ^= 4096ULL << 32;                                       /* node_offset 0, xof_length 4096 */
    for (int i = 0; i < 8; i++)
        m[i] = seed[i], m[i + 8] = 0;
    b2_compress(h, m, 128, 0); /* the key block */
    memset(m, 0, sizeof(m));
    m[0] = counter;
    b2_compress(h, m, 136, 1); /* the 8-byte message */
    for (uint64_t node = 0; node < 64; node++)
    {
        uint64_t o[8];
        for (int i = 0; i < 8; i++)
            o[i] = b2_iv[i], m[i] = h[i], m[i + 8] = 0;
        o[0] ^= 64ULL | (64ULL << 32);   /* digest 64, key 0, fanout 0, depth 0, leaf_length 64 */
        o[1] ^= node | (4096ULL << 32);  /* node_offset, xof_length */
        o[2] ^= 64ULL << 8;              /* node_depth 0, inner_length 64 */
        b2_compress(o, m, 64, 1);
        memcpy(out + 8 * node, o, 64);
    }
}
void orc_blake2xb_stream(const uint64_t seed[8], size_t words, uint64_t *out)
{
    uint64_t buf[512];
    for (size_t w = 0, counter = 0; w < words; counter++)
    {
        b2x_buffer(seed, counter, buf);
        const size_t take = words - w < 512 ? words - w : 512;
        memcpy(out + w, buf, take * 8);
        w += take;
    }
}
void orc_expand_seed(const orc_ctx *c, size_t L, const uint64_t seed[8], uint64_t *out)
{
    /* util/rlwe.cpp:104-132: fill all L*n words from the stream, then replace every word >= max_multiple of its prime, in
       coefficient order, by further words of the same stream; reduce modulo the prime */
    const size_t n = c->n, need = L * n;
    uint64_t buf[512];
    size_t counter = 0, head = 512;
    for (size_t i = 0; i < need; i++)
    {
        if (head == 512)
            b2x_buffer(seed, counter++, buf), head = 0;
        out[i] = buf[head++];
    }
    for (size_t j = 0; j < L; j++)
    {
        const uint64_t q = c->q[j], max_random = ~0ULL, max_multiple = max_random - max_random % q - 1;
        for (size_t i = 0; i < n; i++)
        {
            uint64_t r = out[j * n + i];
            while (r >= max_multiple)
            {
                if (head == 512)
                    b2x_buffer(seed, counter++, buf), head = 0;
                r = buf[head++];
            }
            out[j * n + i] = r % q;
        }
    }
}


/* ---- symmetric-key encryption of zero (util/rlwe.cpp:264-408, encrypt_zero_symmetric) -----------------------------------
 * bootstrap PRNG = Blake2xbPRNG(seed): its first 64 bytes are the public seed of the PRNG that samples c_1 (sample_poly_uniform),
 * the following 6 bytes per coefficient feed the centred binomial noise (sample_poly_cbd, rlwe.cpp:73-102).
 * (c_0, c_1) = (-(c_1 s + e), c_1) [BFV, CKKS], (-(c_1 s + t e), c_1) [BGV].  BFV ciphertexts are in coefficient form: with
 * save_seed the sampled polynomial IS c_1 (coefficient form, re-created from the seed at load time), without it the sampled
 * polynomial is taken to be NTT(c_1).  sk = secret key, NTT form, [k][n]; out = [2][L][n] at the level with L primes (symmetric
 * encryption at a lower level samples at that level directly: Encryptor::encrypt_zero_internal, encryptor.cpp:168-173). */
static int cbd_noise(const unsigned char x[6])
{
    static const unsigned char pop[16] = { 0, 1, 1, 2, 1, 2, 2, 3, 1, 2, 2, 3, 2, 3, 3, 4 };
#define HW(b) (pop[(b) & 15] + pop[(b) >> 4])
    return HW(x[0]) + HW(x[1]) + HW(x[2] & 0x1F) - HW(x[3]) - HW(x[4]) - HW(x[5] & 0x1F);
#undef HW
}
void orc_encrypt_zero_symmetric(const orc_ctx *c, size_t L, const uint64_t *sk, const uint64_t seed[8], int save_seed, uint64_t *out2)
{
    const size_t n = c->n;
    const int ntt_form = c->scheme != ORC_BFV;
    /* bootstrap stream: 64 bytes of public seed, then 6 bytes per coefficient */
    const size_t bwords = (64 + 6 * n + 7) / 8;
    u64 *boot = (u64 *)malloc(bwords * sizeof(u64));
    orc_blake2xb_stream(seed, bwords, boot);
    u64 *c0 = out2, *c1 = out2 + L * n;
    orc_expand_seed(c, L, boot, c1); /* the first 8 words are the public seed */
    u64 *c1n = (u64 *)malloc(L * n * sizeof(u64));
    memcpy(c1n, c1, L * n * sizeof(u64));
    if (!ntt_form)
    {
        if (save_seed)
            for (size_t j = 0; j < L; j++)
                ntt_fwd(&c->tab[j], n, c1n + j * n); /* the sample is c_1 itself: transform a copy for the product */
        else
            for (size_t j = 0; j < L; j++)
                ntt_inv(&c->tab[j], n, c1 + j * n);  /* the sample is NTT(c_1): c_1 is its inverse transform */
    }
    const unsigned char *bytes = (const unsigned char *)boot + 64;
    u64 *e = (u64 *)malloc(n * sizeof(u64));
    for (size_t j = 0; j < L; j++)
    {
        const u64 q = c->q[j];
        for (size_t i = 0; i < n; i++)
        {
            const int noise = cbd_noise(bytes + 6 * i);
            e[i] = noise >= 0 ? (u64)noise : q - (u64)(-noise);
            c0[j * n + i] = mulmod(sk[j * n + i], c1n[j * n + i], q);
        }
        if (ntt_form)
            ntt_fwd(&c->tab[j], n, e);
        else
            ntt_inv(&c->tab[j], n, c0 + j * n);
        for (size_t i = 0; i < n; i++)
        {
            u64 en = e[i];
            if (c->scheme == ORC_BGV)
                en = mulmod(en, c->t % q, q);
            const u64 v = addmod(c0[j * n + i], en, q);
            c0[j * n + i] = v ? q - v : 0;
        }
    }
    free(e);
    free(c1n);
    free(boot);
}


/* ---- CKKSEncoder (ckks.h:455-807, ckks.cpp:20-76; util/croots.cpp; util/dwthandler.h) ----------------------------------------
 * Floating point: every operation below is one IEEE double operation in the order the reference performs it (std::complex
 * products expand to (ac - bd, ad + bc)); compiled without FMA contraction the results are bit-identical. */
typedef struct
{
    double re, im;
} cplx;
/* std::complex<double> * std::complex<double> as C99 Annex G (G.5.1) specifies it and g++ compiles it: (ac - bd, ad + bc), and
 * when both parts come out NaN the infinities are recovered (an infinite factor is "boxed" to +-1 / +-0 with the other factor's
 * NaNs made 0, or, when only a partial product overflowed, every NaN is made 0) and the product recomputed times infinity.  This
 * only changes non-finite results: a decoded slot the naive formula would make NaN can be +-inf. */
static cplx c_mul(cplx z, cplx w)
{
    double a = z.re, b = z.im, c = w.re, d = w.im;
    const double ac = a * c, bd = b * d, ad = a * d, bc = b * c;
    cplx r = { ac - bd, ad + bc };
    if (isnan(r.re) && isnan(r.im))
    {
        int recalc = 0;
        if (isinf(a) || isinf(b))
        {
            a = copysign(isinf(a) ? 1.0 : 0.0, a), b = copysign(isinf(b) ? 1.0 : 0.0, b);
            if (isnan(c))
                c = copysign(0.0, c);
            if (isnan(d))
                d = copysign(0.0, d);
            recalc = 1;
        }
        if (isinf(c) || isinf(d))
        {
            c = copysign(isinf(c) ? 1.0 : 0.0, c), d = copysign(isinf(d) ? 1.0 : 0.0, d);
            if (isnan(a))
                a = copysign(0.0, a);
            if (isnan(b))
                b = copysign(0.0, b);
            recalc = 1;
        }
        if (!recalc && (isinf(ac) || isinf(bd) || isinf(ad) || isinf(bc)))
        {
            if (isnan(a))
                a = copysign(0.0, a);
            if (isnan(b))
                b = copysign(0.0, b);
            if (isnan(c))
                c = copysign(0.0, c);
            if (isnan(d))
                d = copysign(0.0, d);
            recalc = 1;
        }
        if (recalc)
            r.re = INFINITY * (a * c - b * d), r.im = INFINITY * (a * d + b * c);
    }
    return r;
}
/* util/croots.cpp:16-70: one eighth of the m-th roots from polar(), the rest through the 8-fold symmetry */
static cplx croot(const cplx *eighth, size_t m, size_t index)
{
    index &= m - 1;
    cplx r;
    if (index <= m / 8)
        return eighth[index];
    if (index <= m / 4)
    {
        cplx a = eighth[m / 4 - index];
        r.re = a.im, r.im = a.re;
        return r;
    }
    if (index <= m / 2)
    {
        cplx a = croot(eighth, m, m / 2 - index);
        r.re = -a.re, r.im = -(-a.im); /* -conj(a) */
        return r;
    }
    if (index <= 3 * m / 4)
    {
        cplx a = croot(eighth, m, index - m / 2);
        r.re = -a.re, r.im = -a.im;
        return r;
    }
    cplx a = croot(eighth, m, m - index);
    r.re = a.re, r.im = -a.im;
    return r;
}
/* ckks.cpp:33-73: the slot -> coefficient index map and the (inverse) root powers in the order the transforms consume them */
static void ckks_tables(size_t n, size_t *map, cplx *roots, cplx *inv_roots)
{
    const int logn = ilog2(n);
    const size_t slots = n >> 1;
    const u64 m = (u64)n << 1;
    u64 pos = 1;
    for (size_t i = 0; i < slots; i++)
    {
        const u64 index1 = (pos - 1) >> 1, index2 = (m - pos - 1) >> 1;
        map[i] = (size_t)reverse_bits(index1, logn);
        map[slots | i] = (size_t)reverse_bits(index2, logn);
        pos = (pos * 3) & (m - 1);
    }
    roots[0].re = roots[0].im = inv_roots[0].re = inv_roots[0].im = 0;
    if (m >= 8)
    {
        const double PI = 3.1415926535897932384626433832795028842;
        cplx *eighth = (cplx *)malloc((m / 8 + 1) * sizeof(cplx));
        for (size_t i = 0; i <= m / 8; i++)
        {
            const double theta = 2 * PI * (double)i / (double)m;
            eighth[i].re = 1.0 * cos(theta), eighth[i].im = 1.0 * sin(theta);
        }
        for (size_t i = 1; i < n; i++)
        {
            roots[i] = croot(eighth, m, reverse_bits(i, logn));
            inv_roots[i] = croot(eighth, m, reverse_bits(i - 1, logn) + 1);
            inv_roots[i].im = -inv_roots[i].im;
        }
        free(eighth);
    }
    else if (m == 4)
    {
        roots[1].re = 0, roots[1].im = 1;
        inv_roots[1].re = 0, inv_roots[1].im = -1;
    }
}
/* DWTHandler::transform_from_rev with a scalar (dwthandler.h:207-311): Gentleman-Sande butterflies, the scaling merged into the
 * last stage */
static void fft_from_rev(cplx *v, size_t n, const cplx *roots, double scalar)
{
    size_t gap = 1, m = n >> 1;
    for (; m > 1; m >>= 1, gap <<= 1)
        for (size_t i = 0, offset = 0; i < m; i++, offset += gap << 1)
        {
            const cplx r = *++roots;
            for (size_t j = 0; j < gap; j++)
            {
                cplx *x = v + offset + j, *y = x + gap, u = *x, w = *y, d = { u.re - w.re, u.im - w.im };
                x->re = u.re + w.re, x->im = u.im + w.im;
                *y = c_mul(d, r);
            }
        }
    const cplx r = *++roots, sr = { r.re * scalar, r.im * scalar };
    for (size_t j = 0; j < gap; j++)
    {
        cplx *x = v + j, *y = x + gap, u = *x, w = *y, d = { u.re - w.re, u.im - w.im };
        x->re = (u.re + w.re) * scalar, x->im = (u.im + w.im) * scalar;
        *y = c_mul(d, sr);
    }
}
/* DWTHandler::transform_to_rev without a scalar (dwthandler.h:94-205): Cooley-Tukey butterflies */
static void fft_to_rev(cplx *v, size_t n, const cplx *roots)
{
    size_t gap = n >> 1, m = 1;
    for (; m <= (n >> 1); m <<= 1, gap >>= 1)
        for (size_t i = 0, offset = 0; i < m; i++, offset += gap << 1)
        {
            const cplx r = *++roots;
            for (size_t j = 0; j < gap; j++)
            {
                cplx *x = v + offset + j, *y = x + gap, u = *x, w = c_mul(*y, r);
                x->re = u.re + w.re, x->im = u.im + w.im;
                y->re = u.re - w.re, y->im = u.im - w.im;
            }
        }
}
/* CKKSEncoder::encode (vector of complex values, ckks.h:455-690): values = [count][2] doubles (re, im), count <= n/2;
 * out = [L][n] NTT form at the level with L primes.  Returns 0, or 1 = "encoded values are too large" / "scale out of bounds" /
 * "values must be finite". */
int orc_ckks_encode(const orc_ctx *c, size_t L, const double *values, size_t count, double scale, uint64_t *out)
{
    const size_t n = c->n, slots = n >> 1;
    const int total_bits = prod_bit_count(c->q, L);
    if (!isnormal(scale) || scale <= 0 || ((int)log2(scale) + 1 >= total_bits) || count > slots)
        return 1;
    for (size_t i = 0; i < 2 * count; i++)
        if (!isfinite(values[i]))
            return 1;
    size_t *map = (size_t *)malloc(n * sizeof(size_t));
    cplx *roots = (cplx *)malloc(n * sizeof(cplx)), *inv_roots = (cplx *)malloc(n * sizeof(cplx));
    cplx *v = (cplx *)calloc(n, sizeof(cplx));
    ckks_tables(n, map, roots, inv_roots);
    for (size_t i = 0; i < count; i++)
    {
        v[map[i]].re = values[2 * i], v[map[i]].im = values[2 * i + 1];
        v[map[i + slots]].re = values[2 * i], v[map[i + slots]].im = -values[2 * i + 1];
    }
    const double fix = scale / (double)n;
    fft_from_rev(v, n, inv_roots, fix);
    int rc = 0;
    double max_coeff = 0;
    for (size_t i = 0; i < n; i++)
    {
        const double a = fabs(v[i].re);
        if (isnan(a))
            rc = 1;
        max_coeff = a > max_coeff ? a : max_coeff;
    }
    if (!rc && !isfinite(max_coeff))
        rc = 1;
    if (!rc && (int)ceil(log2(max_coeff > 1.0 ? max_coeff : 1.0)) + 1 >= total_bits)
        rc = 1;
    for (size_t i = 0; !rc && i < n; i++)
    {
        /* the three decomposition branches of the reference (<= 64 bits, <= 128 bits, multi-precision) all reduce the exact
         * integer |round(coefficient)|: mantissa * 2^exponent here */
        double d = round(v[i].re);
        const int negative = signbit(d);
        d = fabs(d);
        int e = 0;
        u64 mant = 0;
        if (d >= 1)
        {
            const double f = frexp(d, &e); /* d = f 2^e, f in [0.5, 1) */
            mant = (u64)ldexp(f, 53);      /* exact: 53-bit integer */
            e -= 53;
            while (e < 0)                  /* d is an integer: the shifted-out bits are zero */
                mant >>= 1, e++;
        }
        for (size_t j = 0; j < L; j++)
        {
            const u64 q = c->q[j];
            u64 r = mulmod(mant % q, powmod(2, (u64)e, q), q);
            out[j * n + i] = negative && r ? q - r : r;
        }
    }
    for (size_t j = 0; !rc && j < L; j++)
        ntt_fwd(&c->tab[j], n, out + j * n);
    free(v), free(roots), free(inv_roots), free(map);
    return rc;
}
/* CKKSEncoder::decode (ckks.h:692-790): plain = [L][n] NTT form, scale = Plaintext::scale(); out = [n/2][2] doubles (re, im) */
int orc_ckks_decode(const orc_ctx *c, size_t L, const uint64_t *plain, double scale, double *out)
{
    const size_t n = c->n, slots = n >> 1;
    const int total_bits = prod_bit_count(c->q, L);
    if (!isnormal(scale) || scale <= 0 || ((int)log2(scale) >= total_bits))
        return 1;
    const double inv_scale = 1.0 / scale, two_pow_64 = 18446744073709551616.0;
    /* big integers of L words: Q = prod q_j, the punctured products Q / q_j, the threshold (Q + 1) / 2 (context.cpp:406-412) */
    u64 *Q = (u64 *)calloc(L + 1, sizeof(u64)), *punct = (u64 *)calloc(L * (L + 1), sizeof(u64)), *thr = (u64 *)calloc(L + 1, sizeof(u64));
    u64 *invp = (u64 *)calloc(L, sizeof(u64));
    for (size_t j = 0; j <= L; j++)
    {
        u64 *dst = j < L ? punct + j * (L + 1) : Q;
        dst[0] = 1;
        for (size_t i = 0; i < L; i++)
        {
            if (i == j)
                continue;
            u64 carry = 0;
            for (size_t w = 0; w < L; w++)
            {
                const u128 t = (u128)dst[w] * c->q[i] + carry;
                dst[w] = (u64)t, carry = (u64)(t >> 64);
            }
        }
        if (j < L)
        {
            u64 pm = 1;
            for (size_t i = 0; i < L; i++)
                if (i != j)
                    pm = mulmod(pm, c->q[i] % c->q[j], c->q[j]);
            invp[j] = powmod(pm, c->q[j] - 2, c->q[j]);
        }
    }
    {
        u64 carry = 1; /* (Q + 1) >> 1 */
        for (size_t w = 0; w < L; w++)
        {
            const u64 t = Q[w] + carry;
            carry = t < carry;
            thr[w] = t;
        }
        for (size_t w = 0; w < L; w++)
            thr[w] = (thr[w] >> 1) | (w + 1 < L ? thr[w + 1] << 63 : carry << 63);
    }
    u64 *coef = (u64 *)malloc(L * n * sizeof(u64));
    memcpy(coef, plain, L * n * sizeof(u64));
    for (size_t j = 0; j < L; j++)
        ntt_inv(&c->tab[j], n, coef + j * n);
    size_t *map = (size_t *)malloc(n * sizeof(size_t));
    cplx *roots = (cplx *)malloc(n * sizeof(cplx)), *inv_roots = (cplx *)malloc(n * sizeof(cplx));
    cplx *res = (cplx *)calloc(n, sizeof(cplx));
    ckks_tables(n, map, roots, inv_roots);
    u64 *val = (u64 *)malloc((L + 1) * sizeof(u64)), *tmp = (u64 *)malloc((L + 1) * sizeof(u64));
    for (size_t i = 0; i < n; i++)
    {
        /* RNSBase::compose (rns.cpp:321-352): sum_j [x_j (Q/q_j)^-1 mod q_j] (Q/q_j) mod Q */
        memset(val, 0, (L + 1) * sizeof(u64));
        for (size_t j = 0; j < L; j++)
        {
            const u64 t = mulmod(coef[j * n + i], invp[j], c->q[j]);
            u64 carry = 0;
            for (size_t w = 0; w < L; w++)
            {
                const u128 p = (u128)punct[j * (L + 1) + w] * t + carry;
                tmp[w] = (u64)p, carry = (u64)(p >> 64);
            }
            u64 cy = 0;
            for (size_t w = 0; w < L; w++)
            {
                const u128 a = (u128)val[w] + tmp[w] + cy;
                val[w] = (u64)a, cy = (u64)(a >> 64);
            }
            int ge = cy != 0;
            if (!ge)
            {
                ge = 1;
                for (size_t w = L; w-- > 0;)
                    if (val[w] != Q[w])
                    {
                        ge = val[w] > Q[w];
                        break;
                    }
            }
            if (ge)
            {
                u64 bw = 0;
                for (size_t w = 0; w < L; w++)
                {
                    const u128 a = (u128)val[w] - Q[w] - bw;
                    val[w] = (u64)a, bw = (u64)(a >> 64) & 1;
                }
            }
        }
        int upper = 1;
        for (size_t w = L; w-- > 0;)
            if (val[w] != thr[w])
            {
                upper = val[w] > thr[w];
                break;
            }
        double acc = 0.0, s64 = inv_scale;
        for (size_t w = 0; w < L; w++, s64 *= two_pow_64)
        {
            if (upper)
            {
                if (val[w] > Q[w])
                {
                    const u64 diff = val[w] - Q[w];
                    acc += diff ? (double)diff * s64 : 0.0;
                }
                else
                {
                    const u64 diff = Q[w] - val[w];
                    acc -= diff ? (double)diff * s64 : 0.0;
                }
            }
            else
                acc += val[w] ? (double)val[w] * s64 : 0.0;
        }
        res[i].re = acc, res[i].im = 0.0;
    }
    fft_to_rev(res, n, roots);
    for (size_t i = 0; i < slots; i++)
        out[2 * i] = res[map[i]].re, out[2 * i + 1] = res[map[i]].im;
    free(val), free(tmp), free(res), free(roots), free(inv_roots), free(map), free(coef), free(Q), free(punct), free(thr), free(invp);
    return 0;
}


/* ---- public-key encryption of zero (Encryptor::encrypt_zero_internal, encryptor.cpp:88-174 -> util::encrypt_zero_asymmetric,
 * util/rlwe.cpp:184-276) --------------------------------------------------------------------------------------------------
 * One PRNG (Blake2xb of `seed`) yields, in this order: the ternary polynomial u (sample_poly_ternary, rlwe.cpp:21-39: one 32-bit
 * word per coefficient through std::uniform_int_distribution<uint64_t>(0, 2) -- libstdc++ >= 11 maps a 32-bit generator word r to
 * (r * 3) >> 32 and redraws when the low half of r * 3 is below 2^32 mod 3 = 1, i.e. for r == 0 only, bits/uniform_int_dist.h
 * _S_nd), then the noise polynomials e_0, e_1 (sample_poly_cbd, 6 bytes per coefficient).  c_j = pk_j u + e_j (BGV: t e_j) at
 * the level ABOVE the requested one (one more prime: the level's prev_context_data), followed by the scheme's
 * divide-and-round by that prime; at the key level (L == k) there is no level above and the sample is returned as is.
 * pk = [2][k][n] NTT form (PublicKey::data()); out = [2][L][n]. */
void orc_encrypt_zero_asymmetric(const orc_ctx *c, size_t L, const uint64_t *pk, const uint64_t seed[8], uint64_t *out2)
{
    const size_t n = c->n, k = c->k, Lp = L < k ? L + 1 : L;
    const int ntt_form = c->scheme != ORC_BFV;
    const size_t words = (4 * n + 12 * n + 7) / 8 + 64; /* spare words for (astronomically rare) ternary redraws */
    u64 *stream = (u64 *)malloc(words * sizeof(u64));
    orc_blake2xb_stream(seed, words, stream);
    const uint32_t *w32 = (const uint32_t *)stream;
    size_t pos = 0; /* in 32-bit words */
    u64 *u = (u64 *)malloc(Lp * n * sizeof(u64)), *t2 = (u64 *)malloc(2 * Lp * n * sizeof(u64)), *e = (u64 *)malloc(n * sizeof(u64));
    for (size_t i = 0; i < n; i++)
    {
        uint64_t product = (uint64_t)w32[pos++] * 3u;
        while ((uint32_t)product < 1u)
            product = (uint64_t)w32[pos++] * 3u;
        const u64 r = product >> 32;
        for (size_t j = 0; j < Lp; j++)
            u[j * n + i] = r + (r == 0 ? c->q[j] : 0) - 1;
    }
    for (size_t j = 0; j < Lp; j++)
        ntt_fwd(&c->tab[j], n, u + j * n);
    const unsigned char *bytes = (const unsigned char *)stream + 4 * pos;
    for (size_t p = 0; p < 2; p++)
        for (size_t j = 0; j < Lp; j++)
        {
            const u64 q = c->q[j];
            u64 *dst = t2 + (p * Lp + j) * n;
            const u64 *key = pk + (p * k + j) * n;
            for (size_t i = 0; i < n; i++)
                dst[i] = mulmod(u[j * n + i], key[i], q);
            if (!ntt_form)
                ntt_inv(&c->tab[j], n, dst);
            for (size_t i = 0; i < n; i++)
            {
                const int noise = cbd_noise(bytes + 6 * (p * n + i));
                e[i] = noise >= 0 ? (u64)noise : q - (u64)(-noise);
            }
            if (ntt_form)
                ntt_fwd(&c->tab[j], n, e);
            for (size_t i = 0; i < n; i++)
            {
                u64 en = e[i];
                if (c->scheme == ORC_BGV)
                    en = mulmod(en, c->t % q, q);
                dst[i] = addmod(dst[i], en, q);
            }
        }
    if (Lp == L)
        memcpy(out2, t2, 2 * L * n * sizeof(u64));
    else if (c->scheme == ORC_CKKS)
        orc_rescale(c, Lp, t2, out2);
    else if (c->scheme == ORC_BFV)
        orc_bfv_mod_switch(c, Lp, t2, out2);
    else
        orc_bgv_mod_switch(c, Lp, t2, out2);
    free(stream), free(u), free(t2), free(e);
}
