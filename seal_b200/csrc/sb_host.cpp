// seal_b200/csrc/sb_host.cpp -- host-side precomputation; see sb_host.hpp.
#include <complex>
#include "sb_host.hpp"
#include <algorithm>
#include <map>

namespace sbh
{
    u64 powmod(u64 a, u64 e, u64 q)
    {
        u64 r = 1 % q;
        a %= q;
        for (; e; e >>= 1)
        {
            if (e & 1)
                r = mulmod(r, a, q);
            a = mulmod(a, a, q);
        }
        return r;
    }

    bool invmod(u64 a, u64 m, u64 &out)
    {
        __int128 t = 0, nt = 1, r = m, nr = a % m;
        while (nr != 0)
        {
            __int128 qq = r / nr, tmp = t - qq * nt;
            t = nt, nt = tmp;
            tmp = r - qq * nr;
            r = nr, nr = tmp;
        }
        if (r != 1)
            return false;
        if (t < 0)
            t += m;
        out = static_cast<u64>(t);
        return true;
    }

    // Miller-Rabin with the first 12 primes as bases is exact below 3.3e24, i.e. for every 64-bit input.
    bool is_prime(u64 v)
    {
        static const u64 bases[] = { 2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37 };
        if (v < 2)
            return false;
        for (u64 b : bases)
        {
            if (v == b)
                return true;
            if (v % b == 0)
                return false;
        }
        u64 d = v - 1;
        int r = 0;
        while (!(d & 1))
            d >>= 1, r++;
        for (u64 b : bases)
        {
            u64 x = powmod(b, d, v);
            if (x == 1 || x == v - 1)
                continue;
            bool composite = true;
            for (int j = 1; j < r && composite; j++)
            {
                x = mulmod(x, x, v);
                if (x == v - 1)
                    composite = false;
            }
            if (composite)
                return false;
        }
        return true;
    }

    std::vector<u64> get_primes(u64 factor, int bit_size, std::size_t count)
    {
        std::vector<u64> out;
        u64 value = ((u64(1) << bit_size) - 1) / factor * factor + 1;
        const u64 lower = u64(1) << (bit_size - 1);
        while (out.size() < count && value > lower)
        {
            if (is_prime(value))
                out.push_back(value);
            value -= factor;
        }
        if (out.size() < count)
            throw std::logic_error("failed to find enough qualifying primes");
        return out;
    }

    std::vector<u64> coeff_modulus_create(std::size_t n, const std::vector<int> &bits)
    {
        std::map<int, std::size_t> counts;
        for (int b : bits)
            counts[b]++;
        std::map<int, std::vector<u64>> table;
        for (auto &kv : counts)
            table[kv.first] = get_primes(2 * static_cast<u64>(n), kv.first, kv.second);
        std::vector<u64> out;
        for (int b : bits)
        {
            out.push_back(table[b].back());
            table[b].pop_back();
        }
        return out;
    }

    bool minimal_primitive_root(u64 degree, u64 q, u64 &root)
    {
        if ((q - 1) % degree)
            return false;
        const u64 quot = (q - 1) / degree;
        u64 r = 0;
        for (u64 g = 2; g < 4096 && !r; g++)
        {
            u64 c = powmod(g, quot, q);
            if (powmod(c, degree >> 1, q) == q - 1)
                r = c;
        }
        if (!r)
            return false;
        // all primitive degree-th roots are the odd powers of r; keep the smallest
        const u64 rsq = mulmod(r, r, q);
        u64 cur = r, best = r;
        for (u64 i = 0; i < degree; i += 2)
        {
            best = std::min(best, cur);
            cur = mulmod(cur, rsq, q);
        }
        root = best;
        return true;
    }

    int product_bit_count(const u64 *q, std::size_t count)
    {
        std::vector<u64> limbs{ 1 };
        for (std::size_t i = 0; i < count; i++)
        {
            u64 carry = 0;
            for (auto &l : limbs)
            {
                u128 v = static_cast<u128>(l) * q[i] + carry;
                l = static_cast<u64>(v);
                carry = static_cast<u64>(v >> 64);
            }
            if (carry)
                limbs.push_back(carry);
        }
        int bits = 0;
        for (u64 top = limbs.back(); top; top >>= 1)
            bits++;
        return static_cast<int>(limbs.size() - 1) * 64 + bits;
    }

    static TwPair pair(u64 w, u64 q)
    {
        return TwPair{ w, shoup(w, q) };
    }

    void PrimeTables::build(std::size_t n, u64 modulus)
    {
        q = modulus;
        const int logn = ilog2(n);
        if (!minimal_primitive_root(2 * static_cast<u64>(n), q, root))
            throw std::invalid_argument("invalid modulus: no primitive 2n-th root of unity");
        u64 inv_root = 0;
        if (!invmod(root, q, inv_root))
            throw std::invalid_argument("invalid modulus");
        const u128 all = ~static_cast<u128>(0);
        const u128 ratio = all / q; // q is odd (or 2^32 never gets here) so floor((2^128-1)/q) = floor(2^128/q)
        ratio_lo = static_cast<u64>(ratio);
        ratio_hi = static_cast<u64>(ratio >> 64);

        root_powers.assign(n, TwPair{});
        inv_root_powers.assign(n, TwPair{});
        u64 p = root;
        for (std::size_t i = 1; i < n; i++)
        {
            root_powers[reverse_bits(i, logn)] = pair(p, q);
            p = mulmod(p, root, q);
        }
        root_powers[0] = pair(1, q);
        p = inv_root;
        for (std::size_t i = 1; i < n; i++)
        {
            inv_root_powers[reverse_bits(i - 1, logn) + 1] = pair(p, q);
            p = mulmod(p, inv_root, q);
        }
        inv_root_powers[0] = pair(1, q);

        u64 ninv = 0;
        if (!invmod(static_cast<u64>(n) % q, q, ninv))
            throw std::invalid_argument("invalid modulus");
        inv_n = pair(ninv, q);

        fwd = root_powers;
        inv.assign(n, TwPair{});
        inv[0] = pair(1, q);
        for (std::size_t m = 1; m < n; m <<= 1)
            for (std::size_t i = 0; i < m; i++)
                inv[m + i] = inv_root_powers[n - 2 * m + 1 + i];
        inv_n_w = pair(mulmod(ninv, n > 1 ? inv[1].w : 1, q), q);
    }

    static u64 prod_mod(const std::vector<u64> &base, std::size_t count, std::size_t skip, u64 p)
    {
        u64 r = 1 % p;
        for (std::size_t j = 0; j < count; j++)
            if (j != skip)
                r = mulmod(r, base[j] % p, p);
        return r;
    }
    static int bit_count(u64 v)
    {
        int b = 0;
        for (; v; v >>= 1)
            b++;
        return b;
    }

    std::size_t behz_base_size(const std::vector<u64> &q, std::size_t L, u64 t)
    {
        // rns.cpp:605-612: enlarge B by one prime when K*n*t*q^2 < q*prod(B)*m_sk would not hold
        if (32 + bit_count(t) + product_bit_count(q.data(), L) >= 61 * static_cast<int>(L) + 61)
            return L + 1;
        return L;
    }

    BehzLevel build_behz(std::size_t n, const std::vector<u64> &q, std::size_t L, u64 t)
    {
        BehzLevel b;
        b.L = L;
        b.nB = behz_base_size(q, L, t);
        b.nBsk = b.nB + 1;
        auto aux = get_primes(2 * static_cast<u64>(n), 61, b.nBsk + 1); // [m_sk, gamma, B...]  rns.cpp:626-632
        b.m_sk = aux[0];
        b.B.assign(aux.begin() + 2, aux.begin() + 2 + b.nB);
        b.Bsk = b.B;
        b.Bsk.push_back(b.m_sk);
        const u64 mt = u64(1) << 32;
        const std::size_t none = static_cast<std::size_t>(-1);
        auto inv_or_throw = [](u64 a, u64 m) {
            u64 r = 0;
            if (!invmod(a, m, r))
                throw std::logic_error("invalid rns bases");
            return r;
        };
        for (std::size_t i = 0; i < L; i++)
        {
            b.inv_punc_q.push_back(pair(inv_or_throw(prod_mod(q, L, i, q[i]), q[i]), q[i]));
            b.q_to_mtilde.push_back(prod_mod(q, L, i, mt));
            b.mtilde_mod_q.push_back(pair(mt % q[i], q[i]));
            b.t_mod_q.push_back(pair(t % q[i], q[i]));
            u64 pb = prod_mod(b.B, b.nB, none, q[i]);
            b.prod_B_mod_q.push_back(pair(pb, q[i]));
            b.neg_prod_B_mod_q.push_back(pair((q[i] - pb) % q[i], q[i]));
        }
        b.q_to_Bsk.resize(b.nBsk * L);
        for (std::size_t s = 0; s < b.nBsk; s++)
        {
            const u64 P = b.Bsk[s];
            for (std::size_t i = 0; i < L; i++)
                b.q_to_Bsk[s * L + i] = prod_mod(q, L, i, P);
            const u64 qP = prod_mod(q, L, none, P);
            b.prod_q_mod_Bsk.push_back(pair(qP, P));
            b.inv_q_mod_Bsk.push_back(pair(inv_or_throw(qP, P), P));
            b.inv_mtilde_mod_Bsk.push_back(pair(inv_or_throw(mt % P, P), P));
            b.t_mod_Bsk.push_back(pair(t % P, P));
        }
        b.neg_inv_q_mod_mtilde = (mt - inv_or_throw(prod_mod(q, L, none, mt), mt)) % mt;
        for (std::size_t i = 0; i < b.nB; i++)
        {
            b.inv_punc_B.push_back(pair(inv_or_throw(prod_mod(b.B, b.nB, i, b.B[i]), b.B[i]), b.B[i]));
            b.B_to_msk.push_back(prod_mod(b.B, b.nB, i, b.m_sk));
        }
        b.B_to_q.resize(L * b.nB);
        for (std::size_t j = 0; j < L; j++)
            for (std::size_t i = 0; i < b.nB; i++)
                b.B_to_q[j * b.nB + i] = prod_mod(b.B, b.nB, i, q[j]);
        b.inv_B_mod_msk = pair(inv_or_throw(prod_mod(b.B, b.nB, none, b.m_sk), b.m_sk), b.m_sk);
        return b;
    }

    std::uint32_t galois_elt_from_step(std::size_t n, int step)
    {
        const u64 m = 2 * static_cast<u64>(n);
        if (step == 0)
            return static_cast<std::uint32_t>(m - 1);
        const bool neg = step < 0;
        const u64 pos = static_cast<u64>(neg ? -static_cast<long long>(step) : step);
        if (pos >= (n >> 1))
            throw std::invalid_argument("step count too large");
        u64 s = neg ? (n >> 1) - pos : pos;
        u64 e = 1;
        while (s--)
            e = (e * 3) & (m - 1);
        return static_cast<std::uint32_t>(e);
    }

    std::vector<std::uint32_t> batch_index_map(std::size_t n)
    {
        // slots of row 0 sit at the powers 3^i of the generator, row 1 at their negatives; positions are taken in the
        // bit-reversed order the transform produces
        const int logn = ilog2(n);
        const std::size_t row = n >> 1;
        const u64 m = static_cast<u64>(n) << 1;
        std::vector<std::uint32_t> map(n);
        u64 pos = 1;
        for (std::size_t i = 0; i < row; i++)
        {
            map[i] = static_cast<std::uint32_t>(reverse_bits((pos - 1) >> 1, logn));
            map[row | i] = static_cast<std::uint32_t>(reverse_bits((m - pos - 1) >> 1, logn));
            pos = (pos * 3) & (m - 1);
        }
        return map;
    }

    std::vector<std::uint32_t> galois_table_ntt(std::size_t n, std::uint32_t elt)
    {
        const int logn = ilog2(n);
        std::vector<std::uint32_t> t(n);
        for (std::size_t i = 0; i < n; i++)
        {
            u64 rev = reverse_bits(i + n, logn + 1);
            u64 raw = ((static_cast<u64>(elt) * rev) >> 1) & (n - 1);
            t[i] = static_cast<std::uint32_t>(reverse_bits(raw, logn));
        }
        return t;
    }

    // ---- CKKSEncoder tables ----
    namespace
    {
        using cd = std::complex<double>;
        // ComplexRoots::get_root (util/croots.cpp:41-70)
        cd complex_root(const std::vector<cd> &eighth, std::size_t m, std::size_t index)
        {
            index &= m - 1;
            if (index <= m / 8)
                return eighth[index];
            if (index <= m / 4)
            {
                const cd a = eighth[m / 4 - index];
                return cd(a.imag(), a.real());
            }
            if (index <= m / 2)
                return -std::conj(complex_root(eighth, m, m / 2 - index));
            if (index <= 3 * m / 4)
                return -complex_root(eighth, m, index - m / 2);
            return std::conj(complex_root(eighth, m, m - index));
        }
    } // namespace

    CkksTables ckks_tables(std::size_t n)
    {
        const int logn = ilog2(n);
        const std::size_t m = n << 1;
        CkksTables t;
        t.roots.assign(2 * n, 0.0);
        t.inv_roots.assign(2 * n, 0.0);
        if (m >= 8)
        {
            constexpr double PI = 3.1415926535897932384626433832795028842; // ComplexRoots::PI_ (util/croots.h)
            std::vector<cd> eighth(m / 8 + 1);
            for (std::size_t i = 0; i <= m / 8; i++)
                eighth[i] = std::polar<double>(1.0, 2 * PI * static_cast<double>(i) / static_cast<double>(m));
            for (std::size_t i = 1; i < n; i++)
            {
                const cd r = complex_root(eighth, m, reverse_bits(i, logn));
                const cd ir = std::conj(complex_root(eighth, m, reverse_bits(i - 1, logn) + 1));
                t.roots[2 * i] = r.real(), t.roots[2 * i + 1] = r.imag();
                t.inv_roots[2 * i] = ir.real(), t.inv_roots[2 * i + 1] = ir.imag();
            }
        }
        else if (m == 4)
        {
            t.roots[3] = 1.0;
            t.inv_roots[3] = -1.0;
        }
        return t;
    }

    CkksLevelHost ckks_level(const u64 *q, std::size_t L)
    {
        CkksLevelHost h;
        h.total_bits = product_bit_count(q, L);
        auto product_without = [&](std::size_t skip, u64 *dst) {
            std::vector<u64> acc(L + 1, 0);
            acc[0] = 1;
            for (std::size_t i = 0; i < L; i++)
            {
                if (i == skip)
                    continue;
                u64 carry = 0;
                for (std::size_t w = 0; w <= L; w++)
                {
                    const u128 v = static_cast<u128>(acc[w]) * q[i] + carry;
                    acc[w] = static_cast<u64>(v), carry = static_cast<u64>(v >> 64);
                }
            }
            for (std::size_t w = 0; w < L; w++)
                dst[w] = acc[w];
        };
        h.Q.resize(L), h.threshold.resize(L), h.punctured.resize(L * L), h.inv_punctured.resize(L);
        product_without(L, h.Q.data());
        for (std::size_t j = 0; j < L; j++)
        {
            product_without(j, h.punctured.data() + j * L);
            u64 pm = 1;
            for (std::size_t i = 0; i < L; i++)
                if (i != j)
                    pm = mulmod(pm, q[i] % q[j], q[j]);
            u64 inv = 0;
            invmod(pm, q[j], inv);
            h.inv_punctured[j] = pair(inv, q[j]);
        }
        // (Q + 1) >> 1
        u64 carry = 1;
        for (std::size_t w = 0; w < L; w++)
        {
            h.threshold[w] = h.Q[w] + carry;
            carry = h.threshold[w] < carry ? 1 : 0;
        }
        for (std::size_t w = 0; w < L; w++)
            h.threshold[w] = (h.threshold[w] >> 1) | ((w + 1 < L ? h.threshold[w + 1] : carry) << 63);
        return h;
    }
} // namespace sbh

// ---- key switching through an exact integer convolution: auxiliary 29-bit primes, their transforms' tables, CRT constants ----
#include <cmath>
namespace sbh
{
    KsIntHost build_ksint(std::size_t n, const u64 *q, std::size_t k)
    {
        KsIntHost h;
        const int logn = ilog2(n);
        if (logn < 12 || logn > 17 || k < 2)
            return h; // S = 0: not available
        h.r = logn - 12;
        // |sum_J d_J * k_JI| < L n max(q_J) max(q_I); the reconstruction needs P > 4 x that (fraction of P within (1/4, 3/4))
        u64 qmax = 0;
        for (std::size_t i = 0; i < k; i++)
            qmax = std::max(qmax, q[i]);
        const long double need = 2.0L + std::log2(static_cast<long double>(k - 1)) + logn + 2.0L * std::log2(static_cast<long double>(qmax)) + 0.01L;
        long double have = 0;
        u64 cand = ((u64(1) << 29) / (2 * n)) * (2 * n) + 1;
        while (have < need)
        {
            do
                cand -= 2 * n;
            while (cand > (u64(1) << 28) && !is_prime(cand));
            if (cand <= (u64(1) << 28) || h.p.size() >= 8)
                throw std::logic_error("not enough auxiliary primes");
            h.p.push_back(static_cast<std::uint32_t>(cand));
            have += std::log2(static_cast<long double>(cand));
        }
        const int S = h.S = static_cast<int>(h.p.size());
        const u64 pm1 = *std::max_element(h.p.begin(), h.p.end()) - 1;
        h.max_digits = static_cast<std::size_t>(~u64(0) / (pm1 * pm1));
        const std::size_t nb = std::size_t(1) << h.r;
        auto pair32 = [](u64 w, u64 p, std::uint32_t *dst) {
            dst[0] = static_cast<std::uint32_t>(w);
            dst[1] = static_cast<std::uint32_t>((w << 32) / p);
        };
        h.red.resize(2 * S), h.mu.resize(S), h.c1.resize(2 * S), h.c2.resize(S);
        h.fwd_outer.assign(S * nb * 2, 0), h.inv_outer.assign(S * nb * 2, 0);
        h.fwd_local.assign(S * n * 2, 0), h.inv_local.assign(S * n * 2, 0);
        std::vector<u64> rp(n), irp(n);
        for (int t = 0; t < S; t++)
        {
            const u64 p = h.p[t];
            u64 psi = 0, ipsi = 0;
            if (!minimal_primitive_root(2 * n, p, psi) || !invmod(psi, p, ipsi))
                throw std::logic_error("auxiliary prime without a 2n-th root");
            u64 pw = 1, ipw = 1;
            for (std::size_t e = 0; e < n; e++)
            {
                const std::size_t idx = reverse_bits(e, logn);
                rp[idx] = pw, irp[idx] = ipw;
                pw = mulmod(pw, psi, p), ipw = mulmod(ipw, ipsi, p);
            }
            pair32((u64(1) << 32) % p, p, &h.red[2 * t]);
            h.mu[t] = static_cast<std::uint32_t>((u64(1) << 32) / p);
            for (std::size_t e = 1; e < nb; e++)
            {
                pair32(rp[e], p, &h.fwd_outer[(t * nb + e) * 2]);
                pair32(irp[e], p, &h.inv_outer[(t * nb + e) * 2]);
            }
            for (std::size_t g = 0; g < nb; g++)
            {
                std::uint32_t *f = &h.fwd_local[(t * nb + g) * 4096 * 2], *v = &h.inv_local[(t * nb + g) * 4096 * 2];
                for (int s = 0; s < 12; s++)
                    for (std::size_t i = 0; i < (std::size_t(1) << s); i++)
                    {
                        const std::size_t src = (std::size_t(1) << (h.r + s)) + (g << s) + i;
                        std::size_t e = (std::size_t(1) << s) + i;
                        if (s >= 8)
                        {
                            const std::size_t per = std::size_t(1) << (s - 8), th = i / per, u = i % per;
                            e = 256 + (per - 1 + u) * 256 + th;
                        }
                        pair32(rp[src], p, f + 2 * e);
                        pair32(irp[src], p, v + 2 * e);
                    }
            }
            // CRT: (P/p_t)^-1 mod p_t
            u64 punct = 1;
            for (int u = 0; u < S; u++)
                if (u != t)
                    punct = mulmod(punct, h.p[u] % p, p);
            u64 inv_punct = 0, inv_n = 0;
            if (!invmod(punct, p, inv_punct) || !invmod(n % p, p, inv_n))
                throw std::logic_error("auxiliary primes are not coprime");
            pair32(mulmod(inv_n, inv_punct, p), p, &h.c1[2 * t]);
            h.c2[t] = static_cast<std::uint32_t>(mulmod((p - 1) / 2, inv_punct, p)); // H = (P-1)/2 = -1/2 mod p_t
        }
        h.punct_mod_q.resize(k * S), h.neg_mod_q.resize(k * S);
        for (std::size_t i = 0; i < k; i++)
        {
            const u64 qi = q[i];
            u64 Pq = 1;
            for (int t = 0; t < S; t++)
            {
                Pq = mulmod(Pq, h.p[t] % qi, qi);
                u64 v = 1;
                for (int u = 0; u < S; u++)
                    if (u != t)
                        v = mulmod(v, h.p[u] % qi, qi);
                h.punct_mod_q[i * S + t] = v;
            }
            u64 inv2 = 0;
            if (!invmod(2 % qi, qi, inv2))
                throw std::logic_error("even coefficient modulus");
            const u64 Hq = mulmod((Pq + qi - 1) % qi, inv2, qi);
            for (int a = 0; a < S; a++)
            {
                const u64 aP = mulmod(static_cast<u64>(a), Pq, qi);
                h.neg_mod_q[i * S + a] = (2 * qi - aP - Hq) % qi;
            }
        }
        return h;
    }
} // namespace sbh
