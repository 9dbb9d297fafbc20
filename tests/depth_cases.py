"""Inputs at the depth edges of decryption and the CKKS encoder, and the Python-integer facts each one exists for.  Shared by
test_depth_oracle.py (the oracle against the reference, CPU) and test_gpu_depth.py (the device against both).

BGV decryption rounds sum_i x_i / q_i + 0.5 in doubles (BaseConverter::exact_convert_array, rns.cpp:466-539): a phase next to Q / 2
puts the exact sum within Q^-1 2^21 of a half, so the result is decided by the double rounding in the reference's summation order.
BFV decryption rounds t v / Q: a noise of floor(Delta / 2) puts that within t^2 / Q of a half.  CKKS decode accumulates word w of
each composed coefficient times 2^(64 w) / scale, which is +inf once 64 w - log2(scale) >= 1024."""
import numpy as np

from common import crt_values, product, residue_rows


# ---- BGV: the centring edge ----
def bgv_edge_phases(Q, n, rng):
    """n phases: floor(Q/2), ceil(Q/2), then (Q - 1)/2 + d and (Q + 1)/2 + d alternating, d uniform in [-2^20, 2^20]"""
    out = [Q // 2, (Q + 1) // 2]
    d = rng.integers(-(1 << 20), (1 << 20) + 1, n)
    for j in range(2, n):
        out.append((Q - 1) // 2 + int(d[j]) if j % 2 else (Q + 1) // 2 + int(d[j]))
    return out


def assert_near_half(phases, Q, bits=40):
    """every phase v has |v / Q - 1/2| < 2^-bits"""
    for v in phases:
        assert abs(2 * (v % Q) - Q) << bits < Q, "a phase is not at the centring edge"


def exact_convert_rounding(phase_rows, moduli, reverse=False):
    """the rounded v of exact_convert_array for each column of the coefficient-form phase rows [L][n], in Python doubles: x_i =
    [phase_i (Q/q_i)^-1]_{q_i}, v = sum_i x_i / q_i summed in prime order (or reversed), + 0.5, truncated"""
    L = phase_rows.shape[0]
    Q = product(moduli[:L])
    xs = []
    for i in range(L):
        q = int(moduli[i])
        inv = pow((Q // q) % q, -1, q)
        xs.append([float(int(x) * inv % q) / float(q) for x in phase_rows[i]])
    order = range(L - 1, -1, -1) if reverse else range(L)
    out = []
    for j in range(phase_rows.shape[1]):
        v = 0.0
        for i in order:
            v += xs[i][j]
        out.append(int(v + 0.5))
    return out


def order_sensitive_count(phase_rows, moduli):
    """coefficients whose rounded sum changes when the primes are summed in reverse order"""
    fwd = exact_convert_rounding(phase_rows, moduli)
    rev = exact_convert_rounding(phase_rows, moduli, reverse=True)
    return sum(a != b for a, b in zip(fwd, rev))


# ---- BFV: structured phases Delta m + e ----
def bfv_noises(Delta):
    """noise terms: 0, +-1, +-floor(Delta/4) (decrypt to m) and the rounding edge +-floor(Delta/2), +-(floor(Delta/2) +- 1)"""
    h = Delta // 2
    return [0, 1, -1, Delta // 4, -(Delta // 4), h, -h, h + 1, h - 1, -(h + 1), -(h - 1)]


def bfv_phases(Q, t, n, rng):
    """(phases, m, e): phase_j = Delta m_j + e_j mod Q with m_j uniform below t and e_j cycling through bfv_noises"""
    Delta = Q // t
    noises = bfv_noises(Delta)
    m = [int(x) for x in rng.integers(0, t, n, dtype=np.uint64)]
    e = [noises[j % len(noises)] for j in range(n)]
    return [(Delta * m[j] + e[j]) % Q for j in range(n)], m, e


def assert_bfv_edge(Q, t, phases, e):
    """the edge noises put t v / Q within 2^-40 of a half"""
    Delta = Q // t
    edge = [v for v, x in zip(phases, e) if abs(x) >= Delta // 2 - 1]
    assert edge
    for v in edge:
        frac2 = (2 * t * v) % (2 * Q)  # 2 (t v mod Q)
        assert abs(frac2 - Q) << 40 < Q, "an edge noise is not at the rounding edge"


# ---- CKKS decode: words whose factor overflows ----
def inf_words(L, log2_scale):
    """words w of an L-word coefficient whose factor 2^(64 w) / scale is +inf (scale a power of two)"""
    return [w for w in range(L) if 64 * w - log2_scale >= 1024]


def negative_with_zero_inf_word(vals, Q, L, log2_scale):
    """some composed coefficient is in the upper half and equals Q in a word whose factor is +inf: the upper-half branch meets
    diff = 0 there, and 0 * inf would be NaN"""
    thr, mask = (Q + 1) // 2, (1 << 64) - 1
    words = inf_words(L, log2_scale)
    return any(v >= thr and any((v >> (64 * w)) & mask == (Q >> (64 * w)) & mask for w in words) for v in vals)


def composed(oc, L, plain, moduli):
    """the plaintext [L][n] (NTT form) as n composed coefficients in [0, Q)"""
    return crt_values(oc.ntt_inverse(L, plain[None])[0], moduli)


def decode_plaintexts(oc, moduli, n, L, rng):
    """[name] -> NTT-form plaintext [L][n] built from Python integers: centred coefficients in +-2^100; uniform residues; the same
    small coefficients with one and with two (opposite) coefficients next to +-Q/2, whose slots are +-inf or NaN once the factor of
    their top words overflows"""
    Q = product(moduli[:L])
    small = [(int(x) << 50) + int(y) for x, y in zip(rng.integers(-(1 << 50), 1 << 50, n), rng.integers(0, 1 << 50, n))]
    assert all(abs(x) < 1 << 100 for x in small) and min(small) < 0 < max(small)
    one = list(small)
    one[int(rng.integers(0, n))] = Q // 2 - int(rng.integers(0, 1 << 60))
    two = list(one)
    two[int(rng.integers(0, n))] = -(Q // 2) + int(rng.integers(0, 1 << 60))
    out = {}
    for name, coefs in (("centred 2^100", small), ("one near Q/2", one), ("two near +-Q/2", two)):
        out[name] = oc.ntt_forward(L, residue_rows(coefs, moduli, L)[None])[0]
    out["uniform"] = np.stack([rng.integers(0, int(moduli[j]), n, dtype=np.uint64) for j in range(L)])
    return out


def decode_scales(total_bits):
    """log2 of the legal scales tried: 2^-1000, 2^40 and, where (int) log2(scale) < total_bits allows it, 2^1020"""
    return [-1000, 40] + ([1020] if 1020 < total_bits else [])


def max_exponent(vals, Q):
    """the largest ex of |round(c)| = mant 2^ex over centred coefficients (mant < 2^53, the reduce kernel's decomposition)"""
    top = max(abs(v - Q if v > Q // 2 else v) for v in vals)
    return max(0, top.bit_length() - 53)


def random_values(rng, count, mag=1.0):
    return (rng.uniform(-mag, mag, count) + 1j * rng.uniform(-mag, mag, count)).astype(np.complex128)


def level_bits(moduli, L):
    return product(moduli[:L]).bit_length()
