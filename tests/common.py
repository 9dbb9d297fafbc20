"""Shared helpers for the test-suite: golden fixtures, deterministic synthetic ciphertexts."""
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")


def golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


def rand_ct(rng, moduli, n, size, L, batch=None):
    """uniform residues in [0, q_i), laid out [size][L][n] (or [batch][size][L][n]) like seal::Ciphertext::data()"""
    def one():
        return np.stack(
            [np.stack([rng.integers(0, moduli[i], n, dtype=np.uint64) for i in range(L)]) for _ in range(size)])
    if batch is None:
        return one()
    return np.stack([one() for _ in range(batch)])


def assert_words(got, want, what):
    """word-for-word equality; on failure name the first mismatching index"""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.argwhere(got != want)
    assert len(bad) == 0, f"{what}: {len(bad)} words differ, first at index {tuple(int(v) for v in bad[0])}: " \
                          f"got {int(got[tuple(bad[0])])}, want {int(want[tuple(bad[0])])}"


# ---- structured inputs at the arithmetic bounds (tests/test_gpu_bounds.py) ----
# Each generator returns words laid out like rand_ct, [size][L][n] or [batch][size][L][n]; the prime of row i is moduli[i].

def fill_ct(moduli, n, size, L, word, batch=None):
    """every word of row i = word(q_i) (a Python int below 2^64), e.g. `lambda q: q - 1` or `lambda q: 0`"""
    rows = np.stack([np.full(n, word(int(moduli[i])), dtype=np.uint64) for i in range(L)])
    shape = (size, L, n) if batch is None else (batch, size, L, n)
    return np.broadcast_to(rows, shape).copy()  # a writable array of its own


def max_ct(moduli, n, size, L, batch=None):
    """all words q - 1: the largest canonical residue"""
    return fill_ct(moduli, n, size, L, lambda q: q - 1, batch)


def zero_ct(moduli, n, size, L, batch=None):
    return fill_ct(moduli, n, size, L, lambda q: 0, batch)


def alternating_ct(moduli, n, size, L, batch=None):
    """words 0, q - 1, 0, q - 1, ... along every row"""
    out = max_ct(moduli, n, size, L, batch)
    out[..., 0::2] = 0
    return out


def largest_representative(x, q):
    """the largest 64-bit word congruent to x mod q: x + q * floor((2^64 - 1 - x) / q)"""
    x = np.asarray(x, dtype=np.uint64)
    return x + np.uint64(q) * ((np.uint64(2 ** 64 - 1) - x) // np.uint64(q))


def unreduce(a, moduli, axis_prime=-2):
    """every word replaced by its largest 64-bit representative (the prime of a row is moduli[index along axis_prime])"""
    out = np.array(a, dtype=np.uint64, copy=True)
    view = np.moveaxis(out, axis_prime, 0)
    for i in range(view.shape[0]):
        view[i] = largest_representative(view[i], int(moduli[i]))
    return out


def const_ntt_row(c, n):
    """the NTT form of the constant polynomial c * delta_0: the word c at every point (c below the row's prime).  Its transform
    modulo any auxiliary prime p_t is c mod p_t at every point, so c = p_t - 1 maximises the integer key-switching path's
    transformed digits and key words for prime t."""
    return np.full(n, c, dtype=np.uint64)


def all_coeffs_ntt(ntt_rows, moduli, n, L):
    """NTT form of the polynomial whose every coefficient is q_i - 1 (row i), [L][n]; ntt_rows maps a coefficient-form [L][n]
    array to NTT form (the oracle's ntt_row per row at small n, the library's transform_to_ntt at large n).  For two such
    polynomials alpha and beta the negacyclic product is alpha beta (2x + 2 - n): the digit sums of key switching reach
    +L n (q_J - 1)(q_I - 1) at x = n - 1 and nearly as much, negative, at x = 0."""
    return ntt_rows(max_ct(moduli, n, 1, L)[0])


def negacyclic_ones_square(n):
    """coefficient x of (1 + x + ... + x^(n-1))^2 mod x^n + 1, as Python ints: 2x + 2 - n"""
    return [2 * x + 2 - n for x in range(n)]


def product(values):
    out = 1
    for v in values:
        out *= int(v)
    return out


def centred_extreme_ct(moduli, n, size, L, sign, batch=None):
    """every coefficient the centred extreme of the level's modulus Q = q_0 ... q_{L-1}: floor(Q / 2) mod q_i (sign +1, the
    largest positive centred value) or ceil(Q / 2) mod q_i (sign -1, the most negative one, -floor(Q / 2)).  Two such
    constant-coefficient polynomials c (1 + x + ... + x^(n-1)) multiply to c^2 (2x + 2 - n): coefficient n - 1 of the tensor
    reaches n floor(Q / 2)^2."""
    Q = product(moduli[:L])
    c = Q // 2 if sign > 0 else (Q + 1) // 2
    rows = np.stack([np.full(n, c % int(moduli[i]), dtype=np.uint64) for i in range(L)])
    shape = (size, L, n) if batch is None else (batch, size, L, n)
    return np.broadcast_to(rows, shape).copy()


def alternating_extreme_ct(moduli, n, size, L, batch=None):
    """coefficients floor(Q / 2), ceil(Q / 2), floor(Q / 2), ... (the two centred extremes alternating along every row)"""
    out = centred_extreme_ct(moduli, n, size, L, +1, batch)
    out[..., 1::2] = centred_extreme_ct(moduli, n, size, L, -1, batch)[..., 1::2]
    return out


# ---- big integers behind RNS rows and decoded slots (tests/test_gpu_depth.py, tests/test_depth_oracle.py) ----

def residue_rows(values, moduli, L):
    """[L][n] residues of the signed Python ints `values` modulo the first L primes"""
    v = np.array([int(x) for x in values], dtype=object)
    return np.stack([(v % int(moduli[i])).astype(np.uint64) for i in range(L)])


def crt_values(rows, moduli):
    """the CRT composition in [0, Q) of every column of the coefficient-form rows [L][n], as Python ints"""
    L = rows.shape[0]
    Q = product(moduli[:L])
    acc = np.zeros(rows.shape[1], dtype=object)
    for i in range(L):
        q = int(moduli[i])
        m = Q // q
        acc = acc + rows[i].astype(object) * (m * pow(m % q, -1, q))
    return [int(x) % Q for x in acc]


def centred(values, Q):
    """representatives in (-Q/2, Q/2]"""
    return [v - Q if v > Q // 2 else v for v in values]


def ternary_secret_key(rng, moduli, n, ntt_rows):
    """a secret key with coefficients in {-1, 0, 1}, in NTT form at the key level ([k][n]); ntt_rows maps [k][n] coefficient rows to
    NTT form"""
    s = rng.integers(-1, 2, n)
    return ntt_rows(np.stack([np.where(s < 0, int(q) - 1, s).astype(np.uint64) for q in moduli]))


def assert_slots(got, want, what):
    """decoded complex slots: every double the reference (want) does not make NaN is bit-identical, and exactly its NaNs are NaN
    (IEEE 754 fixes when an operation gives NaN but not the NaN's sign or payload)"""
    g = np.ascontiguousarray(got, dtype=np.complex128).view(np.float64)
    w = np.ascontiguousarray(want, dtype=np.complex128).view(np.float64)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    nan = np.isnan(w)
    bad = np.argwhere(np.isnan(g) != nan)
    assert len(bad) == 0, f"{what}: {len(bad)} doubles differ in NaN-ness, first at index {tuple(int(v) for v in bad[0])}: " \
                          f"got {g[tuple(bad[0])]}, want {w[tuple(bad[0])]}"
    gw, ww = g.view(np.uint64).copy(), w.view(np.uint64).copy()
    gw[nan] = ww[nan] = 0
    assert_words(gw, ww, what)


# ---- primes (numth.cpp:278-311) ----

def is_prime(m):
    """deterministic Miller-Rabin below 2^64"""
    if m < 2:
        return False
    for p in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):
        if m % p == 0:
            return m == p
    d, s = m - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    for a in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):
        x = pow(a, d, m)
        if x in (1, m - 1):
            continue
        for _ in range(s - 1):
            x = x * x % m
            if x == m - 1:
                break
        else:
            return False
    return True


def ntt_primes_below(bits, n, count):
    """the `count` largest primes = 1 mod 2n below 2^bits, largest first: get_primes(2n, bits, count), the BEHZ auxiliary list
    for bits = 61 (CoeffModulus::Create takes the same primes for equal bit sizes, smallest first)"""
    out, c = [], ((1 << bits) - 1) // (2 * n) * (2 * n) + 1
    while len(out) < count:
        assert c > 1 << (bits - 1), "not enough primes"
        if is_prime(c):
            out.append(c)
        c -= 2 * n
    return out
