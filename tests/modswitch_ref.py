"""What rescale and modulus switching compute, stated on big integers rather than step by step.

For one coefficient take X, the CRT composition in [0, Q) of its residues at the level with primes q_0 .. q_{L-1}, let q_l = q_{L-1}
be the top prime and h = floor(q_l / 2):

- CKKS rescale_to_next and BFV mod_switch_to_next: y = floor((X + h) / q_l);
- BGV mod_switch_to_next: with r = X mod q_l, k = (-r q_l^-1) mod t and delta = r + k q_l, y = (X - delta) / q_l (an exact division;
  y is negative when X < delta);

and the result is y mod q_i for every i < L - 1.  CKKS and BGV ciphertexts are in NTT form: their rows go to coefficient form and the
result back through the oracle's per-row transforms (tests/oracle.py).  Every coefficient of every polynomial is one numpy object
array, so a whole batch costs a few passes of Python integer arithmetic.  TEST INFRASTRUCTURE ONLY."""
import numpy as np

from common import product

CKKS_RESCALE, BFV_SWITCH, BGV_SWITCH = "ckks_rescale", "bfv_mod_switch", "bgv_mod_switch"


def compose(rows, moduli):
    """X in [0, Q) of every column of the coefficient-form residues rows [L][m], Q = q_0 ... q_{L-1}: an object array of m ints"""
    L = rows.shape[0]
    Q = product(moduli[:L])
    acc = np.zeros(rows.shape[1], dtype=object)
    for i in range(L):
        q = int(moduli[i])
        m = Q // q
        acc = acc + rows[i].astype(object) * (m * pow(m % q, -1, q))
    return acc % Q


def divide(kind, X, q_top, t=0):
    """y of every X (object array) for CKKS rescale / BFV mod-switch (divide and round) or BGV mod-switch (exact division)"""
    if kind == BGV_SWITCH:
        r = X % q_top
        k = (-r * pow(q_top % t, -1, t)) % t
        return (X - (r + k * q_top)) // q_top
    return (X + q_top // 2) // q_top


def residues(values, moduli, count):
    """[count][m] residues (uint64) of the object array of ints `values` modulo the first `count` primes"""
    return np.stack([(values % int(moduli[i])).astype(np.uint64) for i in range(count)])


def switch_coeff(kind, polys, moduli, t=0):
    """coefficient-form polynomials [P][L][n] at L primes -> [P][L-1][n]: the division above, coefficient by coefficient"""
    P, L, n = polys.shape
    rows = np.ascontiguousarray(polys.transpose(1, 0, 2)).reshape(L, P * n)
    y = divide(kind, compose(rows, moduli), int(moduli[L - 1]), t)
    return np.ascontiguousarray(residues(y, moduli, L - 1).reshape(L - 1, P, n).transpose(1, 0, 2))


def expected(kind, oc, polys, pool=None):
    """the result of `kind` on polynomials [..][L][n] in the form the scheme keeps them (NTT form for CKKS / BGV, coefficient form
    for BFV), computed with big integers; oc: the oracle of the context (its transforms and primes); pool: an executor of processes
    that share the polynomials out (the arithmetic holds the interpreter lock)"""
    polys = np.ascontiguousarray(polys, dtype=np.uint64)
    lead, (L, n) = polys.shape[:-2], polys.shape[-2:]
    flat = polys.reshape(-1, L, n)
    ntt = kind != BFV_SWITCH
    coeff = oc.ntt_inverse(L, flat) if ntt else flat
    if pool is None or len(coeff) * n < 1 << 16:
        out = switch_coeff(kind, coeff, oc.moduli, oc.t)
    else:
        parts = np.array_split(coeff, min(len(coeff), 64))
        out = np.concatenate(list(pool.map(switch_coeff, [kind] * len(parts), parts, [oc.moduli] * len(parts), [oc.t] * len(parts))))
    if ntt:
        out = oc.ntt_forward(L - 1, out)
    return out.reshape(*lead, L - 1, n)


PATTERNS = ("uniform", "max", "turns", "extremes", "bgv_edges")


def patterns(kind):
    """the word patterns of `words` that mean something for `kind` (bgv_edges: BGV only)"""
    return PATTERNS if kind == BGV_SWITCH else PATTERNS[:-1]


def words(kind, pattern, rng, oc, L, polys):
    """`polys` polynomials [polys][L][n] at L primes in the form the scheme keeps them, every word drawn by `pattern`:
    uniform: uniform words; max: every word q_i - 1; turns: coefficients at the rounding turns (rounding_turns); extremes:
    coefficients 0, Q - 1 and floor(Q / 2); bgv_edges: coefficients whose top residue is one of bgv_edges (t of the oracle)"""
    moduli, n, q_top = oc.moduli, oc.n, int(oc.moduli[L - 1])
    if pattern == "uniform":
        return np.stack([np.stack([rng.integers(0, int(moduli[i]), n, dtype=np.uint64) for i in range(L)]) for _ in range(polys)])
    if pattern == "max":
        return np.stack([np.stack([np.full(n, int(moduli[i]) - 1, dtype=np.uint64) for i in range(L)]) for _ in range(polys)])
    if pattern == "extremes":
        Q = product(moduli[:L])
        coeff = np.stack([coeff_rows_of_values(np.roll([0, Q - 1, Q // 2], p), moduli, L, n) for p in range(polys)])
    else:
        tops = rounding_turns(q_top) if pattern == "turns" else bgv_edges(q_top, oc.t)
        coeff = np.stack([coeff_rows_with_top(rng, moduli, L, n, np.roll(tops, p)) for p in range(polys)])
    return oc.ntt_forward(L, coeff) if kind != BFV_SWITCH else coeff


def coeff_rows_with_top(rng, moduli, L, n, tops):
    """coefficient-form residues [L][n] of coefficients X with X mod q_top = tops[j] (cycled along the row) and uniform residues
    modulo the other primes: by the CRT every such X in [0, Q) is reached, the residue at the top prime fixed"""
    rows = np.stack([rng.integers(0, int(moduli[i]), n, dtype=np.uint64) for i in range(L - 1)] +
                    [np.resize(np.array([int(v) for v in tops], dtype=np.uint64), n)])
    return rows


def coeff_rows_of_values(values, moduli, L, n):
    """coefficient-form residues [L][n] of the ints `values` (cycled along the row), taken modulo Q of the level"""
    Q = product(moduli[:L])
    v = np.resize(np.array([int(x) % Q for x in values], dtype=object), n)
    return residues(v, moduli, L)


def rounding_turns(q_top):
    """top-prime residues of X where X + h = 0, 1 and q_top - 1 (mod q_top): the rounding of floor((X + h) / q_top) turns there"""
    h = q_top // 2
    return [(c - h) % q_top for c in (0, 1, q_top - 1)]


def bgv_edges(q_top, t):
    """top-prime residues r = X mod q_top where BGV's correction delta = r + k q_top is extreme, k = (-r q_top^-1) mod t: r = 0 and
    r = q_top - 1; below q_top, where k wraps between 0 and t - 1, the largest r with k = 0 (a multiple of t) and the largest with
    k = t - 1 (r = q_top - t); above it (no such r but 0), r = 1 and q_top - 2"""
    if t >= q_top:
        return [0, q_top - 1, 1, q_top - 2]
    out = [0, q_top - 1, (q_top - 1) // t * t, q_top - t]
    inv = pow(q_top % t, -1, t)
    assert (-out[2] * inv) % t == 0 and (-out[3] * inv) % t == t - 1, (q_top, t)
    return out
