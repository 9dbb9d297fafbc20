"""The arithmetic behind sb200_multiply_plain_sum, in Python integers: the 128-bit accumulation bound of its reduction window and
the folding of add_many's BGV balancing into one constant per term."""
import random

WINDOW = 256  # kPlainSumWindow (seal_b200/csrc/sb_engine.cuh)


def primes_below(bound, count):
    out, c = [], bound - 1
    while len(out) < count:
        if c % 2 and all(c % d for d in range(3, 2000, 2)) and pow(2, c - 1, c) == 1 and pow(3, c - 1, c) == 1:
            out.append(c)
        c -= 1
    return out


def test_window_bound_at_60_bit_primes():
    """a carried residue below q plus WINDOW products of words q - 1 stays below 2^128 for every prime below 2^60, and the
    window is the largest that does: WINDOW + 1 products at the largest 60-bit prime exceed 2^128"""
    for q in primes_below(2**60, 3) + [2**60 - 1]:  # 2^60 - 1 bounds every user prime (at most 60 bits)
        worst = (q - 1) + WINDOW * (q - 1) ** 2
        assert worst < 2**128, q
    q = primes_below(2**60, 1)[0]
    assert (WINDOW + 1) * (q - 1) ** 2 >= 2**128
    assert q - 1 + (WINDOW + 1) * (q - 1) ** 2 >= 2**128


def left_fold(terms, modes, factors, q):
    """sb200_add_many's left fold of already-reduced product words (add / sub, scaled by (e1, e2) on scaled steps)"""
    acc = terms[0]
    for j in range(1, len(terms)):
        m = modes[j - 1]
        y = terms[j]
        if m & 2:
            acc = acc * (factors[j - 1][0] % q) % q
            y = y * (factors[j - 1][1] % q) % q
        acc = (acc - y) % q if m & 1 else (acc + y) % q
    return acc


def folded_constants(K, modes, factors, q):
    """the per-term constants op_multiply_plain_sum forms on the host: +/- e2_t prod_{u > t} e1_u mod q"""
    out, tail = [0] * K, 1
    for t in range(K - 1, -1, -1):
        m = modes[t - 1] if t else 0
        v = (factors[t - 1][1] % q if m & 2 else 1) * tail % q
        out[t] = (q - v) % q if m & 1 else v
        if m & 2:
            tail = tail * (factors[t - 1][0] % q) % q
    return out


def test_folded_constants_match_left_fold():
    """for random factors (any 64-bit words, reduced mod q as the fold reduces them), modes and product words, the sum of the
    constants times the terms is the left fold's residue"""
    rng = random.Random(2024)
    for q in primes_below(2**60, 2) + primes_below(2**30, 1):
        for K in (1, 2, 3, 7, 40):
            for _ in range(20):
                terms = [rng.randrange(q) for _ in range(K)]
                modes = [rng.randrange(4) for _ in range(K - 1)]
                factors = [(rng.randrange(2**64), rng.randrange(2**64)) for _ in range(K - 1)]
                c = folded_constants(K, modes, factors, q)
                assert sum(ci * ti for ci, ti in zip(c, terms)) % q == left_fold(terms, modes, factors, q)
