"""The arithmetic behind sb200_multiply_sum, in Python integers: the 128-bit accumulation bound of its reduction window (two
products per term in c1 = a0 b1 + a1 b0), the folding of add_many's modes and BGV balancing into one constant per term, and the
restated tensor sum against the chain multiply-then-add_many."""
import random

from test_plain_sum_bounds import folded_constants, left_fold, primes_below

CAP = 128  # kMultiplySumWindow (seal_b200/csrc/sb_engine.cuh)


def window(q):
    """sum_window(c, L, 2, kMultiplySumWindow) of seal_b200/csrc/sb_plainsum.cu for a level whose largest prime is q"""
    return min(CAP, (2**128 - 1 - (q - 1)) // (2 * (q - 1) ** 2))


def worst(q, w):
    """the largest c1 accumulator after w terms: a carried residue plus two products of words q - 1 per term"""
    return (q - 1) + 2 * w * (q - 1) ** 2


def test_window_values():
    """the pinned windows: the cap (128) for every prime below 2^60, 32 for the largest 61-bit primes"""
    for bits in (50, 55, 59, 60):
        for q in primes_below(2**bits, 2):
            assert window(q) == 128, (bits, q)
    assert window(2**60 - 1) == 128  # bounds every prime of at most 60 bits
    for q in primes_below(2**61, 3):
        assert window(q) == 32, q


def test_window_fits_and_one_more_overflows():
    """w terms of worst-case words fit in 128 bits at 50/55/59/60/61-bit primes; w + 1 terms overflow at the largest 60- and
    61-bit primes, where the window is the bound (below 60 bits it is the cap, and w + 1 would still fit)"""
    for bits in (50, 55, 59, 60, 61):
        for q in primes_below(2**bits, 2):
            w = window(q)
            assert worst(q, w) < 2**128, (bits, q)
    for bits in (60, 61):
        q = primes_below(2**bits, 1)[0]
        w = window(q)
        assert worst(q, w + 1) >= 2**128, (bits, q, w)
    for bits in (50, 55, 59):
        q = primes_below(2**bits, 1)[0]
        assert worst(q, CAP + 1) < 2**128  # the cap, not the bound, sets these windows


def kernel_sum(q, a, b, consts):
    """multiply_sum_kernel for one coefficient, restated: left words reduced and scaled by the term's constant, 128-bit
    accumulators reduced every window(q) terms (asserting none ever reaches 2^128)"""
    w = window(q)
    acc = [0, 0, 0]
    for t, ((a0, a1), (b0, b1)) in enumerate(zip(a, b)):
        x0, x1 = a0 % q * consts[t] % q, a1 % q * consts[t] % q
        y0, y1 = b0 % q, b1 % q
        acc[0] += x0 * y0
        acc[1] += x0 * y1 + x1 * y0
        acc[2] += x1 * y1
        assert max(acc) < 2**128
        if (t + 1) % w == 0:
            acc = [v % q for v in acc]
    return [v % q for v in acc]


def chain(q, a, b, modes, factors):
    """multiply of every term (canonical tensor words), then add_many's left fold of each polynomial"""
    prods = [((a0 % q) * (b0 % q) % q, ((a0 % q) * (b1 % q) + (a1 % q) * (b0 % q)) % q, (a1 % q) * (b1 % q) % q) for (a0, a1), (b0, b1) in zip(a, b)]
    return [left_fold([p[s] for p in prods], modes, factors, q) for s in range(3)]


def test_folded_constants_match_left_fold_with_sub_and_scaled_steps():
    """the per-term constants equal add_many's left fold for every mode, SUB and SCALED steps included"""
    rng = random.Random(77)
    for q in primes_below(2**61, 1) + primes_below(2**50, 1):
        for K in (1, 2, 5, 33):
            modes = [rng.randrange(4) for _ in range(K - 1)]
            modes[: min(4, K - 1)] = [0, 1, 2, 3][: min(4, K - 1)]
            factors = [(rng.randrange(2**64), rng.randrange(2**64)) for _ in range(K - 1)]
            terms = [rng.randrange(q) for _ in range(K)]
            c = folded_constants(K, modes, factors, q)
            assert sum(ci * ti for ci, ti in zip(c, terms)) % q == left_fold(terms, modes, factors, q)


def test_restated_tensor_sum_equals_chain():
    """the kernel's windowed tensor sum equals multiply-then-add_many for unreduced and all-(q - 1) words, across window
    reductions, at 60- and 61-bit primes"""
    rng = random.Random(78)
    for q in primes_below(2**60, 1) + primes_below(2**61, 1):
        w = window(q)
        for K in (1, 3, w, w + 1, 2 * w + 5):
            for words in ("random", "q-1", "2^64-1"):
                def word():
                    return {"random": rng.randrange(2**64), "q-1": q - 1, "2^64-1": 2**64 - 1}[words]

                a = [(word(), word()) for _ in range(K)]
                b = [(word(), word()) for _ in range(K)]
                modes = [rng.randrange(4) for _ in range(K - 1)]
                factors = [(rng.randrange(2**64), rng.randrange(2**64)) for _ in range(K - 1)]
                consts = folded_constants(K, modes, factors, q)
                assert kernel_sum(q, a, b, consts) == chain(q, a, b, modes, factors), (q, K, words)
