"""The element-wise statement (tests/elementwise_ref.py) against the oracle and, where oracle/_ref/libsealref.so is built, the
reference itself, on small rings and on every word class the GPU matrix (tests/test_gpu_elementwise_matrix.py) feeds the kernels:
canonical words, 0 / 1 / q - 1, unreduced words up to 2^64 - 1, and the pairs that reach each branch of the reference's formulas
(x + y >= 2^64; x >= y with x - y > 2^64 - q; y - x > q; unreduced plaintext words against canonical c_0 and the reverse)."""
import numpy as np
import pytest

import elementwise_ref as E
import oracle as O
import refseal as R

needs_ref = pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsealref.so not built")

TOP = 2 ** 64


def pair_words(kind, rng, q, shape):
    """(x, y) uint64 arrays of `shape` for one prime q, by word class"""
    u = lambda lo, hi: rng.integers(lo, hi, shape, dtype=np.uint64, endpoint=False) if hi <= TOP - 1 else \
        rng.integers(lo, TOP - 1, shape, dtype=np.uint64, endpoint=True)
    if kind == "canonical":
        return u(0, q), u(0, q)
    if kind == "edges":
        e = np.array([0, 1, q - 1], dtype=np.uint64)
        return e[rng.integers(0, 3, shape)], e[rng.integers(0, 3, shape)]
    if kind == "unreduced":
        return u(0, TOP), u(0, TOP)
    r = rng.integers(0, 2 ** 63, shape, dtype=np.uint64)
    top = np.uint64(TOP - 1)
    with np.errstate(over="ignore"):
        if kind == "sum_wraps":  # x + y >= 2^64
            x = u(TOP // 2, TOP)
            return x, top - r % x
        if kind == "difference_wraps":  # x >= y, x - y > 2^64 - q
            y = u(0, q // 2)
            return top - r % (np.uint64(q - 1) - y), y
        if kind == "deep_borrow":  # y - x > q
            x = u(0, q)
            return x, x + np.uint64(q + 1) + r % (top - x - np.uint64(q))
    if kind == "unreduced_vs_canonical":
        return u(q, TOP), u(0, q)
    if kind == "canonical_vs_unreduced":
        return u(0, q), u(q, TOP)
    raise ValueError(kind)


KINDS = ("canonical", "edges", "unreduced", "sum_wraps", "difference_wraps", "deep_borrow", "unreduced_vs_canonical",
         "canonical_vs_unreduced")


def draw(kind, rng, mods, size, L, n):
    x = np.empty((size, L, n), dtype=np.uint64)
    y = np.empty_like(x)
    for i in range(L):
        x[:, i], y[:, i] = pair_words(kind, rng, mods[i], (size, n))
    return x, y


def test_branches_by_hand():
    """the worked cases of the borrow form with a 50-bit q, and the add and negate forms on the same words"""
    q = np.uint64((1 << 50) - 27)
    m = np.uint64(TOP - 1)
    assert int(E.sub(m, np.uint64(0), q)) == TOP - 1  # no borrow: the difference, unreduced
    assert int(E.sub(np.uint64(0), m, q)) == int(q) + 1  # borrow: 1 + q
    assert int(E.add(m, m, q)) == TOP - 2 - int(q)  # the sum wraps, then sheds q once
    assert int(E.negate(m, q)) == (int(q) - (TOP - 1)) % TOP
    assert int(E.negate(np.uint64(0), q)) == 0


def test_products_exact():
    rng = np.random.default_rng(7)
    for q in (5, 65537, (1 << 57) - 111, (1 << 61) - 1):
        x = rng.integers(0, TOP - 1, 2000, dtype=np.uint64, endpoint=True)
        y = rng.integers(0, TOP - 1, 2000, dtype=np.uint64, endpoint=True)
        x[:3], y[:3] = [0, q - 1, TOP - 1], [q - 1, q - 1, TOP - 1]
        got = E.mulmod(x, y, np.uint64(q))
        assert [int(v) for v in got] == [int(a) * int(b) % q for a, b in zip(x, y)]


@pytest.mark.parametrize("kind", KINDS)
def test_statement_vs_oracle(kind):
    n = 64
    mods = O.coeff_modulus_create(n, [20, 50, 57, 60])
    oc = O.Oracle(O.CKKS, n, mods)
    rng = np.random.default_rng(KINDS.index(kind))
    for L in (1, 4):
        for size in (2, 3):
            x, y = draw(kind, rng, mods, size, L, n)
            for mode in (0, 1, 2):
                assert (E.linear(mode, x, y, mods) == oc.linear(mode, L, x, y)).all(), (kind, L, size, mode)
            assert (E.tensor(x, y, mods) == oc.multiply(L, x, y)).all(), (kind, L, size)
            assert (E.multiply_plain(x, y[0], mods) == oc.multiply_plain(L, x, y[0])).all(), (kind, L, size)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("scheme", ["bfv", "bgv"])
def test_coeff_plain_statement_vs_oracle(kind, scheme):
    """add_plain / sub_plain with coefficient-form plaintexts (words below t) on c_0 words of each class"""
    n = 64
    mods = O.coeff_modulus_create(n, [30, 50, 57])
    t = 65537 if scheme == "bgv" else 257
    oc = O.Oracle(O.BFV if scheme == "bfv" else O.BGV, n, mods, t)
    rng = np.random.default_rng(31 + KINDS.index(kind))
    for L in (1, 3):
        a, _ = draw(kind, rng, mods, 2, L, n)
        plain = rng.integers(0, t, n, dtype=np.uint64)
        plain[:3] = [0, t - 1, (t + 1) // 2]
        cf = 1 if scheme == "bfv" else 7
        T = E.bfv_scaled_plain(plain, mods, L, t) if scheme == "bfv" else oc.plain_to_ntt(L, (plain.astype(object) * cf % t).astype(np.uint64))
        for sub in (False, True):
            assert (E.add_plain_c0(a, T, mods, sub) == oc.add_plain_coeff(L, a, plain, sub, cf)).all(), (kind, L, sub)


@needs_ref
@pytest.mark.parametrize("kind", KINDS)
def test_statement_vs_reference(kind):
    n = 64
    mods = R.coeff_modulus_create(n, [20, 50, 57, 60])
    rc = R.RefContext(R.BGV, n, mods, 257)  # the NTT-form tensor of CKKS and BGV, without CKKS's bound on the product's scale
    rng = np.random.default_rng(100 + KINDS.index(kind))
    for L in (1, 3):
        for size in (2, 3):
            x, y = draw(kind, rng, mods, size, L, n)
            for mode in (0, 1, 2):
                assert (E.linear(mode, x, y, mods) == rc.linear(mode, L, x, y)).all(), (kind, L, size, mode)
            assert (E.tensor(x, y, mods) == rc.multiply(L, x, y)).all(), (kind, L, size)
            if size == 2:
                assert (E.tensor(x, x, mods) == rc.square(L, x)).all(), (kind, L)
            assert (E.multiply_plain(x, y[0], mods) == rc.multiply_plain(L, x, y[0])).all(), (kind, L, size)


@needs_ref
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("scheme", ["bfv", "bgv"])
def test_coeff_plain_statement_vs_reference(kind, scheme):
    n = 64
    mods = R.coeff_modulus_create(n, [30, 50, 57])
    t = 65537 if scheme == "bgv" else 257
    rc = R.RefContext(R.BFV if scheme == "bfv" else R.BGV, n, mods, t)
    oc = O.Oracle(O.BFV if scheme == "bfv" else O.BGV, n, mods, t)
    rng = np.random.default_rng(200 + KINDS.index(kind))
    for L in (1, 2):
        a, _ = draw(kind, rng, mods, 2, L, n)
        plain = rng.integers(0, t, n, dtype=np.uint64)
        cf = 1 if scheme == "bfv" else 7
        T = E.bfv_scaled_plain(plain, mods, L, t) if scheme == "bfv" else oc.plain_to_ntt(L, (plain.astype(object) * cf % t).astype(np.uint64))
        for mode, sub in ((1, False), (2, True)):
            assert (E.add_plain_c0(a, T, mods, sub) == rc.plain_op_coeff(mode, L, a, plain, scheme == "bgv", cf)).all(), (kind, L, sub)
