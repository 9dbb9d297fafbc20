"""The big-integer statement of rescale and modulus switching (tests/modswitch_ref.py) against the oracle (tests/oracle.py) and the
reference, word for word.  Both follow SEAL's algorithm step by step; the statement only says what the division computes, so the GPU
matrix (tests/test_gpu_modswitch_matrix.py) can check every output word against it.  Where the statement and SEAL disagree, the
statement is wrong.

Prime sets: the top prime far above every data prime, below every one, and mixed; all primes below 2^57 (with the largest 57-bit
prime) or one of 60 bits.  BGV with t = 65537, with t between the primes and with a 60-bit t above all of them."""
import numpy as np
import pytest

import modswitch_ref as M
import oracle as O
import refseal as R
from common import assert_words, is_prime, product

needs_ref = pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsealref.so not present")

PRIME_SETS = {"above-q57": [30, 34, 38, 57], "below-q60": [60, 50, 40, 30], "mixed-q60": [40, 60, 30, 50], "mixed-q57": [40, 57, 30, 50]}
KINDS = {"CKKS": M.CKKS_RESCALE, "BFV": M.BFV_SWITCH, "BGV": M.BGV_SWITCH}


def prime_below(bound):
    c = bound - 1
    while not is_prime(c):
        c -= 1
    return c


T_MID, T_60 = prime_below(2 ** 36), prime_below(2 ** 60)
CASES = [("CKKS", 0), ("BFV", 65537), ("BGV", 65537), ("BGV", T_MID), ("BGV", T_60)]


def oracle_switch(oc, kind, L, polys):
    """the oracle's rescale / mod-switch of [P][L][n] (P even), two polynomials at a time"""
    fn = {M.CKKS_RESCALE: oc.rescale, M.BFV_SWITCH: oc.bfv_mod_switch, M.BGV_SWITCH: oc.bgv_mod_switch}[kind]
    return np.concatenate([fn(L, np.ascontiguousarray(polys[p:p + 2])) for p in range(0, len(polys), 2)])


def case_id(c):
    return f"{c[0]}-t{c[1]}" if c[1] else c[0]


@pytest.mark.parametrize("n", [256, 4096])
@pytest.mark.parametrize("prime_set", list(PRIME_SETS))
@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_statement_vs_oracle(case, prime_set, n):
    scheme, t = case
    kind = KINDS[scheme]
    mods = O.coeff_modulus_create(n, PRIME_SETS[prime_set])
    oc = O.Oracle(getattr(O, scheme), n, mods, t)
    rng = np.random.default_rng(n + len(prime_set) + t % 1000)
    for L in (4, 3, 2):
        for pattern in M.patterns(kind):
            polys = M.words(kind, pattern, rng, oc, L, 2)
            assert_words(M.expected(kind, oc, polys), oracle_switch(oc, kind, L, polys), f"{scheme} t = {t}, L = {L}, {pattern} words")


def test_statement_edges_hit():
    """the patterned words reach what they are named for: X + h at 0, 1 and q_l - 1 (mod q_l); X at 0, Q - 1, floor(Q / 2);
    BGV's k at 0 and t - 1"""
    n, mods = 256, O.coeff_modulus_create(256, PRIME_SETS["above-q57"])
    oc = O.Oracle(O.BGV, n, mods, 65537)
    rng = np.random.default_rng(1)
    L, ql = 3, mods[2]
    Q = mods[0] * mods[1] * mods[2]
    X = M.compose(oc.ntt_inverse(L, M.words(M.CKKS_RESCALE, "turns", rng, oc, L, 1))[0], mods)
    assert {int(x + ql // 2) % ql for x in X} == {0, 1, ql - 1}
    X = M.compose(oc.ntt_inverse(L, M.words(M.CKKS_RESCALE, "extremes", rng, oc, L, 1))[0], mods)
    assert {int(x) for x in X} == {0, Q - 1, Q // 2}
    X = M.compose(M.words(M.BFV_SWITCH, "bgv_edges", rng, oc, L, 1)[0], mods)
    ks = {(-(int(x) % ql) * pow(ql, -1, 65537)) % 65537 for x in X}
    assert {0, 65536} <= ks


@needs_ref
@pytest.mark.parametrize("n", [256, 4096])
@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_statement_vs_reference(case, n):
    """seal::Evaluator::rescale_to_next / mod_switch_to_next at every level below the key level (the reference's ciphertexts live
    there).  The reference's modulus chain ends above the first level whose modulus is not above t: switching into such a level
    is only compared with the oracle (test_statement_vs_oracle), and here the reference must refuse it."""
    scheme, t = case
    kind = KINDS[scheme]
    compared, refused = 0, 0
    for name, bits in PRIME_SETS.items():
        mods = R.coeff_modulus_create(n, bits)
        oc = O.Oracle(getattr(O, scheme), n, mods, t)
        rc = R.RefContext(getattr(R, scheme), n, mods, t)
        rng = np.random.default_rng(n + t % 1000)
        for L in (3, 2):
            for pattern in M.patterns(kind):
                # c1 uniform: SEAL refuses a result whose c1 is zero ("transparent"), as the max pattern's is
                polys = np.stack([M.words(kind, pattern, rng, oc, L, 1)[0], M.words(kind, "uniform", rng, oc, L, 1)[0]])
                if t and product(mods[:L - 1]) <= t:
                    with pytest.raises(RuntimeError, match="end of modulus switching chain"):
                        rc.mod_switch(L, polys)
                    refused += 1
                    continue
                got = rc.rescale(L, polys) if scheme == "CKKS" else rc.mod_switch(L, polys)
                assert_words(M.expected(kind, oc, polys), got, f"{name}: {scheme} t = {t}, L = {L}, {pattern} words")
                compared += 1
        rc.close()
    assert compared + refused == len(PRIME_SETS) * 2 * len(M.patterns(kind)) and compared >= refused
