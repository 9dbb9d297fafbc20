"""CPU: the Python restatement of Decryptor::invariant_noise_budget (tests/noise_ref.py) against the reference itself, on fresh
encryptions, uniform-random ciphertexts and chosen phases, BFV and BGV, sizes 2-4, one, two and several primes; and the
reference's errors for CKKS and for the wrong form.  The GPU tests hold the device to the same two numbers."""
import numpy as np
import pytest

import noise_ref as N
import refseal as R
from common import rand_ct

needs_ref = pytest.mark.skipif(not N.available(), reason="oracle/_ref/libsealref{,_noise}.so not present")


def _ctx(scheme, n, bits):
    mods = R.coeff_modulus_create(n, bits)
    t = R.plain_modulus_batching(n, 20)
    return R.RefContext(scheme, n, mods, t), mods, t


@needs_ref
@pytest.mark.parametrize("scheme", [R.BFV, R.BGV])
@pytest.mark.parametrize("bits", [[50], [40, 40], [36, 36, 37, 40, 50]])
def test_restatement_matches_reference(scheme, bits):
    n = 256
    rc, mods, t = _ctx(scheme, n, bits + [60])
    sk = rc.secret_key()
    ntt = scheme == R.BGV
    rng = np.random.default_rng(len(bits) * 10 + scheme)
    L = len(bits)
    cases = []
    # fresh symmetric encryptions of random plaintexts (encrypt_zero_symmetric + add_plain)
    for _ in range(2):
        z = rc.encrypt_zero_symmetric(L)
        cases.append(rc.plain_op_coeff(1, L, z, rng.integers(0, t, n, dtype=np.uint64), ntt))
    for size in (2, 3, 4):  # uniform-random ciphertexts
        cases.append(rand_ct(rng, mods, n, size, L, 1)[0])
    Q, tb = N.total_bits(mods, L)
    for v in N.edge_values(Q, tb):  # chosen phases
        vals = [int(x) for x in rng.integers(-4, 5, n)]
        vals[int(rng.integers(0, n))] = v
        cases.append(N.structured_ct(scheme, n, mods, t, L, 2 + len(cases) % 3, vals))
    for ct in cases:
        st, want = N.ref_budget(rc, L, ct, ntt)
        assert st == 0, want
        assert N.restated_budget(scheme, n, mods, t, sk, ct) == want


@needs_ref
def test_structured_phase_budgets_are_exact():
    """the composed noise of a chosen phase is v itself: the budget is total_bits - bits(|v|) - 1"""
    n = 256
    for scheme in (R.BFV, R.BGV):
        rc, mods, t = _ctx(scheme, n, [60, 60, 60])
        L = 2
        Q, tb = N.total_bits(mods, L)
        for v in (0, 1, -1, 1 << 64, -(1 << 100)):
            ct = N.structured_ct(scheme, n, mods, t, L, 2, [v] + [0] * (n - 1))
            mag = v if v >= 0 else -v
            assert N.ref_budget(rc, L, ct, scheme == R.BGV) == (0, max(0, tb - mag.bit_length() - 1))


@needs_ref
def test_reference_errors():
    n = 256
    rc, mods, t = _ctx(R.BFV, n, [40, 40])
    ct = np.zeros((2, 1, n), dtype=np.uint64)
    assert N.ref_budget(rc, 1, ct, True) == (-1, "BFV encrypted cannot be in NTT form")
    rc, mods, t = _ctx(R.BGV, n, [40, 40])
    assert N.ref_budget(rc, 1, ct, False) == (-1, "BGV encrypted must be in NTT form")
    mods = R.coeff_modulus_create(n, [40, 40])
    rc = R.RefContext(R.CKKS, n, mods)
    assert N.ref_budget(rc, 1, ct, True) == (-1, "unsupported scheme")
