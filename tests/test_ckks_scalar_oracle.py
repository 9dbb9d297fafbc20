"""The Python-integer restatement of CKKSEncoder::encode(double) / encode(int64) (tests/ckks_scalar_ref.py) against the reference
itself (oracle/_ref/libsealref_scalar.so): words, plaintext scale and error messages.  CPU only; the device encoder is checked
against both in tests/test_gpu_ckks_scalar.py."""
import math

import numpy as np
import pytest

import ckks_scalar_ref as S
import refseal as R

pytestmark = pytest.mark.skipif(not (S.available() and R.available()), reason="oracle/_ref/libsealref_scalar.so not built")

N = 4096
# (name, prime bits): a two-word level (one-word and two-word branches) and a 240-bit one (the multi-precision branch)
LEVELS = {"60x2": [60, 60], "60x4": [60, 60, 60, 60], "30x2": [30, 30]}


def ref_and_moduli(bits):
    mods = R.coeff_modulus_create(N, bits)
    return S.RefScalar(N, mods), mods


def check(ref, mods, L, kind, value, scale):
    want, werr = S.restate(mods[:L], N, kind, value, scale)
    got, gs = ref.encode(L, kind, value, scale)
    if want is None:
        assert got is None and gs == werr, (value, scale, gs, werr)
        return None
    assert got is not None, (value, scale, gs)
    assert (got == want).all(), (value, scale)
    assert gs == (1.0 if kind == S.INT64 else scale)
    return got


@pytest.mark.parametrize("level", sorted(LEVELS))
def test_real_restatement_matches_reference(level):
    ref, mods = ref_and_moduli(LEVELS[level])
    for L in (len(mods), 1):
        tb = S.total_bits(mods[:L])
        for value, scale in S.real_cases(tb):
            check(ref, mods, L, S.REAL, value, scale)


def test_real_rounding_and_bounds_are_exercised():
    """the pinned cases really hit what they are meant to: half away from zero, -0.0, both sides of the bit bound, both scale tests"""
    ref, mods = ref_and_moduli([60, 60])
    q0 = mods[0]
    word = lambda v, s=1.0: int(check(ref, mods, 2, S.REAL, v, s)[0, 0])
    assert word(0.49) == 0 and word(-0.49) == 0 and word(-0.0) == 0
    assert word(0.5) == 1 and word(-0.5) == q0 - 1 and word(2.5) == 3 and word(-2.5) == q0 - 3
    tb = S.total_bits(mods)
    big = 2.0 ** (tb - 2)
    assert check(ref, mods, 2, S.REAL, 1.5 * big / 2, 1.0) is not None  # bit count tb - 1
    assert ref.encode(2, S.REAL, big, 1.0) == (None, "encoded value is too large")  # bit count tb
    assert ref.encode(2, S.REAL, math.nextafter(big, 0.0), 1.0) == (None, "encoded value is too large")  # log2 rounds up
    # accepted by encode(double), refused by the vector encode: a subnormal scale, and (int)log2(scale) = total bits - 1
    assert check(ref, mods, 2, S.REAL, 1.0, 5e-324) is not None
    assert word(2.0 ** -tb, 2.0 ** (tb - 1)) == 1
    rc = R.RefContext(R.CKKS, N, mods)
    assert rc.ckks_encode(2, [1.0], 5e-324) is None
    assert rc.ckks_encode(2, [0.0], 2.0 ** (tb - 1)) is None
    for scale in (0.0, -1.0, math.inf, math.nan, 2.0 ** tb):
        assert ref.encode(2, S.REAL, 1.0, scale) == (None, "scale out of bounds")
    for value in (math.inf, -math.inf, math.nan):
        assert ref.encode(2, S.REAL, value, 1.0) == (None, "value must be finite")
    assert ref.encode(2, S.REAL, 1e300, 2.0 ** 40) == (None, "encoded value is too large")


def test_real_decomposition_branches():
    """products around 2^64 and 2^128 at a 240-bit level: each of the reference's three branches against the restatement"""
    ref, mods = ref_and_moduli([60, 60, 60, 60])
    for e in (62, 63, 64, 65, 126, 127, 128, 129, 200):
        for f in (1.0 - 2.0 ** -53, 1.0, 1.0 + 2.0 ** -52, 1.75):
            for s in (1.0, -1.0):
                assert check(ref, mods, 4, S.REAL, s * 2.0 ** e * f, 1.0) is not None


@pytest.mark.parametrize("level", sorted(LEVELS))
def test_int64_restatement_matches_reference(level):
    ref, mods = ref_and_moduli(LEVELS[level])
    for L in (len(mods), 1):
        for v in S.int64_cases(mods):
            check(ref, mods, L, S.INT64, v, 1.0)


def test_int64_negative_wrap():
    """two 30-bit primes and v = -2^40: the reference reduces (uint64)v + q_j, which is not -|v| mod q_j"""
    ref, mods = ref_and_moduli([30, 30])
    v = -(1 << 40)
    got = check(ref, mods, 2, S.INT64, v, 1.0)
    for j, q in enumerate(mods):
        assert int(got[j, 0]) == ((1 << 64) - (1 << 40)) % q
        assert int(got[j, 0]) != v % q


def test_int64_bit_bound():
    ref, mods = ref_and_moduli([30, 30])
    tb = S.total_bits(mods)
    assert check(ref, mods, 2, S.INT64, (1 << (tb - 3)) - 1, 1.0) is not None
    assert ref.encode(2, S.INT64, 1 << (tb - 3), 1.0) == (None, "encoded value is too large")
    assert ref.encode(2, S.INT64, (1 << 63) - 1, 1.0) == (None, "encoded value is too large")


def test_int64_min_restatement():
    """INT64_MIN: |v| is taken as 2^63 (what llabs yields here; C leaves it undefined), so a 66-bit level refuses it and a larger
    one reduces (uint64)v + q_j.  Checked against the restatement only; the device encoder is held to the same words."""
    mods = R.coeff_modulus_create(N, [60, 60])
    words, err = S.restate(mods, N, S.INT64, -(1 << 63))
    assert err is None and [int(w) for w in words[:, 0]] == [((1 << 63) + q) % q for q in mods]
    assert S.restate(mods[:1], N, S.INT64, -(1 << 63)) == (None, "encoded value is too large")


def test_level_errors():
    ref, mods = ref_and_moduli([60, 60])
    for kind, value in ((S.REAL, 1.0), (S.COMPLEX, 1 + 2j), (S.INT64, 3)):
        assert ref.encode(3, kind, value, 2.0 ** 20) == (None, "parms_id is not valid for encryption parameters")
        assert ref.encode(0, kind, value, 2.0 ** 20) == (None, "parms_id is not valid for encryption parameters")


def test_complex_is_the_vector_encode_of_copies():
    """the reference's complex overload equals its vector encode of n/2 copies, and keeps the vector path's checks"""
    ref, mods = ref_and_moduli([60, 40, 60])
    rc = R.RefContext(R.CKKS, N, mods)
    for z in (1.5 - 0.25j, -3.0 + 0j, 0j):
        got, s = ref.encode(3, S.COMPLEX, z, 2.0 ** 40)
        assert s == 2.0 ** 40
        assert (got == rc.ckks_encode(3, np.full(N // 2, z), 2.0 ** 40)).all()
    assert ref.encode(3, S.COMPLEX, complex(math.inf, 0), 2.0 ** 40) == (None, "values must be finite")
    assert ref.encode(3, S.COMPLEX, 1e300 + 0j, 2.0 ** 40) == (None, "encoded values are too large")
    assert ref.encode(3, S.COMPLEX, 1.0 + 0j, 5e-324) == (None, "scale out of bounds")
