"""Pins the oracle (oracle/seal_oracle.c) to the reference at depth: decryption at 16 and 60 primes on phases at the BGV centring
edge and the BFV rounding edge, CKKS decode at 31 and 63 primes with non-finite slots, CKKS encode at scale 2^1000 on primes below
2^32.  test_gpu_depth.py compares the device with the oracle wherever the reference is not built, so the oracle must agree with it
at these shapes first.  Each case asserts in Python integers the edge it exists for (tests/depth_cases.py)."""
import numpy as np
import pytest

import depth_cases as D
import oracle as O
import refseal as R
from common import assert_slots, assert_words, crt_values, ntt_primes_below, product, rand_ct, residue_rows

pytestmark = pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsealref.so not built")

N = 4096


def t_of(kind, n, mods):
    if kind == "65537":
        return 65537
    if kind == "batch20":
        return ntt_primes_below(20, n, 1)[0]
    return next(p for p in ntt_primes_below(60, n, len(mods) + 1) if p not in mods)


@pytest.mark.parametrize("L", [16, 60])
@pytest.mark.parametrize("kind", ["65537", "batch60"])
def test_bgv_decrypt_centring_edge(L, kind):
    mods = R.coeff_modulus_create(N, [60] * 61)
    t = t_of(kind, N, mods)
    rc, oc = R.RefContext(R.BGV, N, mods, t), O.Oracle(O.BGV, N, mods, t)
    sk = rc.secret_key()
    Q = product(mods[:L])
    rng = np.random.default_rng(L * 7 + len(kind))
    phases = D.bgv_edge_phases(Q, N, rng)
    D.assert_near_half(phases, Q)
    rows = residue_rows(phases, mods, L)
    assert D.order_sensitive_count(rows[:, :512], mods) > 0, "no coefficient depends on the summation order"
    c0 = oc.ntt_forward(L, rows[None])[0]
    ct = np.stack([c0, np.zeros_like(c0)])
    for cf in (1, t - 1, int(rng.integers(2, t - 1))):
        assert_words(oc.decrypt(L, ct, sk, cf), rc.decrypt(L, ct, True, cf), f"BGV L = {L}, t {kind}, centring edge, factor {cf}")
    for size in (2, 4):
        u = rand_ct(rng, mods, N, size, L)
        assert_words(oc.decrypt(L, u, sk, t - 1), rc.decrypt(L, u, True, t - 1), f"BGV L = {L}, t {kind}, uniform size {size}")


@pytest.mark.parametrize("L", [16, 60])
@pytest.mark.parametrize("kind", ["batch20", "batch60"])
def test_bfv_decrypt_rounding_edge(L, kind):
    mods = R.coeff_modulus_create(N, [60] * 61)
    t = t_of(kind, N, mods)
    rc, oc = R.RefContext(R.BFV, N, mods, t), O.Oracle(O.BFV, N, mods, t)
    sk = rc.secret_key()
    Q = product(mods[:L])
    rng = np.random.default_rng(L * 11 + len(kind))
    phases, m, e = D.bfv_phases(Q, t, N, rng)
    D.assert_bfv_edge(Q, t, phases, e)
    ct = np.stack([residue_rows(phases, mods, L), np.zeros((L, N), dtype=np.uint64)])
    got = oc.decrypt(L, ct, sk)
    assert_words(got, rc.decrypt(L, ct, False), f"BFV L = {L}, t {kind}, structured phases")
    small = [j for j in range(N) if abs(e[j]) <= (Q // t) // 4]
    assert all(int(got[j]) == m[j] for j in small), "a noise of at most Delta / 4 does not decrypt to m"
    u = rand_ct(rng, mods, N, 3, L)
    assert_words(oc.decrypt(L, u, sk), rc.decrypt(L, u, False), f"BFV L = {L}, t {kind}, uniform size 3")


@pytest.mark.parametrize("L", [31, 63])
def test_ckks_decode_non_finite(L):
    mods = R.coeff_modulus_create(N, [60] * 64)
    rc, oc = R.RefContext(R.CKKS, N, mods), O.Oracle(O.CKKS, N, mods)
    rng = np.random.default_rng(L)
    Q, T = product(mods[:L]), D.level_bits(mods, L)
    plains = D.decode_plaintexts(oc, mods, N, L, rng)
    plains["encoded"] = oc.ckks_encode(L, D.random_values(rng, N // 2), 2.0 ** 40)
    assert D.negative_with_zero_inf_word(D.composed(oc, L, plains["encoded"], mods), Q, L, 40)
    classes = set()
    for s in D.decode_scales(T):
        for name, p in plains.items():
            want = rc.ckks_decode(L, p, 2.0 ** s)
            assert_slots(oc.ckks_decode(L, p, 2.0 ** s), want, f"L = {L}, {name}, scale 2^{s}")
            w = want.view(np.float64)
            classes |= {"nan"} if np.isnan(w).any() else set()
            classes |= {"inf"} if np.isinf(w).any() else set()
            if name == "encoded" and s == 40:
                assert np.isfinite(w).all()
    assert classes == {"nan", "inf"}, classes


def test_ckks_encode_scale_2_1000_small_primes():
    mods = R.coeff_modulus_create(N, [30] * 61)
    assert max(mods) < 1 << 32
    L = 60
    rc, oc = R.RefContext(R.CKKS, N, mods), O.Oracle(O.CKKS, N, mods)
    rng = np.random.default_rng(1000)
    v = D.random_values(rng, N // 2)
    want = rc.ckks_encode(L, v, 2.0 ** 1000)
    assert want is not None
    assert D.max_exponent(crt_values(oc.ntt_inverse(L, want[None])[0], mods), product(mods[:L])) >= 900
    assert_words(oc.ckks_encode(L, v, 2.0 ** 1000), want, "encode at scale 2^1000, 30-bit primes")
