"""Decryption and the CKKS encoder at depth (-m gpu): 16 to 64 primes, where the code takes branches a shallow level never reaches.

- BGV decryption rounds sum_i x_i / q_i + 0.5 in doubles, in prime order (bgv_modt_kernel, sb_engine.cu); phases next to Q / 2
  make the result depend on that order.  The noise budget of the same ciphertexts is checked too.
- BFV decryption accumulates up to 60 products in 128 bits (bfv_scale_round_kernel); phases Delta m + e sit at its rounding edge.
- CKKS decode multiplies word w of each composed coefficient by 2^(64 w) / scale, which is +inf from word 17 on at scale 2^40
  (ckks_compose_kernel, sb_ckks.cu); slots can be finite, +-inf or NaN.  Every slot the reference does not make NaN must match it
  bit for bit, and exactly its NaN slots must be NaN (include/seal_b200.h, CKKSEncoder).
- CKKS encode at scale 2^1000 reduces |round(c)| = mant 2^ex with ex near 950 (ckks_reduce_kernel), also on primes below 2^32.
- The transform at n = 8 (a 4-thread block), 2048 (the scaled stage inside the shared-memory kernel) and 131072.

Every output word is compared with the oracle (oracle/seal_oracle.c, itself pinned to the reference at these shapes by
test_depth_oracle.py) and, where oracle/_ref/libsealref.so is present, with the reference.  Each case asserts in Python integers
the edge it exists for (tests/depth_cases.py)."""
import ctypes
import functools

import numpy as np
import pytest

import depth_cases as D
import noise_ref as NR
import oracle as O
import refseal as R
from common import assert_slots, assert_words, ntt_primes_below, product, rand_ct, residue_rows, ternary_secret_key

pytestmark = pytest.mark.gpu

BFV, CKKS, BGV = 1, 2, 3  # the same ids in seal_b200, the oracle and the reference
DEEP = (4096, (60,) * 61)
DEEP64 = (4096, (60,) * 64)
HEADLINE = (65536, (55,) * 32)
DECRYPT_SHAPES = {"n4096-L16": (DEEP, 16), "n4096-L31": (DEEP, 31), "n4096-L60": (DEEP, 60), "n65536-L31": (HEADLINE, 31)}


def decrypt_cases(kinds):
    """(shape, plain modulus kind): every kind at n = 4096, the 60-bit batching prime at the headline shape"""
    return [(sh, k) for sh in DECRYPT_SHAPES for k in kinds if DECRYPT_SHAPES[sh][0] is DEEP or k == "batch60"]


def sb():
    import seal_b200

    return seal_b200


def dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


@functools.lru_cache(maxsize=None)
def moduli(n, bits):
    return tuple(O.coeff_modulus_create(n, list(bits)))


def plain_modulus(kind, n, mods):
    if kind == "65537":
        return 65537
    if kind == "batch20":
        return ntt_primes_below(20, n, 1)[0]
    return next(p for p in ntt_primes_below(60, n, len(mods) + 1) if p not in mods)


class Setup:
    """one parameter set on the device, in the oracle and (when built) in the reference, under one secret key"""

    def __init__(self, scheme, n, bits, t):
        S = sb()
        self.n, self.mods, self.t = n, list(moduli(n, bits)), t
        self.rc = R.RefContext(scheme, n, self.mods, t) if R.available() else None
        self.oc = O.Oracle(scheme, n, self.mods, t)
        self.ctx = S.Context(scheme, n, self.mods, t)
        k = len(self.mods)
        self.sk_host = self.rc.secret_key() if self.rc else ternary_secret_key(
            np.random.default_rng(n + k), self.mods, n, lambda rows: self.oc.ntt_forward(k, rows[None])[0])
        self.sk = self.ctx.load_secret_key(self.sk_host)


@functools.lru_cache(maxsize=3)
def setup(scheme, n, bits, t=0):
    return Setup(scheme, n, bits, t)


@pytest.fixture(scope="module", autouse=True)
def _release_contexts():
    yield
    setup.cache_clear()


def check_decrypt(s, L, ct, cf, is_ntt, what):
    """device decryption of the batch ct [B][size][L][n] against the oracle and the reference, one ciphertext at a time"""
    got = s.ctx.decrypt(ct, s.sk, cf)
    for i in range(ct.shape[0]):
        f = 1 if cf is None else int(cf[i])
        assert_words(got[i], s.oc.decrypt(L, ct[i], s.sk_host, f), f"{what}, ciphertext {i} vs oracle")
        if s.rc is not None:
            assert_words(got[i], s.rc.decrypt(L, ct[i], is_ntt, f), f"{what}, ciphertext {i} vs reference")
    return got


# ------------------------------------------------------------------------------------------------------------------------------
# BGV at the centring edge: c_1 = 0 and c_0 = NTT(v) with v = floor(Q/2), ceil(Q/2), (Q -+ 1)/2 + d (|d| <= 2^20)
@pytest.mark.parametrize("shape,kind", decrypt_cases(["65537", "batch60"]))
def test_bgv_decrypt_centring_edge(shape, kind):
    (n, bits), L = DECRYPT_SHAPES[shape]
    mods = moduli(n, bits)
    t = plain_modulus(kind, n, mods)
    s = setup(BGV, n, bits, t)
    Q = product(mods[:L])
    rng = np.random.default_rng(L + n + t % 97)
    phases = D.bgv_edge_phases(Q, n, rng)
    D.assert_near_half(phases, Q)
    rows = residue_rows(phases, mods, L)
    assert D.order_sensitive_count(rows[:, :256], mods) > 0, "no coefficient's rounding depends on the summation order"
    c0 = s.oc.ntt_forward(L, rows[None])[0]
    edge = np.stack([c0, np.zeros_like(c0)])
    r = int(rng.integers(2, t - 1))
    ct2 = np.stack([edge, edge, edge, rand_ct(rng, mods, n, 2, L)])
    cf2 = np.array([1, t - 1, r, r], dtype=np.uint64)
    check_decrypt(s, L, ct2, cf2, True, f"BGV {shape}, t {kind}, size 2 (centring edge x3, uniform)")
    for size in (3, 4):
        ct = rand_ct(rng, mods, n, size, L, batch=2)
        check_decrypt(s, L, ct, np.array([t - 1, r], dtype=np.uint64), True, f"BGV {shape}, t {kind}, uniform size {size}")
    # invariant_noise_budget of the same ciphertexts: with c_1 = 0 the noise is the centred phase itself
    budgets = s.ctx.invariant_noise_budget(ct2, s.sk)
    norm = max(abs(v - Q if v > Q // 2 else v) for v in phases)
    assert int(budgets[0]) == max(0, Q.bit_length() - norm.bit_length() - 1) == int(budgets[2])
    if s.rc is not None and NR.available():
        for i in range(ct2.shape[0]):
            assert NR.ref_budget(s.rc, L, ct2[i], True) == (0, int(budgets[i])), f"noise budget, ciphertext {i}"


# ------------------------------------------------------------------------------------------------------------------------------
# BFV: phases Delta m + e (c_1 = 0, coefficient form) with e at 0, +-1, +-Delta/4 and the rounding edge +-Delta/2 (+-1)
@pytest.mark.parametrize("shape,kind", decrypt_cases(["batch20", "batch60"]))
def test_bfv_decrypt_rounding_edge(shape, kind):
    (n, bits), L = DECRYPT_SHAPES[shape]
    mods = moduli(n, bits)
    t = plain_modulus(kind, n, mods)
    s = setup(BFV, n, bits, t)
    Q = product(mods[:L])
    assert L * max(mods[:L]) * (1 << 61) < 1 << 128, "the 128-bit sums of bfv_scale_round_kernel hold L products"
    rng = np.random.default_rng(L + n + t % 89)
    phases, m, e = D.bfv_phases(Q, t, n, rng)
    D.assert_bfv_edge(Q, t, phases, e)
    structured = np.stack([residue_rows(phases, mods, L), np.zeros((L, n), dtype=np.uint64)])
    ct2 = np.stack([structured, rand_ct(rng, mods, n, 2, L)])
    got = check_decrypt(s, L, ct2, None, False, f"BFV {shape}, t {kind}, size 2 (structured, uniform)")
    small = [j for j in range(n) if abs(e[j]) <= (Q // t) // 4]
    assert all(int(got[0][j]) == m[j] for j in small), "a noise of at most Delta / 4 does not decrypt to m"
    check_decrypt(s, L, rand_ct(rng, mods, n, 3, L, batch=2), None, False, f"BFV {shape}, t {kind}, uniform size 3")


@pytest.mark.parametrize("L", [60, 63])
def test_ckks_decrypt_deep(L):
    n, bits = DEEP64
    s = setup(CKKS, n, bits)
    rng = np.random.default_rng(L)
    for size in (2, 3):
        check_decrypt(s, L, rand_ct(rng, s.mods, n, size, L, batch=2), None, True, f"CKKS L = {L}, size {size}")


# ------------------------------------------------------------------------------------------------------------------------------
# Chunks: a scratch budget of two ciphertexts cuts a batch of 5 at L = 60 into 2, 2 and 1 (decrypt_phases), correction factors
# following their ciphertexts across the cut; stream and host entry points give the single-chunk words.
@pytest.mark.parametrize("scheme", [BGV, BFV])
def test_decrypt_chunks(scheme):
    import torch

    S = sb()
    n, bits = DEEP
    L, batch, size = 60, 5, 2
    mods = moduli(n, bits)
    t = plain_modulus("batch60", n, mods)
    s = setup(scheme, n, bits, t)
    rng = np.random.default_rng(scheme)
    ct = rand_ct(rng, mods, n, size, L, batch=batch)
    cf = np.array([1, t - 1, 3, 5, t - 2], dtype=np.uint64) if scheme == BGV else None
    want = check_decrypt(s, L, ct, cf, scheme == BGV, f"scheme {scheme}, L = 60, one chunk")  # also builds the key powers
    d_ct = dev(ct)
    out = torch.zeros((batch, n), dtype=torch.int64, device="cuda")
    cf_p = None if cf is None else cf.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64))

    def stream():
        out.zero_()
        l0 = s.ctx.launch_count
        S._check(S.lib().sb200_decrypt(s.ctx.h, s.sk.h, L, size, batch, S._dp(d_ct), cf_p, S._dp(out), s.ctx._stream()))
        torch.cuda.synchronize()
        return s.ctx.launch_count - l0, out.cpu().numpy().view(np.uint64).copy()

    single, got = stream()
    assert_words(got, want, "stream entry point, one chunk")
    per = (L * n * (size if scheme == BFV else 1) + 1) * 8  # decrypt_phases' scratch per ciphertext
    s.ctx.set_limit(S.Context.LIMIT_SCRATCH_BYTES, 2 * per)
    try:
        chunked, got = stream()
        assert chunked == 3 * single, "expected chunks of 2, 2 and 1 ciphertexts"
        assert_words(got, want, "stream entry point, chunks of 2, 2, 1")
        assert_words(s.ctx.decrypt(ct, s.sk, cf), want, "host entry point, chunks of 2, 2, 1")
    finally:
        s.ctx.set_limit(S.Context.LIMIT_SCRATCH_BYTES, 8 << 30)


# ------------------------------------------------------------------------------------------------------------------------------
# CKKS decode at depth.  With 60-bit primes L = 18 is the last level whose Q fits in 17 words (word 17, whose factor is +inf at
# scale 2^40, is zero in Q and in every coefficient), L = 19 the first with a nonzero word 17; 63 and 64 are the top data level and
# the key level of a 64-prime context.
DECODE_LEVELS = {"n4096-L16": (DEEP64, 16), "n4096-L18": (DEEP64, 18), "n4096-L19": (DEEP64, 19), "n4096-L63": (DEEP64, 63),
                 "n4096-L64": (DEEP64, 64), "n65536-L31": (HEADLINE, 31)}


@pytest.mark.parametrize("level", list(DECODE_LEVELS))
def test_ckks_decode_depth(level):
    import torch

    S = sb()
    (n, bits), L = DECODE_LEVELS[level]
    s = setup(CKKS, n, bits)
    mods, Q, T = s.mods, product(s.mods[:L]), D.level_bits(s.mods, L)
    rc = s.rc if L < len(mods) else None  # the reference decodes data levels only
    # the loop runs over L words: from L = 18 on word 17's factor is +inf, and from L = 19 on Q itself is nonzero there
    assert bool(D.inf_words(L, 40)) == (L >= 18)
    assert any(Q >> (64 * w) for w in D.inf_words(L, 40)) == (T > 17 * 64), "Q has a word 17 exactly when it needs 18 words"
    rng = np.random.default_rng(L + n)
    values = D.random_values(rng, n // 2)
    enc = s.ctx.ckks_encode(values, L, 2.0 ** 40)
    assert_words(enc, s.oc.ckks_encode(L, values, 2.0 ** 40), f"{level}: encode at scale 2^40 vs oracle")
    if rc is not None:
        assert_words(enc, rc.ckks_encode(L, values, 2.0 ** 40), f"{level}: encode at scale 2^40 vs reference")
    if D.inf_words(L, 40):
        assert D.negative_with_zero_inf_word(D.composed(s.oc, L, enc, mods), Q, L, 40), "no negative coefficient meets 0 * inf"
    plains = {"encoded": enc, **D.decode_plaintexts(s.oc, mods, n, L, rng)}
    names, batch = list(plains), np.stack(list(plains.values()))
    for sc in D.decode_scales(T):
        got = s.ctx.ckks_decode(batch, 2.0 ** sc)
        for i, name in enumerate(names):
            what = f"{level}: decode of {name} at scale 2^{sc}"
            assert_slots(got[i], s.oc.ckks_decode(L, batch[i], 2.0 ** sc), what + " vs oracle")
            if rc is not None and (n <= 4096 or sc == 40):  # the reference's decode at n = 65536 takes most of a second
                assert_slots(got[i], rc.ckks_decode(L, batch[i], 2.0 ** sc), what + " vs reference")
        if sc == 40:
            assert np.isfinite(got[0].view(np.float64)).all() and np.abs(got[0] - values).max() < 1e-6, "round trip"
            # the host entry point cut into one plaintext per chunk against the stream entry point
            d_out = torch.zeros((len(names), n), dtype=torch.float64, device="cuda")
            s.ctx.d_ckks_decode(dev(batch), d_out, L, len(names), 2.0 ** sc)
            torch.cuda.synchronize()
            stream = d_out.cpu().numpy().view(np.uint64)
            s.ctx.set_limit(S.Context.LIMIT_HOST_STAGE_BYTES, L * n * 8 + n * 8)
            try:
                host = s.ctx.ckks_decode(batch, 2.0 ** sc)
            finally:
                s.ctx.set_limit(S.Context.LIMIT_HOST_STAGE_BYTES, 640 << 20)
            assert_words(host.view(np.uint64), stream, f"{level}: host entry point in chunks vs stream entry point")
            assert_words(got.view(np.uint64), stream, f"{level}: host entry point vs stream entry point")


# ------------------------------------------------------------------------------------------------------------------------------
# CKKS encode at depth: scales up to 2^1000 (ex up to about 950), on 60-bit primes and on primes below 2^32
@pytest.mark.parametrize("shape", ["n4096-60x64-L63", "n4096-30x61-L60"])
def test_ckks_encode_large_scale(shape):
    n, bits, L = {"n4096-60x64-L63": (4096, (60,) * 64, 63), "n4096-30x61-L60": (4096, (30,) * 61, 60)}[shape]
    s = setup(CKKS, n, bits)
    if bits[0] == 30:
        assert max(s.mods) < 1 << 32, "primes below 2^32: the multiplier 2^32 exceeds every modulus"
    rng = np.random.default_rng(L)
    values = np.stack([D.random_values(rng, n // 2) for _ in range(2)])
    for sc in (600, 1000):
        got = s.ctx.ckks_encode(values, L, 2.0 ** sc)
        for i in range(2):
            want = s.oc.ckks_encode(L, values[i], 2.0 ** sc)
            assert_words(got[i], want, f"{shape}: encode at scale 2^{sc}, plaintext {i} vs oracle")
            if s.rc is not None:
                assert_words(got[i], s.rc.ckks_encode(L, values[i], 2.0 ** sc), f"{shape}: scale 2^{sc}, plaintext {i} vs reference")
        if sc == 1000:
            assert D.max_exponent(D.composed(s.oc, L, got[0], s.mods), product(s.mods[:L])) >= 900


def test_ckks_encode_bounds():
    """both sides of each rejection: the bit count of the largest coefficient (T - 1 accepted, T rejected) and of the scale, at a
    level below 1000 bits; at a level above 1024 bits only an overflow to inf rejects"""
    n = 4096
    s = setup(CKKS, n, (60,) * 16)
    L = 15
    T = D.level_bits(s.mods, L)
    assert T < 1000
    slots = n // 2

    def accepted(values, sc, what):
        got = s.ctx.ckks_encode(values, L, sc)
        assert_words(got, s.oc.ckks_encode(L, values, sc), what + " vs oracle")
        if s.rc is not None:
            assert_words(got, s.rc.ckks_encode(L, values, sc), what + " vs reference")

    def rejected(values, sc, msg, what):
        with pytest.raises(ValueError, match=msg):
            s.ctx.ckks_encode(values, L, sc)
        assert s.oc.ckks_encode(L, values, sc) is None, what + ": the oracle accepts"
        if s.rc is not None:
            assert s.rc.ckks_encode(L, values, sc) is None, what + ": the reference accepts"

    # a constant c in every slot encodes to the constant polynomial c * scale: 1.5 * 2^(T-3) has T - 1 bits with the sign, 2.5 * 2^(T-3) T
    accepted(np.full(slots, 1.5 + 0j), 2.0 ** (T - 3), "constant 1.5 at scale 2^(T-3)")
    rejected(np.full(slots, 2.5 + 0j), 2.0 ** (T - 3), "encoded values are too large", "constant 2.5 at scale 2^(T-3)")
    small = D.random_values(np.random.default_rng(15), slots, 1e-3)
    assert int(np.log2(2.0 ** (T - 2))) + 1 == T - 1 and int(np.log2(2.0 ** (T - 1))) + 1 == T
    accepted(small, 2.0 ** (T - 2), "scale 2^(T-2)")
    rejected(small, 2.0 ** (T - 1), "scale out of bounds", "scale 2^(T-1)")
    # above 1024 bits: every finite coefficient has fewer bits than the level, so only inf rejects
    big = setup(CKKS, n, (60,) * 64)
    L2 = 20
    assert D.level_bits(big.mods, L2) > 1025
    got = big.ctx.ckks_encode(np.full(slots, 2.0 ** 10 + 0j), L2, 2.0 ** 1000)
    assert_words(got, big.oc.ckks_encode(L2, np.full(slots, 2.0 ** 10 + 0j), 2.0 ** 1000), "2^10 at scale 2^1000 vs oracle")
    with pytest.raises(ValueError, match="encoded values are too large"):
        big.ctx.ckks_encode(np.full(slots, 2.0 ** 30 + 0j), L2, 2.0 ** 1000)
    assert big.oc.ckks_encode(L2, np.full(slots, 2.0 ** 30 + 0j), 2.0 ** 1000) is None
    if big.rc is not None:
        assert big.rc.ckks_encode(L2, np.full(slots, 2.0 ** 30 + 0j), 2.0 ** 1000) is None


# ------------------------------------------------------------------------------------------------------------------------------
# Transform sizes: n = 8 (a 4-thread block), 2048 (the scaled last stage inside the shared-memory kernel, 1024 threads) and 131072
FFT_SHAPES = {"n8": (8, (40, 40, 40)), "n2048": (2048, (50, 50, 50)), "n131072": (131072, (60, 60, 60))}


@pytest.mark.parametrize("shape", list(FFT_SHAPES))
def test_ckks_fft_sizes(shape):
    n, bits = FFT_SHAPES[shape]
    s = setup(CKKS, n, bits)
    L, batch = 2, 3
    rng = np.random.default_rng(n)
    values = np.stack([D.random_values(rng, n // 2) for _ in range(batch)])
    enc = s.ctx.ckks_encode(values, L, 2.0 ** 40)
    uni = np.stack([np.stack([rng.integers(0, s.mods[j], n, dtype=np.uint64) for j in range(L)]) for _ in range(batch)])
    dec, dec_uni = s.ctx.ckks_decode(enc, 2.0 ** 40), s.ctx.ckks_decode(uni, 2.0 ** 40)
    for i in range(batch):
        want = s.oc.ckks_encode(L, values[i], 2.0 ** 40)
        assert_words(enc[i], want, f"{shape}: encode {i} vs oracle")
        assert_slots(dec[i], s.oc.ckks_decode(L, enc[i], 2.0 ** 40), f"{shape}: round trip {i} vs oracle")
        assert_slots(dec_uni[i], s.oc.ckks_decode(L, uni[i], 2.0 ** 40), f"{shape}: decode of uniform {i} vs oracle")
        if s.rc is not None:
            assert_words(enc[i], s.rc.ckks_encode(L, values[i], 2.0 ** 40), f"{shape}: encode {i} vs reference")
            assert_slots(dec[i], s.rc.ckks_decode(L, enc[i], 2.0 ** 40), f"{shape}: round trip {i} vs reference")
            assert_slots(dec_uni[i], s.rc.ckks_decode(L, uni[i], 2.0 ** 40), f"{shape}: decode of uniform {i} vs reference")
    assert np.isfinite(dec.view(np.float64)).all() and np.abs(dec - values).max() < 1e-6, "round trip"
