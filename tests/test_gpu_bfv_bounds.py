"""BFV multiplication and the BFV / BGV plain-modulus range at their bounds (-m gpu).

BFV multiplication (seal_b200/csrc/sb_bfv.cu) lifts both operands into the auxiliary base Bsk, multiplies there and divides by q
on the way back.  Bsk is sized so that the tensor, at most K n t q^2, fits below q prod(B) m_sk (rns.cpp:605-612); uniform random
operands stay far below that.  Here the operands are the centred extremes floor(Q / 2) and ceil(Q / 2) = -floor(Q / 2) of the
level's modulus Q in every coefficient: the tensor of two such constant-coefficient polynomials reaches n floor(Q / 2)^2 at
coefficient n - 1.  Each test asserts in Python integers what its inputs reach and compares every output word with the reference
(tests/refseal.py) or the oracle.  The plain-modulus tests cover 60-bit and power-of-two plain moduli, where the ratio
floor((2^128 - 1) / t) of every t-Barrett step is one below floor(2^128 / t), and the guarded transform of batch_decode
(t >= 2^57)."""
import math

import numpy as np
import pytest

import oracle as O
import refseal as R
from common import (alternating_extreme_ct, assert_words, centred_extreme_ct, max_ct, negacyclic_ones_square, ntt_primes_below,
                    product, rand_ct, zero_ct)

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsealref.so not present")

KS_64, KS_INT = 0, 2  # SB200_LIMIT_KS_ALGORITHM
LIMIT_MSG = "BFV multiplication supports at most 64 primes per level"


def sb():
    import seal_b200

    return seal_b200


def batching_prime_60(n, mods):
    """the largest 60-bit prime = 1 mod 2n that is not a coefficient prime (a 60-bit batching plain modulus)"""
    return next(p for p in ntt_primes_below(60, n, len(mods) + 1) if p not in mods)


def extreme_mixes(mods, n, L, rng, size=2):
    """[name] -> (a, b): the operand pairs of the tensor-bound tests"""
    pos, neg = centred_extreme_ct(mods, n, size, L, +1), centred_extreme_ct(mods, n, size, L, -1)
    alt = alternating_extreme_ct(mods, n, size, L)
    return {"floor(Q/2) x floor(Q/2)": (pos, pos), "floor(Q/2) x ceil(Q/2)": (pos, neg),
            "all q-1 (the integer -1)": (max_ct(mods, n, size, L), max_ct(mods, n, size, L)),
            "alternating floor/ceil(Q/2)": (alt, alt), "random": (rand_ct(rng, mods, n, size, L), rand_ct(rng, mods, n, size, L))}


def check_tensor_reach(ctx, mods, n, L, t):
    """the centred extremes reach n floor(Q/2)^2 at coefficient n - 1 of the tensor; returns the margin in bits of the Bsk rule,
    log2(Q prod(B) m_sk) - log2(n t Q^2)"""
    Q = product(mods[:L])
    bsk = ctx.base_bsk(L)
    c = Q // 2
    top = c * c * negacyclic_ones_square(n)[n - 1]
    assert top == n * c * c and 4 * top >= n * (Q - 1) ** 2, "the tensor reaches n floor(Q/2)^2"
    margin = math.log2(Q * product(bsk)) - math.log2(n * t * Q * Q)
    assert margin > 0, f"n = {n}, t = {t}, |Bsk| = {len(bsk)}: Q prod(B) m_sk does not exceed n t Q^2 (margin {margin:.2f} bits)"
    return margin


# ------------------------------------------------------------------------------------------------------------------------------
# The tensor bound at three shapes: 60-bit primes and a 60-bit batching t; mixed primes and t = 2^59; the largest BFV ring of
# SEAL's default moduli (n = 32768, LOGNA = 7 in the lift and floor kernels' grids).
TENSOR_SHAPES = {
    "n4096-60x4-t60": (4096, lambda: R.coeff_modulus_create(4096, [60] * 4), None),
    "n8192-40.50.60.60-t2^59": (8192, lambda: R.coeff_modulus_create(8192, [40, 50, 60, 60]), 1 << 59),
    "n32768-default-t20": (32768, lambda: R.coeff_modulus_bfv_default(32768), 20),
}


@needs_ref
@pytest.mark.parametrize("shape", list(TENSOR_SHAPES))
def test_tensor_bound_vs_reference(shape):
    S = sb()
    n, mods_fn, t = TENSOR_SHAPES[shape]
    mods = mods_fn()
    t = batching_prime_60(n, mods) if t is None else R.plain_modulus_batching(n, t) if t < 64 else t
    L = len(mods) - 1
    rb = R.RefContext(R.BFV, n, mods, t)
    ctx = S.Context(S.BFV, n, mods, t)
    assert ctx.base_bsk(L) == rb.base_bsk(L)
    margin = check_tensor_reach(ctx, mods, n, L, t)
    mixes = extreme_mixes(mods, n, L, np.random.default_rng(n + L))
    a = np.stack([p[0] for p in mixes.values()])
    b = np.stack([p[1] for p in mixes.values()])
    got, got_sq = ctx.multiply(a, b), ctx.square(a)
    want = []
    for i, name in enumerate(mixes):
        want.append(rb.multiply(L, a[i], b[i]))
        assert_words(got[i], want[i], f"{shape} multiply, {name} (Bsk margin {margin:.2f} bits)")
        assert_words(got_sq[i], rb.square(L, a[i]), f"{shape} square, {name}")
    if shape == "n4096-60x4-t60":
        rk = ctx.load_key(rb.relin_key())
        mr = ctx.multiply_relinearize(a, b, rk)
        for i, name in enumerate(mixes):
            assert_words(mr[i], rb.relinearize(L, want[i]), f"{shape} multiply_relinearize, {name}")


# ------------------------------------------------------------------------------------------------------------------------------
# The |B| rule on both sides: a plain modulus of b* = 61 L + 61 - 32 - bits(Q_L) bits enlarges B by one prime, one of b* - 1
# bits does not and leaves the smallest margin the rule allows.
@needs_ref
@pytest.mark.parametrize("L", [1, 2, 3])
def test_base_size_rule_both_sides_vs_reference(L):
    S = sb()
    n = 4096
    mods = R.coeff_modulus_create(n, [60] * 4)
    b_star = 61 * L + 61 - 32 - product(mods[:L]).bit_length()
    for bits, nB in ((b_star, L + 1), (b_star - 1, L)):
        t = (1 << (bits - 1)) + 1
        rb = R.RefContext(R.BFV, n, mods, t)
        ctx = S.Context(S.BFV, n, mods, t)
        bsk = ctx.base_bsk(L)
        assert bsk == rb.base_bsk(L) and len(bsk) == nB + 1, (L, bits, len(bsk))
        margin = check_tensor_reach(ctx, mods, n, L, t)
        # the rule keeps 32 bits for K (rns.cpp:605-612): without the extra prime the margin is below that
        assert (margin < 32) == (nB == L), f"t of {bits} bits at L = {L}, |B| = {nB}: margin {margin:.2f} bits"
        pos, neg = centred_extreme_ct(mods, n, 2, L, +1), centred_extreme_ct(mods, n, 2, L, -1)
        a, b = np.stack([pos, pos]), np.stack([pos, neg])
        got, got_sq = ctx.multiply(a, b), ctx.square(a)
        for i in range(2):
            assert_words(got[i], rb.multiply(L, a[i], b[i]), f"L = {L}, t of {bits} bits, |B| = {nB}, pair {i}")
        assert_words(got_sq[0], rb.square(L, pos), f"L = {L}, t of {bits} bits, square")


def test_key_level_with_enlarged_base_vs_oracle():
    """multiply at the key level (L = k) when B is enlarged there: |B| = k + 1 primes of the auxiliary list"""
    S = sb()
    n = 4096
    mods = O.coeff_modulus_create(n, [60] * 4)
    k = len(mods)
    t = batching_prime_60(n, mods)
    ctx = S.Context(S.BFV, n, mods, t)
    oc = O.Oracle(O.BFV, n, mods, t)
    assert ctx.base_bsk(k) == oc.base_bsk(k) and len(ctx.base_bsk(k)) == k + 2, "|B| = k + 1 at the key level"
    check_tensor_reach(ctx, mods, n, k, t)
    pos, neg = centred_extreme_ct(mods, n, 2, k, +1), centred_extreme_ct(mods, n, 2, k, -1)
    got = ctx.multiply(np.stack([pos, pos]), np.stack([pos, neg]))
    assert_words(got[0], oc.multiply(k, pos, pos), "key level, floor(Q/2) x floor(Q/2)")
    assert_words(got[1], oc.multiply(k, pos, neg), "key level, floor(Q/2) x ceil(Q/2)")


# ------------------------------------------------------------------------------------------------------------------------------
# General sizes through BEHZ: tensor_general_kernel on the 61-bit Bsk primes and the per-polynomial lift / floor steps.
@needs_ref
@pytest.mark.parametrize("s1,s2", [(3, 3), (2, 15), (8, 8)])
def test_general_sizes_centred_extremes_vs_reference(s1, s2):
    S = sb()
    n = 4096
    mods = R.coeff_modulus_create(n, [60] * 4)
    L = 3
    t = batching_prime_60(n, mods)
    rb = R.RefContext(R.BFV, n, mods, t)
    ctx = S.Context(S.BFV, n, mods, t)
    check_tensor_reach(ctx, mods, n, L, t)
    a = np.stack([centred_extreme_ct(mods, n, s1, L, +1)] * 2)
    b = np.stack([centred_extreme_ct(mods, n, s2, L, -1), centred_extreme_ct(mods, n, s2, L, +1)])
    got = ctx.multiply(a, b)
    for i in range(2):
        assert_words(got[i], rb.multiply(L, a[i], b[i]), f"{s1}x{s2} multiply, pair {i}")


# ------------------------------------------------------------------------------------------------------------------------------
# Chunks: a scratch budget of three ciphertexts cuts a batch of 7 into 3, 3, 1 (op_bfv_multiply), through both entry points.
@needs_ref
def test_multiply_chunks_vs_reference():
    import torch

    S = sb()
    n, batch = 4096, 7
    mods = R.coeff_modulus_create(n, [60] * 4)
    L = 3
    t = batching_prime_60(n, mods)
    rb = R.RefContext(R.BFV, n, mods, t)
    ctx = S.Context(S.BFV, n, mods, t)
    mixes = extreme_mixes(mods, n, L, np.random.default_rng(7))
    rng = np.random.default_rng(8)
    pairs = list(mixes.values()) + [(rand_ct(rng, mods, n, 2, L), rand_ct(rng, mods, n, 2, L)) for _ in range(batch - len(mixes))]
    a, b = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
    want = [rb.multiply(L, a[i], b[i]) for i in range(batch)]
    da, db = torch.from_numpy(a.view(np.int64)).cuda(), torch.from_numpy(b.view(np.int64)).cuda()
    out = torch.empty((batch, 3, L, n), dtype=torch.int64, device="cuda")
    l0 = ctx.launch_count
    ctx.d_multiply(da, db, out, L, batch)
    torch.cuda.synchronize()
    single = ctx.launch_count - l0
    nS = len(ctx.base_bsk(L))
    per = (4 + 3) * (L + nS) * n * 8  # scratch words of one ciphertext: XQ, XS, DQ, DS
    ctx.set_limit(S.Context.LIMIT_SCRATCH_BYTES, 3 * per)
    out.zero_()
    l0 = ctx.launch_count
    ctx.d_multiply(da, db, out, L, batch)
    torch.cuda.synchronize()
    assert ctx.launch_count - l0 == 3 * single, "expected chunks of 3, 3 and 1 ciphertexts"
    got_stream = out.cpu().numpy().view(np.uint64)
    got_host = ctx.multiply(a, b)
    for i in (0, 2, 3, 5, 6):  # first, middle and last chunk
        assert_words(got_stream[i], want[i], f"stream entry point, ciphertext {i} (chunk {i // 3})")
        assert_words(got_host[i], want[i], f"host entry point, ciphertext {i}")
    assert_words(got_stream, got_host, "stream vs host entry point")


# ------------------------------------------------------------------------------------------------------------------------------
# The deepest level the reference serves: 64 primes of 60 bits at n = 4096.  L = 63 (the top data level) against the reference
# and the oracle, L = 64 (the key level) against the oracle; multiply_relinearize at L = 63 in both key-switching modes (63 digits
# is inside the integer path's 64-digit limit at n = 4096).
@needs_ref
def test_deepest_reference_level():
    S = sb()
    n = 4096
    mods = R.coeff_modulus_create(n, [60] * 64)
    t = batching_prime_60(n, mods)
    rb = R.RefContext(R.BFV, n, mods, t)
    ctx = S.Context(S.BFV, n, mods, t)
    oc = O.Oracle(O.BFV, n, mods, t)
    for L in (63, 64):
        assert ctx.base_bsk(L) == oc.base_bsk(L) and len(ctx.base_bsk(L)) == L + 1, "|B| = L: the widest accepted base"
        check_tensor_reach(ctx, mods, n, L, t)
        pos, neg = centred_extreme_ct(mods, n, 2, L, +1), centred_extreme_ct(mods, n, 2, L, -1)
        a, b = np.stack([pos, pos]), np.stack([pos, neg])
        got, got_sq = ctx.multiply(a, b), ctx.square(a)
        for i in range(2):
            w = oc.multiply(L, a[i], b[i])
            assert_words(got[i], w, f"L = {L}, pair {i}, vs oracle")
            if L == 63:
                assert_words(w, rb.multiply(L, a[i], b[i]), f"L = {L}, pair {i}: oracle vs reference")
        assert_words(got_sq[0], oc.multiply(L, pos, pos), f"L = {L}, square, vs oracle")
    L = 63
    assert ctx.base_bsk(L) == rb.base_bsk(L)
    rk = ctx.load_key(rb.relin_key())
    pos, neg = centred_extreme_ct(mods, n, 2, L, +1), centred_extreme_ct(mods, n, 2, L, -1)
    want = rb.relinearize(L, rb.multiply(L, pos, neg))
    for mode in (KS_INT, KS_64):
        ctx.set_limit(S.Context.LIMIT_KS_ALGORITHM, mode)
        assert_words(ctx.multiply_relinearize(pos, neg, rk), want, f"multiply_relinearize at L = 63, key-switching mode {mode}")


# ------------------------------------------------------------------------------------------------------------------------------
# The level limit: at 65 primes every BFV-multiply entry point returns the argument error before any launch; the same context
# then multiplies at 64 primes (BEHZ at a level depends only on that level's primes, t and n, so the oracle of the first 64
# primes is the reference for it).
def test_multiply_level_limit():
    import torch

    S = sb()
    n, t = 4096, 65537
    mods = ntt_primes_below(30, n, 66)
    ctx = S.Context(S.BFV, n, mods, t)
    L = 65
    a = centred_extreme_ct(mods, n, 2, L, +1, batch=1)
    a3 = centred_extreme_ct(mods, n, 3, L, +1, batch=1)
    key = ctx.load_key(np.zeros((L, 2, len(mods), n), dtype=np.uint64))
    err = f"error -1: {LIMIT_MSG}"
    host_calls = {"multiply": lambda: ctx.multiply(a, a), "square": lambda: ctx.square(a), "multiply_sized": lambda: ctx.multiply(a3, a),
                  "multiply_relinearize": lambda: ctx.multiply_relinearize(a, a, key), "base_bsk": lambda: ctx.base_bsk(L)}
    for name, call in host_calls.items():
        with pytest.raises(ValueError, match=err):
            call()
    da, da3 = torch.from_numpy(a.view(np.int64)).cuda(), torch.from_numpy(a3.view(np.int64)).cuda()
    out3 = torch.zeros((1, 3, L, n), dtype=torch.int64, device="cuda")
    out4 = torch.zeros((1, 4, L, n), dtype=torch.int64, device="cuda")
    out2 = torch.zeros((1, 2, L, n), dtype=torch.int64, device="cuda")

    def stream_square():
        S._check(S.lib().sb200_square(ctx.h, L, 1, S._dp(da), S._dp(out3), ctx._stream()))

    stream_calls = {"multiply": lambda: ctx.d_multiply(da, da, out3, L, 1), "square": stream_square,
                    "multiply_sized": lambda: ctx.d_multiply_sized(da3, da, out4, L, 3, 2, 1),
                    "multiply_relinearize": lambda: ctx.d_multiply_relinearize(da, da, key, out2, L, 1)}
    for name, call in stream_calls.items():
        with pytest.raises(ValueError, match=err):
            call()
    torch.cuda.synchronize()
    assert not out3.any() and not out4.any() and not out2.any(), "a rejected call wrote its output"
    L = 64
    oc = O.Oracle(O.BFV, n, mods[:L], t)
    assert ctx.base_bsk(L) == oc.base_bsk(L)
    pos, neg = centred_extreme_ct(mods, n, 2, L, +1), centred_extreme_ct(mods, n, 2, L, -1)
    assert_words(ctx.multiply(pos, neg), oc.multiply(L, pos, neg), "multiply at 64 primes after the rejected calls")


# ------------------------------------------------------------------------------------------------------------------------------
# Plain-modulus edges outside multiplication: a 60-bit batching t (batch_decode's guarded transform, t >= 2^57) and t = 2^59
# (floor((2^128 - 1) / t) is one below floor(2^128 / t), so every t-Barrett step needs its extra conditional subtraction).
PLAIN_BITS = [60, 60, 60, 50]


def plain_edges(t):
    return [t - 1, 0, (t - 1) // 2, (t + 1) // 2, t // 2 - 1, t // 2]


def edge_rows(t, rng, batch, n):
    v = rng.integers(0, t, (batch, n), dtype=np.uint64)
    v[0] = np.resize(np.array(plain_edges(t), dtype=np.uint64), n)
    v[1, :6] = plain_edges(t)
    return v


def t_of(kind, n, mods):
    t = batching_prime_60(n, mods) if kind == "prime60" else 1 << 59
    if kind == "pow2_59":
        assert (2 ** 128 - 1) // t == 2 ** 128 // t - 1, "the t-Barrett ratio is one below floor(2^128 / t)"
    else:
        assert t >> 57 and (t - 1) % (2 * n) == 0, "a batching plain modulus above 2^57"
    return t


@needs_ref
def test_batch_codec_60bit_plain_modulus_vs_reference():
    S = sb()
    n, batch = 4096, 3
    mods = R.coeff_modulus_create(n, PLAIN_BITS)
    t = t_of("prime60", n, mods)
    rc = R.RefContext(R.BFV, n, mods, t)
    ctx = S.Context(S.BFV, n, mods, t)
    rng = np.random.default_rng(60)
    v, w = edge_rows(t, rng, batch, n), edge_rows(t, rng, batch, n)
    p, d = ctx.batch_encode(v), ctx.batch_decode(w)
    for i in range(batch):
        assert_words(p[i], rc.batch_codec(v[i], False), f"batch_encode, row {i}")
        assert_words(d[i], rc.batch_codec(w[i], True), f"batch_decode, row {i}")
    assert_words(ctx.batch_decode(p), v, "decode(encode(v))")


@needs_ref
@pytest.mark.parametrize("kind", ["prime60", "pow2_59"])
def test_bfv_decrypt_large_plain_modulus_vs_reference(kind):
    """phases all-(q-1) (the integer -1), floor(Q/2), ceil(Q/2) (c_1 = 0, so the phase is c_0) and random ciphertexts of sizes
    2 and 3"""
    S = sb()
    n = 4096
    mods = R.coeff_modulus_create(n, PLAIN_BITS)
    t = t_of(kind, n, mods)
    rc = R.RefContext(R.BFV, n, mods, t)
    ctx = S.Context(S.BFV, n, mods, t)
    sk = ctx.load_secret_key(rc.secret_key())
    rng = np.random.default_rng(61)
    for L in (3, 1):
        zero = zero_ct(mods, n, 1, L)[0]
        phases = [max_ct(mods, n, 1, L)[0], centred_extreme_ct(mods, n, 1, L, +1)[0], centred_extreme_ct(mods, n, 1, L, -1)[0]]
        ct = np.stack([np.stack([c0, zero]) for c0 in phases] + [rand_ct(rng, mods, n, 2, L)])
        for c in (ct, rand_ct(rng, mods, n, 3, L, batch=2)):
            got = ctx.decrypt(c, sk)
            for i in range(c.shape[0]):
                assert_words(got[i], rc.decrypt(L, c[i], False), f"t {kind}, L = {L}, size {c.shape[1]}, ciphertext {i}")


@needs_ref
def test_bfv_plain_ops_power_of_two_plain_modulus_vs_reference():
    S = sb()
    n, batch = 4096, 3
    mods = R.coeff_modulus_create(n, PLAIN_BITS)
    t = t_of("pow2_59", n, mods)
    rc = R.RefContext(R.BFV, n, mods, t)
    ctx = S.Context(S.BFV, n, mods, t)
    rng = np.random.default_rng(62)
    for L in (3, 1):
        plain = edge_rows(t, rng, batch, n)
        for a in (rand_ct(rng, mods, n, 2, L, batch), max_ct(mods, n, 2, L, batch)):
            ap, sp = ctx.add_plain_coeff(a, plain, False), ctx.add_plain_coeff(a, plain, True)
            for ntt in (False, True):
                mp = ctx.multiply_plain_coeff(a, plain, ntt)
                for i in range(batch):
                    assert_words(mp[i], rc.plain_op_coeff(0, L, a[i], plain[i], ntt), f"multiply_plain, L = {L}, ntt {ntt}, row {i}")
            for i in range(batch):
                assert_words(ap[i], rc.plain_op_coeff(1, L, a[i], plain[i], False), f"add_plain, L = {L}, row {i}")
                assert_words(sp[i], rc.plain_op_coeff(2, L, a[i], plain[i], False), f"sub_plain, L = {L}, row {i}")


@needs_ref
@pytest.mark.parametrize("kind", ["prime60", "pow2_59"])
def test_bgv_plain_modulus_edges_vs_reference(kind):
    """decrypt, mod_switch_to_next and add_plain / sub_plain with correction factors up to t - 1 (the plaintext is scaled by the
    factor modulo t before the lift)"""
    S = sb()
    n, batch = 4096, 3
    mods = R.coeff_modulus_create(n, PLAIN_BITS)
    t = t_of(kind, n, mods)
    rc = R.RefContext(R.BGV, n, mods, t)
    ctx = S.Context(S.BGV, n, mods, t)
    sk = ctx.load_secret_key(rc.secret_key())
    rng = np.random.default_rng(63)
    cf = np.array([1, t - 1, t - 3], dtype=np.uint64)
    for L in (3, 2):
        a = np.stack([max_ct(mods, n, 2, L), rand_ct(rng, mods, n, 2, L), rand_ct(rng, mods, n, 2, L)])
        plain = edge_rows(t, rng, batch, n)
        got, ms = ctx.decrypt(a, sk, cf), ctx.mod_switch_to_next(a)
        ap, sp = ctx.add_plain_coeff(a, plain, False, cf), ctx.add_plain_coeff(a, plain, True, cf)
        for i in range(batch):
            f = int(cf[i])
            assert_words(got[i], rc.decrypt(L, a[i], True, f), f"BGV decrypt, L = {L}, ciphertext {i}")
            assert_words(ms[i], rc.mod_switch(L, a[i]), f"BGV mod_switch_to_next, L = {L}, ciphertext {i}")
            assert_words(ap[i], rc.plain_op_coeff(1, L, a[i], plain[i], True, f), f"BGV add_plain, L = {L}, ciphertext {i}")
            assert_words(sp[i], rc.plain_op_coeff(2, L, a[i], plain[i], True, f), f"BGV sub_plain, L = {L}, ciphertext {i}")
