"""Sums of ciphertext products (sb200_multiply_sum / _host): output j = add_many over i of multiply(lhs_{j K + i}, rhs_i), word for
word against the chained device calls (sb200_multiply of every term, then sb200_add_many, both pinned to the reference by
tests/test_gpu_parity.py and tests/test_gpu_compositions.py), against a Python-integer restatement (NTT-form schemes) and against
the reference's own multiply + add chain (oracle/_ref); and the C++ members (tests/cpp/shim_multsum_test.cpp) against
seal::Evaluator."""
import os
import subprocess

import numpy as np
import pytest

import oracle as O
import refseal as R
from common import assert_words, rand_ct

pytestmark = pytest.mark.gpu

WINDOW = 128  # kMultiplySumWindow (seal_b200/csrc/sb_engine.cuh), at every prime below 2^60
WINDOW_61 = 32  # at the largest 61-bit primes (tests/test_multiply_sum_bounds.py)


def sb():
    import seal_b200

    return seal_b200


def dev(x):
    import torch

    return torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint64)


def context(scheme, n, bits, t=0):
    mods = O.coeff_modulus_create(n, bits)
    if scheme != sb().CKKS and not t:
        t = int(O.get_primes(2 * n, 20, 1)[0])
    return mods, t, sb().Context(scheme, n, mods, t)


def chain(ctx, lhs, rhs, modes=None, factors=None):
    """the chained device calls: multiply of every term, then one add_many per output"""
    K = len(rhs)
    M = len(lhs) // K
    return [ctx.add_many([ctx.multiply(lhs[j * K + i], rhs[i]) for i in range(K)], modes, factors) for j in range(M)]


def constants(q, K, modes, factors):
    consts, tail = [0] * K, 1
    for i in range(K - 1, -1, -1):
        m = modes[i - 1] if (i and modes is not None) else 0
        v = (int(factors[i - 1][1]) % q if m & 2 else 1) * tail % q
        consts[i] = (q - v) % q if m & 1 else v
        if m & 2:
            tail = tail * (int(factors[i - 1][0]) % q) % q
    return consts


def restate(mods, lhs, rhs, modes=None, factors=None):
    """Python integers: sum_i c_i (a0 b0, a0 b1 + a1 b0, a1 b1) mod q, words reduced first, c_i the fold's per-term constant"""
    K = len(rhs)
    M = len(lhs) // K
    B, _, L, n = rhs[0].shape
    outs = []
    for j in range(M):
        o = np.zeros((B, 3, L, n), dtype=np.uint64)
        for li in range(L):
            q = int(mods[li])
            c = constants(q, K, modes, factors)
            for b in range(B):
                acc = [np.zeros(n, dtype=object) for _ in range(3)]
                for i in range(K):
                    a0, a1 = (lhs[j * K + i][b, s, li].astype(object) % q for s in (0, 1))
                    b0, b1 = (rhs[i][b, s, li].astype(object) % q for s in (0, 1))
                    a0, a1 = a0 * c[i] % q, a1 * c[i] % q
                    acc[0] = acc[0] + a0 * b0
                    acc[1] = acc[1] + a0 * b1 + a1 * b0
                    acc[2] = acc[2] + a1 * b1
                for s in range(3):
                    o[b, s, li] = (acc[s] % q).astype(np.uint64)
        outs.append(o)
    return outs


def fused_both(ctx, lhs, rhs, modes=None, factors=None):
    """the host entry point, and the stream entry point on device tensors (inputs checked unchanged); returns the host result"""
    import torch

    got = ctx.multiply_sum(lhs, rhs, modes, factors)
    B, _, L, n = rhs[0].shape
    K, M = len(rhs), len(lhs) // len(rhs)
    d_rhs = [dev(c) for c in rhs]
    d_lhs = [d_rhs[[i for i in range(K) if rhs[i] is a][0]] if any(rhs[i] is a for i in range(K)) else dev(a) for a in lhs]
    d_outs = [dev(np.zeros((B, 3, L, n), dtype=np.uint64)) for _ in range(M)]
    ctx.d_multiply_sum(d_lhs, d_rhs, d_outs, L, B, modes, factors)
    torch.cuda.synchronize()
    for j in range(M):
        assert_words(host(d_outs[j]), got[j], f"stream vs host entry point, output {j}")
    for i in range(K):
        assert_words(host(d_rhs[i]), rhs[i], "right-hand operand unchanged")
    return got


def inputs(rng, mods, n, L, B, K, M):
    return [rand_ct(rng, mods, n, 2, L, B) for _ in range(M * K)], [rand_ct(rng, mods, n, 2, L, B) for _ in range(K)]


@pytest.mark.parametrize("K", [1, 2, 17, 300])
@pytest.mark.parametrize("M", [1, 3, 5])
@pytest.mark.parametrize("B", [1, 3])
def test_ckks_matrix(K, M, B):
    """CKKS over K (300 crosses two window reductions), M (output tiles of 2: ragged at 3 and 5) and B, against the chain; the
    Python-integer restatement where it is cheap"""
    n, L = 1024, 2
    mods, _, ctx = context(sb().CKKS, n, [50, 40, 60])
    rng = np.random.default_rng(100 * K + 10 * M + B)
    lhs, rhs = inputs(rng, mods, n, L, B, K, M)
    got = fused_both(ctx, lhs, rhs)
    want = chain(ctx, lhs, rhs)
    for j in range(M):
        assert_words(got[j], want[j], f"K={K} M={M} B={B} output {j} vs chain")
    if K * M * B <= 51:
        ref = restate(mods, lhs, rhs)
        for j in range(M):
            assert_words(got[j], ref[j], f"K={K} M={M} B={B} output {j} vs Python integers")


def test_bgv_sub_and_scaled_steps():
    """BGV: scaled steps (random balancing factors, any 64-bit words) and subtracting steps"""
    n = 4096
    mods, t, ctx = context(sb().BGV, n, [50, 40, 60])
    rng = np.random.default_rng(3000)
    K, M, L, B = 6, 3, 2, 2
    lhs, rhs = inputs(rng, mods, n, L, B, K, M)
    modes = [2, 0, 3, 1, 2]
    factors = [[int(v) for v in rng.integers(0, 2**64, 2, dtype=np.uint64)] for _ in range(K - 1)]
    factors[4] = [t - 1, 1]
    got = fused_both(ctx, lhs, rhs, modes, factors)
    want = chain(ctx, lhs, rhs, modes, factors)
    ref = restate(mods, lhs, rhs, modes, factors)
    for j in range(M):
        assert_words(got[j], want[j], f"BGV output {j} vs chain")
        assert_words(got[j], ref[j], f"BGV output {j} vs Python integers")


def test_bfv_chunks_of_terms():
    """BFV: the products go through scratch in chunks of terms; with a 1 MiB scratch budget K = 10 terms take 4 chunks, and the
    result does not depend on the budget (scaled and subtracting steps too)"""
    n = 4096
    mods, t, ctx = context(sb().BFV, n, [50, 40, 60, 50])
    rng = np.random.default_rng(4000)
    K, M, L, B = 10, 2, 3, 1
    lhs, rhs = inputs(rng, mods, n, L, B, K, M)
    modes = [0, 1, 2, 3, 0, 0, 1, 2, 0]
    factors = [[int(v) for v in rng.integers(1, t, 2)] for _ in range(K - 1)]
    whole = fused_both(ctx, lhs, rhs, modes, factors)
    per_term = B * 3 * L * n * 8
    assert (1 << 20) // per_term == 3  # 3 terms per chunk: 3, 3, 3, 1
    ctx.set_limit(ctx.LIMIT_SCRATCH_BYTES, 1 << 20)
    cut = fused_both(ctx, lhs, rhs, modes, factors)
    want = chain(ctx, lhs, rhs, modes, factors)
    for j in range(M):
        assert_words(cut[j], want[j], f"BFV chunked output {j} vs chain")
        assert_words(whole[j], want[j], f"BFV one chunk output {j} vs chain")


@pytest.mark.parametrize("scheme", ["CKKS", "BFV"])
def test_squares(scheme):
    """lhs is rhs: sum_i x_i^2, against sb200_square's words"""
    S = sb()
    n = 4096
    mods, t, ctx = context(getattr(S, scheme), n, [50, 40, 60])
    rng = np.random.default_rng(5000)
    K, L, B = 5, 2, 2
    rhs = [rand_ct(rng, mods, n, 2, L, B) for _ in range(K)]
    got = fused_both(ctx, list(rhs), rhs)
    want = ctx.add_many([ctx.square(x) for x in rhs])
    assert_words(got[0], want, f"{scheme} squares vs square + add_many")
    assert_words(got[0], chain(ctx, list(rhs), rhs)[0], f"{scheme} squares vs chain")


@pytest.mark.parametrize("bits,window", [(60, WINDOW), (61, WINDOW_61)])
@pytest.mark.parametrize("extra", [0, 1])
@pytest.mark.parametrize("word", ["q-1", "unreduced"])
def test_word_bounds(bits, window, extra, word):
    """all-(q - 1) words (the window's worst case) and unreduced words up to 2^64 - 1 at 60- and 61-bit primes, with K = window
    and window + 1, against the chain and the Python-integer restatement"""
    n = 1024
    mods = [int(q) for q in O.get_primes(2 * n, bits, 2)]
    ctx = sb().Context(sb().CKKS, n, mods, 0)
    rng = np.random.default_rng(6000 + bits + extra)
    K, M, L, B = window + extra, 2, 2, 1
    if word == "q-1":
        one = np.stack([np.stack([np.stack([np.full(n, mods[li] - 1, dtype=np.uint64) for li in range(L)])] * 2)])
        lhs, rhs = [one.copy() for _ in range(M * K)], [one.copy() for _ in range(K)]
    else:
        lhs = [rng.integers(0, 2**64, (B, 2, L, n), dtype=np.uint64) for _ in range(M * K)]
        rhs = [rng.integers(0, 2**64, (B, 2, L, n), dtype=np.uint64) for _ in range(K)]
        for c in lhs + rhs:
            c[0, :, :, :2] = [2**64 - 1, 0]
    got = fused_both(ctx, lhs, rhs)
    want = chain(ctx, lhs, rhs)
    ref = restate(mods, lhs, rhs)
    for j in range(M):
        assert_words(got[j], want[j], f"{bits}-bit {word} K={K} output {j} vs chain")
        assert_words(got[j], ref[j], f"{bits}-bit {word} K={K} output {j} vs Python integers")


@pytest.mark.parametrize("n,L,K,M", [(65536, 31, 3, 2), (4096, 60, 3, 2)])
def test_deep_levels(n, L, K, M):
    """n = 65536 with L = 31 (of 32 primes), and a 60-prime level at n = 4096"""
    bits = [50] * 32 if n == 65536 else [30] * 60
    mods, _, ctx = context(sb().CKKS, n, bits)
    rng = np.random.default_rng(n + L)
    lhs, rhs = inputs(rng, mods, n, L, 1, K, M)
    got = fused_both(ctx, lhs, rhs)
    want = chain(ctx, lhs, rhs)
    for j in range(M):
        assert_words(got[j], want[j], f"n={n} L={L} output {j}")


def test_host_staging_chunks():
    """the host entry point cut into several staging chunks with a ragged last one, equal to the stream form"""
    import torch

    n = 4096
    mods, _, ctx = context(sb().CKKS, n, [50, 40, 60])
    rng = np.random.default_rng(7000)
    K, M, L, B = 3, 2, 2, 7
    lhs, rhs = inputs(rng, mods, n, L, B, K, M)
    d_outs = [dev(np.zeros((B, 3, L, n), dtype=np.uint64)) for _ in range(M)]
    ctx.d_multiply_sum([dev(a) for a in lhs], [dev(a) for a in rhs], d_outs, L, B)
    torch.cuda.synchronize()
    per_ct = ((M * K + K) * 2 + M * 3) * L * n * 8
    ctx.set_limit(ctx.LIMIT_HOST_STAGE_BYTES, 2 * per_ct)  # chunks of 2, 2, 2, 1 members
    cut = ctx.multiply_sum(lhs, rhs)
    for j in range(M):
        assert_words(cut[j], host(d_outs[j]), f"chunked host form vs stream form, output {j}")


def test_errors_leave_outputs_unchanged():
    """every error of the entry points, raised before the first launch: the outputs and the operands keep their words"""
    import torch

    S = sb()
    n = 4096
    mods, _, ctx = context(S.CKKS, n, [50, 40, 60])
    rng = np.random.default_rng(8000)
    L, B, K, M = 2, 3, 2, 2
    lhs, rhs = inputs(rng, mods, n, L, B, K, M)
    d_lhs, d_rhs = [dev(c) for c in lhs], [dev(c) for c in rhs]
    sentinel = rng.integers(0, 2**64, (B, 3, L, n), dtype=np.uint64)
    d_outs = [dev(sentinel) for _ in range(M)]
    pool = dev(np.zeros((B, 6, L, n), dtype=np.uint64))  # room for a right operand and an output slab overlapping it, and nothing else

    def call(lhs_=None, rhs_=None, outs_=None, modes=None, factors=None, batch=B):
        ctx.d_multiply_sum(d_lhs if lhs_ is None else lhs_, d_rhs if rhs_ is None else rhs_, d_outs if outs_ is None else outs_, L, batch,
                           modes, factors)

    cases = [
        (ValueError, "encrypteds cannot be empty", dict(lhs_=[], rhs_=[])),
        (ValueError, "outputs cannot be empty", dict(lhs_=[], outs_=[])),
        (ValueError, "invalid add_many mode", dict(modes=[4])),
        (ValueError, "invalid add_many mode", dict(modes=[-1])),
        (ValueError, "null pointer: h_factors", dict(modes=[2])),
        (ValueError, "must not overlap a left-hand operand", dict(outs_=[d_outs[0], d_lhs[3]])),
        (ValueError, "must not overlap a left-hand operand", dict(outs_=[d_outs[0], d_lhs[1].data_ptr() + 8 * L * n])),
        (ValueError, "must not overlap a right-hand operand", dict(rhs_=[d_rhs[0], pool], outs_=[d_outs[0], pool])),
        (ValueError, "must not overlap a right-hand operand", dict(rhs_=[pool, d_rhs[1]], outs_=[pool.data_ptr() + 8 * L * n, d_outs[1]])),
        (ValueError, "output slabs must not overlap", dict(outs_=[d_outs[0], d_outs[0]])),
        (ValueError, "output slabs must not overlap", dict(outs_=[d_outs[0], d_outs[0].data_ptr() + 8 * n])),
        (ValueError, "batch must be positive", dict(batch=0)),
        (ValueError, "null pointer", dict(rhs_=[d_rhs[0], 0])),
        (ValueError, "null pointer", dict(lhs_=[d_lhs[0], 0, d_lhs[2], d_lhs[3]])),
        (ValueError, "null pointer", dict(outs_=[d_outs[0], 0])),
    ]
    for exc, msg, kw in cases:
        with pytest.raises(exc) as e:
            call(**kw)
        assert msg in str(e.value), (msg, str(e.value))
        torch.cuda.synchronize()
        for j in range(M):
            assert_words(host(d_outs[j]), sentinel, f"output {j} unchanged after '{msg}'")
        for i in range(K):
            assert_words(host(d_rhs[i]), rhs[i], f"right operand {i} unchanged after '{msg}'")
        for x in range(M * K):
            assert_words(host(d_lhs[x]), lhs[x], f"left operand {x} unchanged after '{msg}'")
    # the host form refuses the same overlaps: here output 0 on left-hand operand 1 (SB200_E_INVALID_ARG, nothing written)
    import ctypes as C

    lib = S.lib()
    h_lhs, h_rhs = [np.ascontiguousarray(a) for a in lhs], [np.ascontiguousarray(a) for a in rhs]
    big = rng.integers(0, 2**64, (B, 3, L, n), dtype=np.uint64)  # left-hand operand 1 with room for the output's three polynomials
    before = big.copy()
    h_outs = [big, np.zeros((B, 3, L, n), dtype=np.uint64)]
    p_lhs = (C.c_void_p * (M * K))(*[big.ctypes.data if x == 1 else h_lhs[x].ctypes.data for x in range(M * K)])
    p_rhs = (C.c_void_p * K)(*[a.ctypes.data for a in h_rhs])
    p_outs = (C.c_void_p * M)(*[o.ctypes.data for o in h_outs])
    assert lib.sb200_multiply_sum_host(ctx.h, L, B, K, M, p_lhs, p_rhs, None, None, p_outs) == -1
    assert b"multiply_sum: an output slab must not overlap a left-hand operand [1]" in lib.sb200_last_error()
    assert_words(big, before, "host output after a rejected call")
    assert_words(h_outs[1], np.zeros_like(h_outs[1]), "second host output after a rejected call")
    # BFV: a level above sb200_multiply's limit, raised before add_many's mode check (the chain's order)
    n_b, L_b = 4096, 65
    mods_b = [int(q) for q in O.get_primes(2 * n_b, 30, 66)]
    ctx_b = S.Context(S.BFV, n_b, mods_b, 65537)
    a = dev(np.zeros((1, 2, L_b, n_b), dtype=np.uint64))
    o = dev(rng.integers(0, 2**64, (1, 3, L_b, n_b), dtype=np.uint64))
    before = host(o)
    with pytest.raises(ValueError, match="at most 64 primes"):
        ctx_b.d_multiply_sum([a, a], [a, a], [o], L_b, 1, [9])
    torch.cuda.synchronize()
    assert_words(host(o), before, "output unchanged after the BFV level limit")
    with pytest.raises(ValueError, match="invalid add_many mode"):
        ctx.multiply_sum(lhs, rhs, [7])


@pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsealref.so not present")
def test_against_reference_chain():
    """every member against the reference's own multiply + add chain (CKKS at a small n)"""
    n, bits, L, B, K, M = 4096, [50, 40, 40, 60], 3, 2, 4, 2
    mods = R.coeff_modulus_create(n, bits)
    ctx = sb().Context(sb().CKKS, n, mods)
    rc = R.RefContext(R.CKKS, n, mods, 0)
    rng = np.random.default_rng(9000)
    lhs, rhs = inputs(rng, mods, n, L, B, K, M)
    got = ctx.multiply_sum(lhs, rhs)
    for j in range(M):
        for b in range(B):
            want = rc.multiply(L, lhs[j * K][b], rhs[0][b])
            for i in range(1, K):
                want = rc.linear(0, L, want, rc.multiply(L, lhs[j * K + i][b], rhs[i][b]))
            assert_words(got[j][b], want, f"output {j} member {b} vs reference")


def test_cpp_multiply_sum_against_seal_evaluator():
    """tests/cpp/shim_multsum_test.cpp: Evaluator::multiply_sum and multiply_relinearize_sum against seal::Evaluator's multiply +
    add_many + relinearize chain -- words, scale, correction factor, size, parms_id, exception types and messages"""
    exe = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref", "bin", "shim_multsum_test")
    if not os.path.exists(exe):
        pytest.skip("shim_multsum_test not built (reference sources absent at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert "shim_multsum_test ok" in r.stdout
