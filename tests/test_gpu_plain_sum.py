"""Sums of plaintext products (sb200_multiply_plain_sum / _host): output j = add_many over i of multiply_plain(ct_i, plain_{j K + i}),
word for word against the chained device calls (multiply_plain_n / multiply_plain_coeff_n, then add_many, both pinned to the
reference by tests/test_gpu_plain_batch.py and tests/test_gpu_compositions.py) and against a Python-integer restatement."""
import numpy as np
import pytest

import oracle as O
from common import assert_words, rand_ct

pytestmark = pytest.mark.gpu

WINDOW = 256  # kPlainSumWindow (seal_b200/csrc/sb_engine.cuh)


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


def make_inputs(rng, mods, n, L, B, K, M, sizes, counts, ct_ntt, plain_ntt, t):
    cts = [rand_ct(rng, mods, n, sizes[i], L, B) for i in range(K)]
    plains = []
    for x in range(M * K):
        c = counts[x]
        if plain_ntt:
            plains.append(rand_ct(rng, mods, n, 1, L, c)[:, 0])
        else:
            p = rng.integers(0, t, (c, n), dtype=np.uint64)
            p[:, :4] = [0, t - 1, (t + 1) // 2, (t + 1) // 2 - 1]  # the lift edges
            plains.append(p)
    return cts, plains


def chain(ctx, cts, plains, K, M, ct_ntt, plain_ntt, modes=None, factors=None):
    """the chained device calls: multiply_plain of every term, then one add_many per output"""
    outs = []
    for j in range(M):
        terms = []
        for i in range(K):
            a, p = cts[i], plains[j * K + i]
            p = p[0] if p.shape[0] == 1 else p
            if not plain_ntt:
                terms.append(ctx.multiply_plain_coeff_n(a, p, ct_ntt))
            elif ct_ntt:
                terms.append(ctx.multiply_plain_n(a, p))
            else:  # BFV coefficient form x NTT-form plaintext: to NTT form, multiply, back (evaluator.cpp:2006-2011)
                terms.append(ctx.transform_from_ntt(ctx.multiply_plain_n(ctx.transform_to_ntt(a), p)))
        outs.append(ctx.add_many(terms, modes, factors))
    return outs


def restate(mods, cts, plains, K, M, modes=None, factors=None):
    """Python integers: sum_i c_i (x_i mod q) (p mod q) mod q with c_i the fold's per-term constant (NTT-form operands)"""
    L = cts[0].shape[2]
    B = cts[0].shape[0]
    out_size = max(c.shape[1] for c in cts)
    outs = []
    for j in range(M):
        o = np.zeros((B, out_size, L, cts[0].shape[3]), dtype=np.uint64)
        for li in range(L):
            q = int(mods[li])
            consts, tail = [0] * K, 1
            for i in range(K - 1, -1, -1):
                m = modes[i - 1] if (i and modes is not None) else 0
                v = (int(factors[i - 1][1]) % q if m & 2 else 1) * tail % q
                consts[i] = (q - v) % q if m & 1 else v
                if m & 2:
                    tail = tail * (int(factors[i - 1][0]) % q) % q
            for b in range(B):
                for s in range(out_size):
                    acc = np.zeros(cts[0].shape[3], dtype=object)
                    for i in range(K):
                        if s >= cts[i].shape[1]:
                            continue
                        p = plains[j * K + i]
                        pw = p[0 if p.shape[0] == 1 else b][li].astype(object) % q
                        acc = acc + consts[i] * (cts[i][b, s, li].astype(object) % q) * pw
                    o[b, s, li] = (acc % q).astype(np.uint64)
        outs.append(o)
    return outs


def fused_both(ctx, cts, plains, K, M, ct_ntt, plain_ntt, modes=None, factors=None):
    """the host entry point, and the stream entry point on device tensors (inputs checked unchanged); returns the host result"""
    got = ctx.multiply_plain_sum(cts, plains, modes, factors, ct_ntt, plain_ntt)
    B, _, L, n = cts[0].shape
    sizes = [c.shape[1] for c in cts]
    d_cts, d_plains = [dev(c) for c in cts], [dev(p) for p in plains]
    d_outs = [dev(np.zeros((B, max(sizes), L, n), dtype=np.uint64)) for _ in range(M)]
    ctx.d_multiply_plain_sum(d_cts, d_plains, d_outs, L, B, sizes, [p.shape[0] for p in plains], ct_ntt, plain_ntt, modes, factors)
    import torch

    torch.cuda.synchronize()
    for j in range(M):
        assert_words(host(d_outs[j]), got[j], f"stream vs host entry point, output {j}")
    for i in range(K):
        assert_words(host(d_cts[i]), cts[i], "ciphertext operand unchanged")
    return got


BFV_FORMS = [(True, True), (False, True), (True, False), (False, False)]  # (ct_is_ntt, plain_is_ntt)


@pytest.mark.parametrize("K,M,B", [(1, 1, 1), (2, 2, 3), (WINDOW - 1, 1, 1), (WINDOW, 2, 1), (WINDOW + 1, 1, 3), (130, 5, 1), (3, 33, 3)])
def test_ckks_ntt_matrix(K, M, B):
    """CKKS NTT x NTT over the shapes of the term and output tiles: K around the reduction window, ragged output tiles, M = 33,
    mixed sizes 2 and 3, shared and per-member plaintexts"""
    n = 4096
    mods, _, ctx = context(sb().CKKS, n, [50, 40, 60])
    rng = np.random.default_rng(1000 + K * 7 + M)
    L = 2
    sizes = [2 + (i % 2) for i in range(K)]
    counts = [1 if (x % 3 == 1) else B for x in range(M * K)]
    cts, plains = make_inputs(rng, mods, n, L, B, K, M, sizes, counts, True, True, 0)
    got = fused_both(ctx, cts, plains, K, M, True, True)
    want = chain(ctx, cts, plains, K, M, True, True)
    for j in range(M):
        assert_words(got[j], want[j], f"K={K} M={M} B={B} output {j}")


@pytest.mark.parametrize("ct_ntt,plain_ntt", BFV_FORMS)
@pytest.mark.parametrize("B", [1, 3])
def test_bfv_forms(ct_ntt, plain_ntt, B):
    """BFV: all four NTT-form combinations of multiply_plain, shared and per-member plaintexts, sizes 2 and 3"""
    n = 4096
    mods, t, ctx = context(sb().BFV, n, [50, 40, 60, 50])
    rng = np.random.default_rng(2000 + 10 * ct_ntt + plain_ntt + B)
    K, M, L = 5, 3, 3
    sizes = [2, 3, 2, 2, 3]
    counts = [1 if x % 2 else B for x in range(M * K)]
    cts, plains = make_inputs(rng, mods, n, L, B, K, M, sizes, counts, ct_ntt, plain_ntt, t)
    got = fused_both(ctx, cts, plains, K, M, ct_ntt, plain_ntt)
    want = chain(ctx, cts, plains, K, M, ct_ntt, plain_ntt)
    for j in range(M):
        assert_words(got[j], want[j], f"BFV forms ct_ntt={ct_ntt} plain_ntt={plain_ntt} B={B} output {j}")


@pytest.mark.parametrize("plain_ntt", [True, False])
def test_bgv_balancing(plain_ntt):
    """BGV: NTT-form ciphertexts with NTT- and coefficient-form plaintexts, terms whose correction factors differ (scaled add
    steps with random factors) and subtracting steps"""
    n = 4096
    mods, t, ctx = context(sb().BGV, n, [50, 40, 60])
    rng = np.random.default_rng(3000 + plain_ntt)
    K, M, L, B = 6, 2, 2, 3
    sizes = [2, 3, 2, 3, 2, 2]
    counts = [B if x % 2 else 1 for x in range(M * K)]
    cts, plains = make_inputs(rng, mods, n, L, B, K, M, sizes, counts, True, plain_ntt, t)
    modes = [2, 0, 3, 1, 2]
    factors = [[int(v) for v in rng.integers(1, t, 2)] for _ in range(K - 1)]
    factors[4] = [t - 1, 1]
    got = fused_both(ctx, cts, plains, K, M, True, plain_ntt, modes, factors)
    want = chain(ctx, cts, plains, K, M, True, plain_ntt, modes, factors)
    for j in range(M):
        assert_words(got[j], want[j], f"BGV plain_ntt={plain_ntt} output {j}")


@pytest.mark.parametrize("word", ["q-1", "unreduced"])
@pytest.mark.parametrize("K", [WINDOW, WINDOW + 1])
def test_word_bounds_60_bit(word, K):
    """all-(q - 1) words (the window's worst case) and unreduced words up to 2^64 - 1 at 60-bit primes, against the chain and
    the Python-integer restatement"""
    n = 1024
    mods, _, ctx = context(sb().CKKS, n, [60, 60, 60])
    rng = np.random.default_rng(4000 + K)
    L, B, M = 2, 1, 2
    sizes = [2] * K
    if word == "q-1":
        cts = [np.stack([np.stack([np.full((L, n), 0, dtype=np.uint64)] * 2)]) for _ in range(K)]
        for c in cts:
            for li in range(L):
                c[:, :, li, :] = mods[li] - 1
        plains = [np.stack([np.stack([np.full(n, mods[li] - 1, dtype=np.uint64) for li in range(L)])]) for _ in range(M * K)]
    else:
        cts = [rng.integers(0, 2**64, (B, 2, L, n), dtype=np.uint64) for _ in range(K)]
        for c in cts:
            c[0, 0, 0, :2] = [2**64 - 1, 0]
        plains = [rng.integers(0, 2**64, (1, L, n), dtype=np.uint64) for _ in range(M * K)]
    got = fused_both(ctx, cts, plains, K, M, True, True)
    want = chain(ctx, cts, plains, K, M, True, True)
    ref = restate(mods, cts, plains, K, M)
    for j in range(M):
        assert_words(got[j], want[j], f"{word} K={K} output {j} vs chain")
        assert_words(got[j], ref[j], f"{word} K={K} output {j} vs Python integers")


def test_window_at_61_bit_primes():
    """a level with primes of 61 bits takes a shorter reduction window (64 terms): all-(q - 1) words over K = 130 terms"""
    n = 1024
    mods = [int(q) for q in O.get_primes(2 * n, 61, 2)]
    ctx = sb().Context(sb().CKKS, n, mods, 0)
    K, M, L = 130, 1, 2
    cts = [np.stack([np.stack([np.stack([np.full(n, mods[li] - 1, dtype=np.uint64) for li in range(L)])] * 2)]) for _ in range(K)]
    plains = [np.stack([np.stack([np.full(n, mods[li] - 1, dtype=np.uint64) for li in range(L)])]) for _ in range(M * K)]
    got = fused_both(ctx, cts, plains, K, M, True, True)
    assert_words(got[0], chain(ctx, cts, plains, K, M, True, True)[0], "61-bit primes vs chain")
    assert_words(got[0], restate(mods, cts, plains, K, M)[0], "61-bit primes vs Python integers")


def test_cpp_multiply_plain_sum_against_seal_evaluator():
    """tests/cpp/shim_plainsum_test.cpp: Evaluator::multiply_plain_sum against seal::Evaluator's multiply_plain + add_many chain --
    words, scale, correction factor, exception types and messages; CKKS with a baby-step/giant-step case, BFV in all four forms,
    BGV with differing correction factors"""
    import os
    import subprocess

    exe = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref", "bin", "shim_plainsum_test")
    if not os.path.exists(exe):
        pytest.skip("shim_plainsum_test not built (reference sources absent at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert "shim_plainsum_test ok" in r.stdout


def test_restatement_scaled_small_n():
    """Python-integer restatement of the folded constants: scaled and subtracting steps, mixed sizes, unreduced words"""
    n = 1024
    mods, _, ctx = context(sb().CKKS, n, [60, 50])
    rng = np.random.default_rng(5)
    K, M, L, B = 4, 3, 2, 3
    cts = [rng.integers(0, 2**64, (B, 2 + i % 2, L, n), dtype=np.uint64) for i in range(K)]
    plains = [rng.integers(0, 2**64, (B if x % 2 else 1, L, n), dtype=np.uint64) for x in range(M * K)]
    modes = [3, 1, 2]
    factors = [[int(v) for v in rng.integers(0, 2**64, 2, dtype=np.uint64)] for _ in range(K - 1)]
    got = fused_both(ctx, cts, plains, K, M, True, True, modes, factors)
    ref = restate(mods, cts, plains, K, M, modes, factors)
    want = chain(ctx, cts, plains, K, M, True, True, modes, factors)
    for j in range(M):
        assert_words(got[j], ref[j], f"output {j} vs Python integers")
        assert_words(got[j], want[j], f"output {j} vs chain")


@pytest.mark.parametrize("n,L,K,M", [(4096, 60, 3, 2), (8192, 60, 2, 1), (8192, 20, 4, 3), (65536, 32, 2, 1)])
def test_deep_levels(n, L, K, M):
    """n = 4096 and 8192 with up to 60 primes, and the n = 65536, 32-prime level (BFV coefficient-form operands at n = 8192)"""
    scheme = sb().BFV if (n, L) == (8192, 20) else sb().CKKS
    bits = [60] * L if n >= 8192 else [30] * L
    mods, t, ctx = context(scheme, n, bits)
    rng = np.random.default_rng(n + L)
    B = 1
    sizes = [2] * K
    forms = (False, False) if scheme == sb().BFV else (True, True)
    counts = [1] * (M * K)
    cts, plains = make_inputs(rng, mods, n, L, B, K, M, sizes, counts, *forms, t)
    got = fused_both(ctx, cts, plains, K, M, *forms)
    want = chain(ctx, cts, plains, K, M, *forms)
    for j in range(M):
        assert_words(got[j], want[j], f"n={n} L={L} output {j}")


@pytest.mark.parametrize("forms", [(True, True), (False, False)])
def test_host_staging_chunks(forms):
    """the host entry point cut into several staging chunks (a ragged last one), shared plaintexts uploaded once, equal word for
    word to the stream form"""
    import torch

    n = 4096
    mods, t, ctx = context(sb().BFV, n, [50, 40, 60])
    rng = np.random.default_rng(6000 + forms[0])
    K, M, L, B = 3, 2, 2, 7
    sizes = [2, 3, 2]
    counts = [1 if x % 2 else B for x in range(M * K)]
    cts, plains = make_inputs(rng, mods, n, L, B, K, M, sizes, counts, *forms, t)
    whole = ctx.multiply_plain_sum(cts, plains, None, None, *forms)
    pw = L * n if forms[1] else n
    per_ct = (sum(sizes) * L * n + sum(pw for c in counts if c != 1) + M * 3 * L * n) * 8
    ctx.set_limit(ctx.LIMIT_HOST_STAGE_BYTES, 2 * per_ct)  # chunks of 2, 2, 2, 1 members
    cut = ctx.multiply_plain_sum(cts, plains, None, None, *forms)
    want = chain(ctx, cts, plains, K, M, *forms)
    d_outs = [dev(np.zeros_like(w)) for w in whole]
    ctx.d_multiply_plain_sum([dev(c) for c in cts], [dev(p) for p in plains], d_outs, L, B, sizes, counts, *forms)
    torch.cuda.synchronize()
    for j in range(M):
        assert_words(cut[j], whole[j], f"chunked vs default staging, output {j}")
        assert_words(cut[j], want[j], f"chunked vs chain, output {j}")
        assert_words(cut[j], host(d_outs[j]), f"chunked host form vs stream form, output {j}")


def test_errors_leave_outputs_unchanged():
    """every error of the entry points, raised before the first launch: the outputs and the operands keep their words"""
    import torch

    S = sb()
    n = 4096
    mods, _, ctx = context(S.CKKS, n, [50, 40, 60])
    rng = np.random.default_rng(7)
    L, B, K, M = 2, 3, 2, 2
    cts, plains = make_inputs(rng, mods, n, L, B, K, M, [2, 2], [B] * (M * K), True, True, 0)
    d_cts, d_plains = [dev(c) for c in cts], [dev(p) for p in plains]
    sentinel = rng.integers(0, 2**64, (B, 2, L, n), dtype=np.uint64)
    d_outs = [dev(sentinel) for _ in range(M)]

    def call(cts_=None, plains_=None, outs_=None, sizes=None, counts=None, plain_ntt=True, modes=None, factors=None, batch=B):
        ctx.d_multiply_plain_sum(d_cts if cts_ is None else cts_, d_plains if plains_ is None else plains_, d_outs if outs_ is None else outs_,
                                 L, batch, [2] * K if sizes is None else sizes, [B] * (M * K) if counts is None else counts, True, plain_ntt,
                                 modes, factors)

    cases = [
        (ValueError, "encrypteds cannot be empty", dict(cts_=[], plains_=[], sizes=[], counts=[])),
        (ValueError, "outputs cannot be empty", dict(plains_=[], counts=[], outs_=[])),
        (ValueError, "plain_count must be 1 or batch", dict(counts=[B, 2, B, B])),
        (ValueError, "invalid ciphertext size", dict(sizes=[2, 17])),
        (ValueError, "invalid add_many mode", dict(modes=[4])),
        (ValueError, "null pointer: h_factors", dict(modes=[2])),
        (ValueError, "must not overlap a ciphertext operand", dict(outs_=[d_outs[0], d_cts[1]])),
        (ValueError, "must not overlap a ciphertext operand", dict(outs_=[d_outs[0], d_cts[1].data_ptr() + 8 * L * n])),
        (ValueError, "must not overlap a plaintext operand", dict(outs_=[d_plains[3], d_outs[1]])),
        (ValueError, "must not overlap a plaintext operand", dict(outs_=[d_plains[3].data_ptr() - 8 * n, d_outs[1]])),
        (ValueError, "output slabs must not overlap", dict(outs_=[d_outs[0], d_outs[0]])),
        (ValueError, "output slabs must not overlap", dict(outs_=[d_outs[0], d_outs[0].data_ptr() + 8 * n])),
        (ValueError, "plain_count must be 1 or batch", dict(counts=[B, 2, B, B], sizes=[2, 17])),
        (ValueError, "unsupported operation for scheme type", dict(plain_ntt=False)),
        (ValueError, "batch must be positive", dict(batch=0)),
    ]
    for exc, msg, kw in cases:
        with pytest.raises(exc) as e:
            call(**kw)
        assert msg in str(e.value), (msg, str(e.value))
        torch.cuda.synchronize()
        for j in range(M):
            assert_words(host(d_outs[j]), sentinel, f"output {j} unchanged after '{msg}'")
        for i in range(K):
            assert_words(host(d_cts[i]), cts[i], f"ciphertext {i} unchanged after '{msg}'")
    # a NULL operand (SB200_E_POINTER) and the host entry point's checks
    with pytest.raises(ValueError, match="null pointer"):
        call(cts_=[d_cts[0], 0])
    with pytest.raises(ValueError, match="plain_count must be 1 or batch"):
        ctx.multiply_plain_sum(cts, [p[:2] for p in plains])
