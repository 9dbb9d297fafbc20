"""Batch compositions: sb200_add_many (a left fold of add / sub steps over operands of any sizes, with optional BGV balancing
scalars, in one pass) through the Python binding, word for word against a Python-integer restatement of the reference's chain of
add_inplace / sub_inplace calls, against chained sb200_add / sb200_sub calls and against the reference (oracle/_ref/libsealref.so);
and the C++ members built on it and on the product scheduler (tests/cpp/shim_compose_test.cpp) against seal::Evaluator."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import refseal as R
from common import assert_words

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsealref.so not present")


def sb():
    import seal_b200

    return seal_b200


def batching_prime(n, bits):
    """the largest prime below 2^bits that is 1 mod 2n (an NTT-friendly plain modulus)"""
    p = ((1 << bits) - 1) // (2 * n) * (2 * n) + 1
    while any(p % d == 0 for d in range(3, int(p ** 0.5) + 1, 2)):
        p -= 2 * n
    return p


def context(n, bits, scheme=None):
    mods = sb().coeff_modulus_create(n, bits)
    S = sb()
    return mods, S.Context(S.CKKS if scheme is None else scheme, n, mods)


def rand_ops(rng, mods, n, L, B, sizes):
    return [np.stack([np.stack([np.stack([rng.integers(0, mods[i], n, dtype=np.uint64) for i in range(L)]) for _ in range(s)])
                      for _ in range(B)]) for s in sizes]


def shoup_mul(x, e, q):
    """multiply_uint_mod(x, MultiplyUIntModOperand{e}) of the reference, for any 64-bit words x (Python integers)"""
    w = (e << 64) // q
    xs = x.astype(object)
    hi = (xs * w) >> 64
    r = (xs * e - hi * q) % (1 << 64)
    return np.array([v - q if v >= q else v for v in r.ravel()], dtype=object).reshape(x.shape).astype(np.uint64)


def restate(ops, mods, modes=None, factors=None):
    """the reference's chain acc = ops[0]; acc.add_inplace / sub_inplace(ops[j]) restated on the words: absent polynomials are
    copied (add) or negated (sub), scaled steps multiply the accumulator's present polynomials and the operand first"""
    B, _, L, n = ops[0].shape
    q = np.array(mods[:L], dtype=np.uint64)[None, :, None]
    acc = [ops[0][:, p].copy() for p in range(ops[0].shape[1])]
    with np.errstate(over="ignore"):
        for j in range(1, len(ops)):
            m = 0 if modes is None else modes[j - 1]
            y = [ops[j][:, p].copy() for p in range(ops[j].shape[1])]
            if m & 2:
                e1, e2 = (int(v) for v in factors[j - 1])
                sc = lambda xs, e: np.stack([shoup_mul(xs[:, i], e % mods[i], mods[i]) for i in range(L)], axis=1)
                acc = [sc(a, e1) for a in acc]
                y = [sc(v, e2) for v in y]
            for p, v in enumerate(y):
                if p < len(acc):
                    if m & 1:  # sub_poly_coeffmod's borrow form: the 64-bit difference, plus q when it borrowed
                        acc[p] = np.where(acc[p] < v, acc[p] - v + q, acc[p] - v)
                    else:
                        s = acc[p] + v
                        acc[p] = np.where(s >= q, s - q, s)
                else:
                    acc.append(np.where(v != 0, q - v, np.uint64(0)) if m & 1 else v)
    return np.stack(acc, axis=1)


@pytest.mark.parametrize("m", [1, 2, 3, 17])
def test_add_many_vs_restatement(m):
    n, bits, L, B = 4096, [50, 40, 40, 60], 3, 3
    mods, ctx = context(n, bits)
    rng = np.random.default_rng(100 + m)
    sizes = [int(rng.integers(2, 5)) for _ in range(m)]
    modes = [int(rng.integers(0, 2)) for _ in range(m - 1)]
    ops = rand_ops(rng, mods, n, L, B, sizes)
    want = restate(ops, mods, modes)
    assert_words(ctx.add_many(ops, modes), want, f"add_many host m={m}")
    d = [_dev(o) for o in ops]
    out = _dev(np.zeros_like(want))
    ctx.profile(True)
    ctx.d_add_many(d, out, L, B, sizes, modes)
    import torch

    torch.cuda.synchronize()
    launches = {k: v for k, _, v, _ in ctx.profile_read()}
    ctx.profile(False)
    # one launch takes 16 operands; a longer fold continues from the partial result, 15 more operands per launch
    assert launches.get("add_many") == (1 if m <= 16 else 1 + -(-(m - 16) // 15)), launches
    assert_words(_host(out), want, f"add_many device m={m}")


@pytest.mark.parametrize("order", [[2, 3, 4], [4, 3, 2], [2, 4], [3, 2, 4, 2]])
def test_mixed_sizes_and_sub_tails(order):
    """sizes in both orders; a longer subtrahend's tail is negated"""
    n, bits, L, B = 4096, [50, 40, 60], 2, 2
    mods, ctx = context(n, bits)
    rng = np.random.default_rng(len(order) * 7 + order[0])
    ops = rand_ops(rng, mods, n, L, B, order)
    for modes in ([0] * (len(order) - 1), [1] * (len(order) - 1)):
        assert_words(ctx.add_many(ops, modes), restate(ops, mods, modes), f"sizes {order} modes {modes}")


def test_bgv_scaled_steps():
    """BGV balancing: distinct factor pairs per step, with and without size changes"""
    S = sb()
    n, bits, L, B = 4096, [50, 40, 60], 2, 2
    mods = sb().coeff_modulus_create(n, bits)
    t = batching_prime(n, 20)
    ctx = S.Context(S.BGV, n, mods, t)
    rng = np.random.default_rng(5)
    sizes = [2, 3, 2, 4, 2]
    ops = rand_ops(rng, mods, n, L, B, sizes)
    modes = [S.FOLD_SCALED, S.FOLD_SUB | S.FOLD_SCALED, S.FOLD_ADD, S.FOLD_SUB | S.FOLD_SCALED]
    factors = [[int(rng.integers(1, t)), int(rng.integers(1, t))] for _ in range(4)]
    factors[2] = [0, 0]
    assert_words(ctx.add_many(ops, modes, factors), restate(ops, mods, modes, factors), "BGV scaled steps")


@pytest.mark.parametrize("word", ["q-1", "2^64-1"])
def test_bound_words_equal_chained_add_sub(word):
    """every input word at q - 1 or at 2^64 - 1: the fold equals chained sb200_add / sb200_sub calls word for word"""
    n, bits, L, B, size = 4096, [50, 40, 60], 2, 2, 2
    mods, ctx = context(n, bits)
    full = np.empty((B, size, L, n), dtype=np.uint64)
    for i in range(L):
        full[:, :, i] = np.uint64(mods[i] - 1) if word == "q-1" else np.uint64(2 ** 64 - 1)
    ops = [full.copy() for _ in range(5)]
    modes = [0, 1, 1, 0]
    chained = ops[0]
    for j, md in enumerate(modes):
        chained = ctx.sub(chained, ops[j + 1]) if md else ctx.add(chained, ops[j + 1])
    got = ctx.add_many(ops, modes)
    assert_words(got, chained, f"fold vs chained add/sub at {word}")
    assert_words(got, restate(ops, mods, modes), f"fold vs restatement at {word}")


def test_sub_steps_on_unreduced_words():
    """sub steps whose words reach the borrow form's two branches away from the canonical range: x - 0 with x = 2^64 - 1 stays
    2^64 - 1 (no borrow, no reduction), 0 - (2^64 - 1) is q + 1 (one q added on the borrow); then uniform 64-bit words.  The fold,
    chained sb200_sub calls and the restatement agree word for word"""
    n, bits, L, B, size = 4096, [50, 40, 60], 2, 2, 2
    mods, ctx = context(n, bits)
    top = np.uint64(2 ** 64 - 1)
    rng = np.random.default_rng(64)
    for x, y in ((top, np.uint64(0)), (np.uint64(0), top), (None, None)):
        if x is None:
            ops = [rng.integers(0, top, (B, size, L, n), dtype=np.uint64, endpoint=True) for _ in range(4)]
        else:
            ops = [np.full((B, size, L, n), x), np.full((B, size, L, n), y)]
        modes = [1] * (len(ops) - 1)
        want = restate(ops, mods, modes)
        if x is not None:
            first = int(want[0, 0, 0, 0])
            assert first == (2 ** 64 - 1 if x == top else mods[0] + 1), first
        chained = ops[0]
        for j in range(1, len(ops)):
            chained = ctx.sub(chained, ops[j])
        assert_words(chained, want, f"chained sub from {x}, {y}")
        assert_words(ctx.add_many(ops, modes), want, f"fold of sub steps from {x}, {y}")


@needs_ref
def test_equal_sizes_vs_reference():
    n, bits, L, B = 4096, [50, 40, 40, 60], 3, 2
    mods = R.coeff_modulus_create(n, bits)
    ctx = sb().Context(sb().CKKS, n, mods)
    rc = R.RefContext(R.CKKS, n, mods, 0)
    rng = np.random.default_rng(17)
    ops = rand_ops(rng, mods, n, L, B, [3, 3, 3, 3])
    modes = [0, 1, 0]
    got = ctx.add_many(ops, modes)
    for b in range(B):
        want = ops[0][b]
        for j, md in enumerate(modes):
            want = rc.linear(md, L, want, ops[j + 1][b])
        assert_words(got[b], want, f"ciphertext {b}")


def test_n65536_32_primes():
    n = 65536
    mods, ctx = context(n, [50] * 32)
    L, B = 32, 1
    rng = np.random.default_rng(65536)
    ops = rand_ops(rng, mods, n, L, B, [2, 3, 2])
    modes = [1, 0]
    assert_words(ctx.add_many(ops, modes), restate(ops, mods, modes), "n = 65536, 32 primes")


def test_chunked_by_scratch_limit():
    """the device entry point does not depend on the scratch budget, nor the host one on its staging size"""
    S = sb()
    n, bits, L, B = 4096, [50, 40, 60], 2, 7
    mods = sb().coeff_modulus_create(n, bits)
    t = batching_prime(n, 20)
    ctx = S.Context(S.BGV, n, mods, t)
    rng = np.random.default_rng(9)
    ops = rand_ops(rng, mods, n, L, B, [2, 3, 2])
    modes, factors = [S.FOLD_SCALED, S.FOLD_SUB], [[3, 5], [0, 0]]
    want = restate(ops, mods, modes, factors)
    ctx.set_limit(ctx.LIMIT_SCRATCH_BYTES, 1 << 20)
    ctx.set_limit(ctx.LIMIT_HOST_STAGE_BYTES, 3 * 5 * L * n * 8)  # a few ciphertexts per staging chunk
    assert_words(ctx.add_many(ops, modes, factors), want, "small staging")
    out = _dev(np.zeros_like(want))
    ctx.d_add_many([_dev(o) for o in ops], out, L, B, [2, 3, 2], modes, factors)
    assert_words(_host(out), want, "small scratch budget")


def test_host_staging_chunks():
    """the host entry point cut into several staging chunks with a ragged last one, equal word for word to the stream form"""
    import torch

    S = sb()
    n, bits, L, B = 4096, [50, 40, 60], 2, 7
    mods = sb().coeff_modulus_create(n, bits)
    ctx = S.Context(S.BGV, n, mods, batching_prime(n, 20))
    rng = np.random.default_rng(13)
    sizes = [3, 2, 4, 2]
    ops = rand_ops(rng, mods, n, L, B, sizes)
    modes, factors = [S.FOLD_SUB, S.FOLD_SCALED, S.FOLD_SUB | S.FOLD_SCALED], [[0, 0], [3, 5], [7, 11]]
    out = _dev(np.zeros((B, 4, L, n), dtype=np.uint64))
    ctx.d_add_many([_dev(o) for o in ops], out, L, B, sizes, modes, factors)
    torch.cuda.synchronize()
    per_ct = (sum(sizes) + 4) * L * n * 8
    ctx.set_limit(ctx.LIMIT_HOST_STAGE_BYTES, 2 * per_ct)  # chunks of 2, 2, 2, 1 members
    assert_words(ctx.add_many(ops, modes, factors), _host(out), "chunked host form vs stream form")


def test_argument_errors_leave_output_untouched():
    S = sb()
    n, bits, L, B = 4096, [50, 40, 60], 2, 2
    mods, ctx = context(n, bits)
    rng = np.random.default_rng(1)
    ops = rand_ops(rng, mods, n, L, B, [2, 3])
    d = [_dev(o) for o in ops]
    sentinel = np.full((B, 3, L, n), 7, dtype=np.uint64)
    out = _dev(sentinel)

    def call(exc, operands, sizes, modes=None, factors=None, target=None):
        with pytest.raises(exc):
            ctx.d_add_many(operands, out if target is None else target, L, B, sizes, modes, factors)
        assert_words(_host(out), sentinel, "output after a rejected call")

    call(ValueError, [], [])                                   # count = 0
    call(ValueError, d, [2, 17])                               # size above SEAL_CIPHERTEXT_SIZE_MAX
    call(ValueError, d, [0, 3])                                # size 0
    call(ValueError, d, [2, 3], [4])                           # mode outside 0..3
    call(ValueError, [d[0], 0], [2, 3])                        # NULL operand (SB200_E_POINTER)
    call(ValueError, d, [2, 3], [S.FOLD_SCALED], None)         # scaled step without factors (SB200_E_POINTER)
    call(ValueError, [d[0], out], [2, 3])                      # output aliases operand 1
    big = _dev(np.zeros((B, 2, L, n), dtype=np.uint64))
    with pytest.raises(ValueError):                            # in place on operand 0, which is smaller than the output
        ctx.d_add_many([big, d[1]], big, L, B, [2, 3])
    with pytest.raises(ValueError):
        ctx.add_many([], None)
    # the host form refuses the same overlaps: here the output on operand 0, which is smaller (SB200_E_INVALID_ARG, nothing written)
    lib = S.lib()
    h = rng.integers(0, 2**63, (B, 3, L, n), dtype=np.uint64)  # room for the output's three polynomials
    before = h.copy()
    c_sizes, c_modes, _ = ctx._fold_args([2, 3], None, None)
    ptrs = (C.c_void_p * 2)(h.ctypes.data, np.ascontiguousarray(ops[1]).ctypes.data)
    assert lib.sb200_add_many_host(ctx.h, L, B, 2, c_sizes, ptrs, c_modes, None, S._hp(h)) == -1
    assert b"add_many: the output slab must not overlap an operand [0] other than exactly in place" in lib.sb200_last_error()
    assert_words(h, before, "host output after a rejected call")


@needs_ref
def test_cpp_compositions_against_seal_evaluator():
    """tests/cpp/shim_compose_test.cpp: add_inplace / sub_inplace across sizes and correction factors, add_many, multiply_many,
    exponentiate, mod_switch_to / rescale_to of seal_b200::Evaluator on CiphertextBatch against seal::Evaluator (words, metadata,
    errors, key-switching passes and distinct products)"""
    exe = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref", "bin", "shim_compose_test")
    if not os.path.exists(exe):
        pytest.skip("shim_compose_test not built (reference sources absent at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert "shim_compose_test ok" in r.stdout


def _dev(x):
    import torch

    return torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).cuda()


def _host(t):
    return t.cpu().numpy().view(np.uint64)
