"""Plaintext operations on batches with one plaintext per ciphertext (plain_count = batch) or one plaintext for the whole batch
(plain_count = 1): sb200_multiply_plain_n, sb200_multiply_plain_coeff_n, sb200_add_plain_coeff_n and sb200_add_plain_ntt, their
host-buffer and stream entry points, word for word against the reference (oracle/_ref/libsealref.so)."""
import ctypes as C

import numpy as np
import pytest

import refseal as R
from common import assert_words, rand_ct

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsealref.so not present")

BITS = [50, 36, 45, 60]
BATCH = 3
SCHEMES = {"ckks": R.CKKS, "bfv": R.BFV, "bgv": R.BGV}


def sb():
    import seal_b200

    return seal_b200


def contexts(scheme, n, bits=BITS, t_bits=20):
    mods = R.coeff_modulus_create(n, bits)
    sid = SCHEMES[scheme]
    t = 0 if scheme == "ckks" else R.plain_modulus_batching(n, t_bits)
    return mods, t, R.RefContext(sid, n, mods, t), sb().Context(sid, n, mods, t)


def edge_plain(rng, t, n, count):
    """coefficient-form plaintexts [count][n] < t whose first words sit at the lift edges 0, t - 1, (t + 1) / 2, (t + 1) / 2 - 1"""
    p = rng.integers(0, t, (count, n), dtype=np.uint64)
    p[:, :4] = [0, t - 1, (t + 1) // 2, (t + 1) // 2 - 1]
    return p


def ref_add_ntt(rc, subtract, L, a, plain):
    """CKKS add_plain / sub_plain of one ciphertext: c_0 +/- plain, the other polynomials unchanged (Evaluator::add / sub with a
    ciphertext whose c_0 is the plaintext and whose other polynomials are zero: the same add_poly_coeffmod on every row)"""
    pad = np.zeros_like(a)
    pad[0] = plain
    return rc.linear(1 if subtract else 0, L, a, pad)


def dev(x):
    import torch

    return torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint64)


@needs_ref
@pytest.mark.parametrize("scheme", ["ckks", "bfv", "bgv"])
def test_ntt_form_plain_ops_vs_reference(scheme):
    """multiply_plain with NTT-form plaintexts (CKKS, BGV, transformed BFV) and CKKS add_plain / sub_plain, per ciphertext and
    shared, at the first level (size 2) and a lower level (size 3)"""
    n = 4096
    mods, _, rc, ctx = contexts(scheme, n)
    rng = np.random.default_rng(71)
    for L, size in ((3, 2), (2, 3)):
        a = rand_ct(rng, mods, n, size, L, BATCH)
        per = rand_ct(rng, mods, n, 1, L, BATCH)[:, 0]
        one = per[1]
        rep = np.stack([one] * BATCH)
        got_per, got_one = ctx.multiply_plain_n(a, per), ctx.multiply_plain_n(a, one)
        assert_words(got_per, ctx.multiply_plain(a, per), "plain_count = batch vs sb200_multiply_plain")
        assert_words(got_one, ctx.multiply_plain_n(a, rep), "shared vs replicated multiply_plain")
        for i in range(BATCH):
            assert_words(got_per[i], rc.multiply_plain(L, a[i], per[i]), f"multiply_plain L={L} ct {i}")
            assert_words(got_one[i], rc.multiply_plain(L, a[i], one), f"shared multiply_plain L={L} ct {i}")
        if scheme != "ckks":
            continue
        for subtract in (False, True):
            gp, go = ctx.add_plain_ntt(a, per, subtract), ctx.add_plain_ntt(a, one, subtract)
            assert (gp[:, 1:] == a[:, 1:]).all() and (go[:, 1:] == a[:, 1:]).all(), "only c_0 changes"
            assert_words(go, ctx.add_plain_ntt(a, rep, subtract), "shared vs replicated add_plain")
            for i in range(BATCH):
                assert_words(gp[i], ref_add_ntt(rc, subtract, L, a[i], per[i]), f"add_plain sub={subtract} L={L} ct {i}")
                assert_words(go[i], ref_add_ntt(rc, subtract, L, a[i], one), f"shared add_plain sub={subtract} L={L} ct {i}")


@needs_ref
@pytest.mark.parametrize("scheme,t_bits", [("bfv", 20), ("bfv", 38), ("bgv", 20), ("bgv", 38)])
def test_coeff_plain_ops_vs_reference(scheme, t_bits):
    """coefficient-form plaintexts: multiply_plain, add_plain, sub_plain per ciphertext and shared, plaintext words at the lift
    edges; BGV with correction factors 1, a general value and t - 1 (one per plaintext)"""
    n = 4096
    mods, t, rc, ctx = contexts(scheme, n, t_bits=t_bits)
    rng = np.random.default_rng(73 + t_bits)
    ntt = scheme == "bgv"
    factors = [1, 12345 % t, t - 1]
    for L, size in ((3, 2), (1, 3)):
        a = rand_ct(rng, mods, n, size, L, BATCH)
        per = edge_plain(rng, t, n, BATCH)
        one = per[2]
        rep = np.stack([one] * BATCH)
        mp, mo = ctx.multiply_plain_coeff_n(a, per, ntt), ctx.multiply_plain_coeff_n(a, one, ntt)
        assert_words(mp, ctx.multiply_plain_coeff(a, per, ntt), "plain_count = batch vs sb200_multiply_plain_coeff")
        assert_words(mo, ctx.multiply_plain_coeff_n(a, rep, ntt), "shared vs replicated multiply_plain")
        for i in range(BATCH):
            assert_words(mp[i], rc.plain_op_coeff(0, L, a[i], per[i], ntt), f"multiply_plain L={L} ct {i}")
            assert_words(mo[i], rc.plain_op_coeff(0, L, a[i], one, ntt), f"shared multiply_plain L={L} ct {i}")
        if scheme == "bfv":  # transformed BFV ciphertexts: the NTT branch of multiply_plain, shared
            mn = ctx.multiply_plain_coeff_n(a, one, True)
            assert_words(mn[0], rc.plain_op_coeff(0, L, a[0], one, True), "shared multiply_plain, transformed BFV")
        for subtract in (False, True):
            mode = 2 if subtract else 1
            cf = None if scheme == "bfv" else np.array(factors, dtype=np.uint64)
            ap = ctx.add_plain_coeff_n(a, per, subtract, cf)
            assert_words(ap, ctx.add_plain_coeff(a, per, subtract, cf), "plain_count = batch vs sb200_add_plain_coeff")
            for i in range(BATCH):
                assert_words(ap[i], rc.plain_op_coeff(mode, L, a[i], per[i], ntt, 1 if cf is None else factors[i]), f"mode {mode} ct {i}")
            for f in ([None] if scheme == "bfv" else factors):
                ao = ctx.add_plain_coeff_n(a, one, subtract, None if f is None else [f])
                want = ctx.add_plain_coeff_n(a, rep, subtract, None if f is None else [f] * BATCH)
                assert_words(ao, want, f"shared vs replicated mode {mode} cf {f}")
                for i in range(BATCH):
                    assert_words(ao[i], rc.plain_op_coeff(mode, L, a[i], one, ntt, 1 if f is None else f), f"shared mode {mode} cf {f} ct {i}")


@needs_ref
@pytest.mark.parametrize("scheme", ["ckks", "bfv", "bgv"])
def test_stream_entry_points_in_and_out_of_place(scheme):
    """the stream entry points on device slabs give the host entry points' words, out of place and in place"""
    import torch

    n, L, size = 4096, 3, 2
    mods, t, rc, ctx = contexts(scheme, n)
    rng = np.random.default_rng(79)
    a = rand_ct(rng, mods, n, size, L, BATCH)
    ntt_per = rand_ct(rng, mods, n, 1, L, BATCH)[:, 0]
    coeff_per = edge_plain(rng, t, n, BATCH) if t else None
    cases = [("multiply_plain", ntt_per, lambda p, cnt: ctx.multiply_plain_n(a, p),
              lambda da, dp, do, cnt: ctx.d_multiply_plain_n(da, dp, do, L, size, BATCH, cnt))]
    if scheme == "ckks":
        for s in (False, True):
            cases.append((f"add_plain sub={s}", ntt_per, lambda p, cnt, s=s: ctx.add_plain_ntt(a, p, s),
                          lambda da, dp, do, cnt, s=s: ctx.d_add_plain_ntt(da, dp, do, L, size, BATCH, cnt, s)))
    else:
        ntt = scheme == "bgv"
        cases.append(("multiply_plain_coeff", coeff_per, lambda p, cnt: ctx.multiply_plain_coeff_n(a, p, ntt),
                      lambda da, dp, do, cnt: ctx.d_multiply_plain_coeff_n(da, dp, do, L, size, BATCH, cnt, ntt)))
        for s in (False, True):
            def cf(cnt):
                return None if scheme == "bfv" else [t - 1] * cnt
            cases.append((f"add_plain_coeff sub={s}", coeff_per, lambda p, cnt, s=s: ctx.add_plain_coeff_n(a, p, s, cf(cnt)),
                          lambda da, dp, do, cnt, s=s: ctx.d_add_plain_coeff_n(da, dp, do, L, size, BATCH, cnt, s, cf(cnt))))
    for name, per, on_host, on_dev in cases:
        for cnt, p in ((BATCH, per), (1, per[0])):
            want = on_host(p, cnt)
            da, dp = dev(a), dev(p)
            do = torch.zeros_like(da)
            on_dev(da, dp, do, cnt)
            torch.cuda.synchronize()
            assert_words(host(do), want, f"{name} plain_count={cnt} out of place")
            assert_words(host(da), a, f"{name} plain_count={cnt}: input unchanged")
            assert_words(host(dp), p, f"{name} plain_count={cnt}: plaintext unchanged")
            on_dev(da, dp, da, cnt)
            torch.cuda.synchronize()
            assert_words(host(da), want, f"{name} plain_count={cnt} in place")
    # one sample against the reference through the stream path
    if scheme == "ckks":
        assert_words(cases[1][2](ntt_per[0], 1)[2], ref_add_ntt(rc, False, L, a[2], ntt_per[0]), "shared add_plain ct 2")
    else:
        assert_words(cases[1][2](coeff_per[0], 1)[2], rc.plain_op_coeff(0, L, a[2], coeff_per[0], scheme == "bgv"), "shared multiply_plain ct 2")


@needs_ref
def test_shared_multiply_accepts_unreduced_words_like_the_reference():
    """a shared NTT-form plaintext (and ciphertext) whose words are congruent but not reduced gives the reference's words, as the
    per-ciphertext form does (test_dyadic_kernels_accept_unreduced_words_like_the_reference)"""
    import torch

    n, L = 4096, 3
    mods, _, rc, ctx = contexts("ckks", n)
    rng = np.random.default_rng(83)
    a = rand_ct(rng, mods, n, 2, L, BATCH)
    one = rand_ct(rng, mods, n, 1, L)[0]
    ua, up = a.copy(), one.copy()
    for i in range(L):
        q = np.uint64(mods[i])
        for arr in (ua[:, :, i, :], up[i, :]):
            mask = rng.integers(0, 3, arr.shape) == 0
            arr[mask] += q * np.uint64((2 ** 63 // mods[i]) - 1)
    assert (up != one).any()
    got = ctx.multiply_plain_n(ua, up)
    da = dev(ua)
    ctx.d_multiply_plain_n(da, dev(up), da, L, 2, BATCH, 1)
    torch.cuda.synchronize()
    assert_words(host(da), got, "stream vs host")
    for i in range(BATCH):
        assert_words(got[i], rc.multiply_plain(L, a[i], one), f"ct {i}")


@needs_ref
@pytest.mark.parametrize("scheme", ["ckks", "bgv"])
def test_chunked_batches_give_the_same_words(scheme):
    """7 ciphertexts cut into chunks of 2 (3 full chunks and a ragged tail) by a small scratch budget (device chunks of the
    per-ciphertext coefficient-form operations) and a small host staging budget (the host pipeline) give the words of one chunk"""
    import torch

    n, L, size, batch = 16384, 3, 2, 7
    mods, t, rc, ctx = contexts(scheme, n)
    small = sb().Context(SCHEMES[scheme], n, mods, t)
    small.set_limit(small.LIMIT_SCRATCH_BYTES, 1 << 20)  # L n words of one transformed plaintext: 2 per chunk
    small.set_limit(small.LIMIT_HOST_STAGE_BYTES, 4 << 20)  # ~1.7 MB per ciphertext: 2 per host chunk
    rng = np.random.default_rng(89)
    a = rand_ct(rng, mods, n, size, L, batch)
    if scheme == "ckks":
        per = rand_ct(rng, mods, n, 1, L, batch)[:, 0]
        ops = [lambda c, p: c.multiply_plain_n(a, p), lambda c, p: c.add_plain_ntt(a, p, True)]
        dops = [lambda c, da, dp, cnt: c.d_multiply_plain_n(da, dp, da, L, size, batch, cnt)]
    else:
        per = edge_plain(rng, t, n, batch)
        ops = [lambda c, p: c.multiply_plain_coeff_n(a, p, True),
               lambda c, p: c.add_plain_coeff_n(a, p, False, [5] * (1 if p.ndim == 1 else batch))]
        dops = [lambda c, da, dp, cnt: c.d_multiply_plain_coeff_n(da, dp, da, L, size, batch, cnt, True),
                lambda c, da, dp, cnt: c.d_add_plain_coeff_n(da, dp, da, L, size, batch, cnt, True, [7] * cnt)]
    for p, cnt in ((per, batch), (per[3], 1)):
        for op in ops:
            assert_words(op(small, p), op(ctx, p), f"host pipeline chunks, plain_count={cnt}")
        for dop in dops:
            got, want = dev(a), dev(a)
            dop(small, got, dev(p), cnt)
            dop(ctx, want, dev(p), cnt)
            torch.cuda.synchronize()
            assert torch.equal(got, want), f"device chunks, plain_count={cnt}"
    want0 = rc.multiply_plain(L, a[6], per[6]) if scheme == "ckks" else rc.plain_op_coeff(0, L, a[6], per[3], True)
    got0 = ops[0](small, per if scheme == "ckks" else per[3])[6]
    assert_words(got0, want0, "ragged tail vs the reference")


@needs_ref
def test_headline_shape_sample():
    """n = 65536 with 32 primes, level 31, 8 ciphertexts: shared and per-ciphertext multiply_plain and add_plain on the device,
    sampled ciphertexts against the reference"""
    import torch

    n, L, batch = 65536, 31, 8
    mods = R.coeff_modulus_create(n, [55] * 32)
    rc, ctx = R.RefContext(R.CKKS, n, mods), sb().Context(sb().CKKS, n, mods)
    rng = np.random.default_rng(97)
    a = rand_ct(rng, mods, n, 2, L, batch)
    per = rand_ct(rng, mods, n, 1, L, batch)[:, 0]
    da = dev(a)
    out = torch.empty_like(da)
    for cnt, p in ((batch, per), (1, per[5])):
        dp = dev(p)
        ctx.d_multiply_plain_n(da, dp, out, L, 2, batch, cnt)
        torch.cuda.synchronize()
        for i in (0, batch - 1):
            assert_words(host(out[i]), rc.multiply_plain(L, a[i], per[i] if cnt == batch else per[5]), f"multiply_plain {cnt} ct {i}")
        ctx.d_add_plain_ntt(da, dp, out, L, 2, batch, cnt)
        torch.cuda.synchronize()
        for i in (1, batch - 2):
            assert_words(host(out[i]), ref_add_ntt(rc, False, L, a[i], per[i] if cnt == batch else per[5]), f"add_plain {cnt} ct {i}")


def test_argument_errors():
    import torch

    n, L, size = 4096, 2, 2
    mods = sb().coeff_modulus_create(n, [50, 45, 60])
    ckks = sb().Context(sb().CKKS, n, mods)
    rng = np.random.default_rng(101)
    a = rand_ct(rng, mods, n, size, L, BATCH)
    two = rand_ct(rng, mods, n, 1, L, 2)[:, 0]
    lib, hp = sb().lib(), sb()._hp
    out = np.zeros_like(a)
    for fn in (lib.sb200_multiply_plain_n_host, lambda *x: lib.sb200_add_plain_ntt_host(*x[:5], 0, *x[5:])):
        assert fn(ckks.h, L, size, BATCH, 2, hp(a), hp(two), hp(out)) == -1, "plain_count neither 1 nor batch"
        assert b"plain_count" in lib.sb200_last_error()
        assert fn(ckks.h, L, size, BATCH, 0, hp(a), hp(two), hp(out)) == -1
        assert fn(ckks.h, L, size, BATCH, 1, hp(a), None, hp(out)) == -6, "NULL plaintext"
    with pytest.raises(ValueError, match="plain_count"):
        ckks.d_multiply_plain_n(dev(a), dev(two), dev(out), L, size, BATCH, 2)
    with pytest.raises(ValueError):
        ckks.d_add_plain_ntt(dev(a), 0, dev(out), L, size, BATCH, 1)
    dp = dev(two[0])
    with pytest.raises(ValueError, match="must not alias"):
        ckks.d_multiply_plain_n(dev(a), dp, dp, L, size, BATCH, 1)
    t = 65537
    for sid, name in ((sb().BFV, "BFV"), (sb().BGV, "BGV")):
        c = sb().Context(sid, n, mods, t)
        with pytest.raises(ValueError, match=f"{name} plain cannot be in NTT form"):
            c.add_plain_ntt(a, two[0])
        plain = rng.integers(0, t, (2, n), dtype=np.uint64)
        with pytest.raises(ValueError, match="plain_count"):
            c.d_add_plain_coeff_n(dev(a), dev(plain), dev(out), L, size, BATCH, 2)
        rc = lib.sb200_multiply_plain_coeff_n_host(c.h, L, size, BATCH, 1, 0, hp(a), None, hp(out))
        assert rc == -6, "NULL plaintext"
    torch.cuda.synchronize()


@needs_ref
@pytest.mark.parametrize("scheme", ["ckks", "bgv"])
def test_shared_kernel_over_several_ciphertext_groups(scheme):
    """19 ciphertexts: the shared-plaintext kernel's CTAs cover groups of 8, so three groups with a ragged one, on the stream entry
    points (one launch for the whole batch) against the replicated plaintext and the reference"""
    import torch

    n, L, size, batch = 4096, 3, 3, 19
    mods, t, rc, ctx = contexts(scheme, n)
    rng = np.random.default_rng(103)
    a = rand_ct(rng, mods, n, size, L, batch)
    one = rand_ct(rng, mods, n, 1, L)[0]
    ops = [(lambda da, dp, cnt: ctx.d_multiply_plain_n(da, dp, da, L, size, batch, cnt), lambda i: rc.multiply_plain(L, a[i], one))]
    if scheme == "ckks":
        for s in (False, True):
            ops.append((lambda da, dp, cnt, s=s: ctx.d_add_plain_ntt(da, dp, da, L, size, batch, cnt, s),
                        lambda i, s=s: ref_add_ntt(rc, s, L, a[i], one)))
    else:  # BGV add_plain: the transformed shared plaintext, correction factor t - 1
        c = edge_plain(rng, t, n, 1)[0]
        for s in (False, True):
            ops.append((lambda da, dp, cnt, s=s: ctx.d_add_plain_coeff_n(da, dev(c if cnt == 1 else np.stack([c] * batch)), da, L, size,
                                                                         batch, cnt, s, [t - 1] * cnt),
                        lambda i, s=s: rc.plain_op_coeff(2 if s else 1, L, a[i], c, True, t - 1)))
    for run, want in ops:
        shared, rep = dev(a), dev(a)
        run(shared, dev(one), 1)
        run(rep, dev(np.stack([one] * batch)), batch)
        torch.cuda.synchronize()
        assert torch.equal(shared, rep), "shared vs replicated"
        got = host(shared)
        for i in (0, 7, 8, 15, 16, 18):
            assert_words(got[i], want(i), f"ct {i}")


@needs_ref
def test_cpp_plaintext_batch_against_seal_evaluator():
    """tests/cpp/shim_plain_test.cpp: PlaintextBatch, the device encoders and the plaintext members of seal_b200::Evaluator on
    CiphertextBatch against seal::Evaluator (CKKS, BFV and BGV chains, metadata after every step, errors, the transparent result)"""
    import os
    import subprocess

    exe = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref", "bin", "shim_plain_test")
    if not os.path.exists(exe):
        pytest.skip("shim_plain_test not built (reference sources absent at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert "shim_plain_test ok" in r.stdout
