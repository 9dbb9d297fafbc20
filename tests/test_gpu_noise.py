"""GPU (-m gpu): sb200_invariant_noise_budget[_host] against the reference's Decryptor::invariant_noise_budget and the Python
restatement (tests/noise_ref.py), exactly: chosen phases at the arithmetic edges, multiplication chains down to a zero budget,
the shapes and limits of decryption, both entry points, the argument errors; decryption itself after the shared phase helper;
and the C++ stand-in (tests/cpp/shim_noise_test.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import noise_ref as N
import refseal as R
from common import rand_ct

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not N.available(), reason="oracle/_ref/libsealref{,_noise}.so not present")
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")


def sb():
    import seal_b200

    return seal_b200


def _pair(scheme, n, mods, t):
    rc = R.RefContext(scheme, n, mods, t)
    ctx = sb().Context(scheme, n, mods, t)
    return rc, ctx, ctx.load_secret_key(rc.secret_key())


def _structured_batch(scheme, n, mods, t, L, size, rng, extremes):
    """one ciphertext per extreme value, placed at index 0, n - 1 or in between, over small noise elsewhere"""
    cts = []
    for j, v in enumerate(extremes):
        vals = [int(x) for x in rng.integers(-3, 4, n)]
        vals[(0, n - 1, int(rng.integers(1, n - 1)))[j % 3]] = v
        cts.append(N.structured_ct(scheme, n, mods, t, L, size, vals))
    return np.stack(cts)


def _d_budgets(ctx, sk, ct):
    import torch

    B, size, L, _ = ct.shape
    d = torch.from_numpy(ct.view(np.int64)).cuda()
    out = torch.full((B,), -5, dtype=torch.int32, device="cuda")
    ctx.d_invariant_noise_budget(d, sk, out, L, size, B)
    torch.cuda.synchronize()
    return out.cpu().numpy()


@needs_ref
@pytest.mark.parametrize("scheme", [R.BFV, R.BGV])
@pytest.mark.parametrize("n,bits,L", [(256, [40, 40, 40, 50], 3), (4096, [60, 60, 60, 60, 60], 4), (8192, [50], 1)])
def test_structured_phases(scheme, n, bits, L):
    mods = R.coeff_modulus_create(n, bits)
    t = R.plain_modulus_batching(n, 20)
    rc, ctx, sk = _pair(scheme, n, mods, t)
    rng = np.random.default_rng(n + scheme)
    Q, tb = N.total_bits(mods, L)
    ext = N.edge_values(Q, tb)
    for size in (2, 3):
        ct = _structured_batch(scheme, n, mods, t, L, size, rng, ext)
        got_h, got_d = ctx.invariant_noise_budget(ct, sk), _d_budgets(ctx, sk, ct)
        assert (got_h == got_d).all()
        for i, v in enumerate(ext):
            mag = min(v % Q, Q - v % Q)
            want = max(0, tb - mag.bit_length() - 1) if mag > 3 else max(0, tb - 3)  # (small noise elsewhere: |.| <= 3)
            assert N.ref_budget(rc, L, ct[i], scheme == R.BGV) == (0, int(got_h[i])), (i, v)
            assert got_h[i] == want, (i, v)
    if n == 256:
        sk_ntt = rc.secret_key()
        assert all(N.restated_budget(scheme, n, mods, t, sk_ntt, ct[i]) == got_h[i] for i in range(len(ext)))


@needs_ref
@pytest.mark.parametrize("scheme,n", [(R.BFV, 4096), (R.BFV, 8192), (R.BGV, 4096)])
def test_multiplication_chain_to_zero(scheme, n):
    import torch

    mods = R.coeff_modulus_bfv_default(n) if scheme == R.BFV else R.coeff_modulus_create(n, [60, 50, 50, 50, 60])
    t = R.plain_modulus_batching(n, 20)
    rc, ctx, sk = _pair(scheme, n, mods, t)
    rk = ctx.load_key(rc.relin_key())
    L, B = len(mods) - 1, 3
    d = torch.zeros((B, 2, L, n), dtype=torch.int64, device="cuda")
    ctx.d_encrypt_zero_symmetric(sk, d, L, B)
    torch.cuda.synchronize()
    ct = d.cpu().numpy().view(np.uint64).copy()  # fresh encryptions of zero on the device
    steps = 0
    while True:
        got = ctx.invariant_noise_budget(ct, sk)
        assert (got == _d_budgets(ctx, sk, ct)).all()
        for i in range(B):
            assert N.ref_budget(rc, L, ct[i], scheme == R.BGV) == (0, int(got[i])), (steps, i)
        if (got == 0).all() or steps > 12:
            break
        ct = ctx.multiply_relinearize(ct, ct, rk)
        if scheme == R.BGV and L > 1:
            ct, L = ctx.mod_switch_to_next(ct), L - 1
        steps += 1
    assert (got == 0).all(), got


@needs_ref
def test_levels_sizes_and_chunks():
    # L = 60 thirty-bit primes at n = 4096 (the decryption limit), L = 61 rejected before any launch
    n = 4096
    mods = R.coeff_modulus_create(n, [30] * 62)
    t = R.plain_modulus_batching(n, 20)
    rc, ctx, sk = _pair(R.BFV, n, mods, t)
    rng = np.random.default_rng(60)
    Q, tb = N.total_bits(mods, 60)
    ct = _structured_batch(R.BFV, n, mods, t, 60, 2, rng, [0, 1 << 100, -(1 << 1000), (Q - 1) // 2])
    got = ctx.invariant_noise_budget(ct, sk)
    assert [N.ref_budget(rc, 60, c, False) for c in ct] == [(0, int(g)) for g in got]
    assert got[0] == tb - 3 and got[3] == 0
    before = ctx.launch_count
    with pytest.raises(ValueError, match="decryption supports at most 60 primes per level"):
        ctx.invariant_noise_budget(np.zeros((1, 2, 61, n), dtype=np.uint64), sk)
    assert ctx.launch_count == before
    # sizes 2, 3, 4, 16 of uniform-random ciphertexts, BFV and BGV
    for scheme in (R.BFV, R.BGV):
        mods = R.coeff_modulus_create(256, [40, 40, 40])
        rc, ctx, sk = _pair(scheme, 256, mods, 65537)
        for size in (2, 3, 4, 16):
            ct = rand_ct(rng, mods, 256, size, 2, 3)
            got = ctx.invariant_noise_budget(ct, sk)
            assert [N.ref_budget(rc, 2, c, scheme == R.BGV)[1] for c in ct] == list(got)
    # a few hundred ciphertexts at n = 32768 through many scratch chunks (BFVDefault: 15 data primes)
    n = 32768
    mods = R.coeff_modulus_bfv_default(n)
    t = R.plain_modulus_batching(n, 20)
    rc, ctx, sk = _pair(R.BFV, n, mods, t)
    ctx.set_limit(ctx.LIMIT_SCRATCH_BYTES, 1 << 20)  # two ciphertexts per chunk
    L, B = 1, 300
    Q, tb = N.total_bits(mods, L)
    ext = [(1 << (i % (tb - 2))) * (-1) ** i for i in range(B)]
    ct = _structured_batch(R.BFV, n, mods, t, L, 2, rng, ext)
    got_d = _d_budgets(ctx, sk, ct)
    want = [max(0, tb - max(2, abs(v).bit_length()) - 1) for v in ext]
    assert list(got_d) == want
    for i in range(0, B, 37):
        assert N.ref_budget(rc, L, ct[i], False) == (0, int(got_d[i]))
    ctx.set_limit(ctx.LIMIT_HOST_STAGE_BYTES, 7 * ct[0].nbytes + 100)  # chunks of 7 ciphertexts: 300 = 42 x 7 + 6
    assert (ctx.invariant_noise_budget(ct, sk) == got_d).all()


@needs_ref
@pytest.mark.parametrize("scheme,n", [(R.BFV, 256), (R.BGV, 256), (R.BFV, 4096), (R.BGV, 8192), (R.BFV, 32768)])
def test_decrypt_unchanged(scheme, n):
    """decryption after moving the phase into the helper it shares with the noise budget"""
    mods = R.coeff_modulus_bfv_default(n) if n >= 4096 else R.coeff_modulus_create(n, [50, 45, 60, 55])
    t = R.plain_modulus_batching(n, 20)
    rc, ctx, sk = _pair(scheme, n, mods, t)
    rng = np.random.default_rng(n)
    for L, size in ((len(mods) - 1, 2), (1, 3), (2, 4)):
        ct = rand_ct(rng, mods, n, size, L, 2)
        cf = np.array([1, 12345], dtype=np.uint64) if scheme == R.BGV else None
        got = ctx.decrypt(ct, sk, cf)
        for i in range(2):
            assert (got[i] == rc.decrypt(L, ct[i], scheme == R.BGV, 1 if cf is None else int(cf[i]))).all()


_INVALID, _BATCH = "encrypted is not valid for encryption parameters", "batch must be positive"


def test_argument_errors():
    import torch

    S = sb()
    lib = C.CDLL(S.LIB_PATH)
    lib.sb200_last_error.restype = C.c_char_p
    n, k = 256, 3
    mods = S.coeff_modulus_create(n, [40, 40, 40])
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    words = 2 * 16 * k * n
    h_ct, h_out = np.zeros(words, dtype=np.uint64), np.zeros(16, dtype=np.int32)
    d_ct, d_out = torch.zeros(words, dtype=torch.int64, device="cuda"), torch.zeros(16, dtype=torch.int32, device="cuda")
    rng = np.random.default_rng(3)
    for scheme in (S.BFV, S.BGV, S.CKKS):
        ctx = S.Context(scheme, n, mods, 0 if scheme == S.CKKS else 65537)
        sk = ctx.load_secret_key(rng.integers(0, 1 << 39, (k, n), dtype=np.uint64))
        for variant in ("host", "stream"):
            ct = C.c_void_p(h_ct.ctypes.data if variant == "host" else d_ct.data_ptr())
            out = C.c_void_p(h_out.ctypes.data if variant == "host" else d_out.data_ptr())

            def call(c=ctx.h, key=sk.h, L=2, size=2, batch=1, a=ct, o=out):
                args = [c, key, C.c_size_t(L), C.c_size_t(size), C.c_size_t(batch), a, o]
                rc = lib.sb200_invariant_noise_budget_host(*args) if variant == "host" else lib.sb200_invariant_noise_budget(*args, stream)
                torch.cuda.synchronize()
                return rc, lib.sb200_last_error().decode()

            assert call(c=None)[0] == -6
            assert call(key=None)[0] == -6
            assert call(a=None)[0] == -6
            assert call(o=None)[0] == -6
            assert call(L=0) == (-1, _INVALID)
            assert call(L=k + 1) == (-1, _INVALID)
            assert call(batch=0) == (-1, _BATCH)
            for size in (0, 1, 17):
                assert call(size=size) == (-1, _INVALID)
            if scheme == S.CKKS:
                assert call() == (-2, "unsupported scheme")
            else:
                assert call()[0] == 0


@needs_ref
def test_cpp_stand_in():
    exe = os.path.join(ROOT, "oracle", "_ref", "bin", "shim_noise_test")
    if not os.path.exists(exe):
        pytest.skip("shim_noise_test not built (reference sources absent at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert "shim_noise_test ok" in r.stdout
