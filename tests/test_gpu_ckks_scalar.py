"""CKKSEncoder::encode of one scalar per plaintext on the device (sb200_ckks_encode_scalar / _host): real and int64 constant
polynomials from the fill kernel, complex through the vector transform, word for word against the Python-integer restatement
(tests/ckks_scalar_ref.py) and the reference (oracle/_ref/libsealref_scalar.so); errors with the reference's messages; scalar
batches through multiply_plain / add_plain; and the C++ overloads (tests/cpp/shim_scalar_test.cpp)."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import ckks_scalar_ref as S
import refseal as R
from common import assert_words, rand_ct

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not (S.available() and R.available()), reason="oracle/_ref/libsealref_scalar.so not built")

HERE = os.path.dirname(os.path.abspath(__file__))
BIN = os.path.join(HERE, "..", "oracle", "_ref", "bin", "shim_scalar_test")
DTYPE = {S.REAL: np.float64, S.COMPLEX: np.complex128, S.INT64: np.int64}
E_INVALID_ARG, E_POINTER = -1, -6


def sb():
    import seal_b200

    return seal_b200


def host_encode(ctx, L, kind, values, scale, out=None):
    """sb200_ckks_encode_scalar_host -> (status, message, out [B][L][n])"""
    v = np.ascontiguousarray(values, dtype=DTYPE[kind])
    if out is None:
        out = np.zeros((len(v), L, ctx.n), dtype=np.uint64)
    rc = sb().lib().sb200_ckks_encode_scalar_host(ctx.h, L, len(v), kind, v.ctypes.data, float(scale), out.ctypes.data_as(C.POINTER(C.c_uint64)))
    return rc, sb().lib().sb200_last_error().decode() if rc else "", out


def device_encode(ctx, L, kind, values, scale, sentinel=0):
    """sb200_ckks_encode_scalar on device tensors -> (status, message, out [B][L][n])"""
    import torch

    v = np.ascontiguousarray(values, dtype=DTYPE[kind])
    raw = v.view(np.float64).reshape(len(v), -1) if kind == S.COMPLEX else v.view(np.int64)
    d_v = torch.from_numpy(raw.copy()).cuda()
    d_out = torch.full((len(v), L, ctx.n), sentinel, dtype=torch.int64, device="cuda")
    try:
        ctx.d_ckks_encode_scalar(d_v, d_out, L, len(v), kind, scale)
        rc, msg = 0, ""
    except ValueError:
        rc, msg = E_INVALID_ARG, sb().lib().sb200_last_error().decode()
    torch.cuda.synchronize()
    return rc, msg, d_out.cpu().numpy().view(np.uint64)


def check_cases(ctx, ref, mods, L, kind, cases, with_ref=True):
    """every case against the restatement (and the reference): accepted ones in one batch through both entry points, refused
    ones one by one with the reference's message and the output left untouched"""
    good, want = [], []
    for value, scale in cases:
        w, err = S.restate(mods[:L], ctx.n, kind, value, scale)
        if with_ref:
            rw, rinfo = ref.encode(L, kind, value, scale)
            if w is None:
                assert rw is None and rinfo == err, (value, scale, rinfo, err)
            else:
                assert_words(rw, w, f"restatement vs reference, value {value!r} scale {scale!r}")
        if w is None:
            sentinel = 0x5A5A
            out = np.full((1, L, ctx.n), sentinel, dtype=np.uint64)
            rc, msg, out = host_encode(ctx, L, kind, [value], scale, out)
            assert (rc, msg) == (E_INVALID_ARG, err), (value, scale)
            assert (out == sentinel).all(), "the host entry point wrote the plaintext of a refused value"
            rc, msg, out = device_encode(ctx, L, kind, [value], scale, sentinel)
            assert (rc, msg) == (E_INVALID_ARG, err), (value, scale)
            assert (out == sentinel).all(), "the stream entry point wrote the plaintext of a refused value"
        else:
            good.append((value, scale))
            want.append(w)
    # one batch per scale (the scale is one argument for the whole batch)
    for scale in sorted({s for _, s in good}):
        idx = [i for i, (_, s) in enumerate(good) if s == scale]
        vals = [good[i][0] for i in idx]
        for name, fn in (("host", host_encode), ("device", device_encode)):
            rc, msg, out = fn(ctx, L, kind, vals, scale)
            assert rc == 0, (name, msg)
            for b, i in enumerate(idx):
                assert_words(out[b], want[i], f"{name} entry, value {good[i][0]!r} scale {scale!r}")
    return len(good)


@needs_ref
@pytest.mark.parametrize("n", [4096, 8192, 16384, 32768, 65536])
def test_real_and_int64_match_restatement_and_reference(n):
    mods = R.coeff_modulus_create(n, [60, 40, 40, 60])
    ctx, ref = sb().Context(sb().CKKS, n, mods), S.RefScalar(n, mods)
    for L in (len(mods) - 1, 1):
        assert check_cases(ctx, ref, mods, L, S.REAL, S.real_cases(S.total_bits(mods[:L]))) > 10
        assert check_cases(ctx, ref, mods, L, S.INT64, [(v, 1.0) for v in S.int64_cases(mods)]) > 10


@needs_ref
def test_sixty_prime_level():
    """a level of 60 primes (the reference's multi-precision decomposition for every large product)"""
    n = 4096
    mods = R.coeff_modulus_create(n, [50] * 61)
    ctx, ref = sb().Context(sb().CKKS, n, mods), S.RefScalar(n, mods)
    L = 60
    cases = S.real_cases(S.total_bits(mods[:L])) + [(s * 2.0 ** e * 1.25, 1.0) for e in (300, 700, 1000) for s in (1, -1)]
    cases += [(1e300, 2.0 ** 40), (-1e250, 2.0 ** 400)]
    assert check_cases(ctx, ref, mods, L, S.REAL, cases) > 20
    assert check_cases(ctx, ref, mods, L, S.INT64, [(v, 1.0) for v in S.int64_cases(mods[:4])]) > 10


def test_int64_min_against_restatement():
    n = 4096
    mods = R.coeff_modulus_create(n, [60, 60, 60])
    ctx = sb().Context(sb().CKKS, n, mods)
    want, err = S.restate(mods[:2], n, S.INT64, -(1 << 63))
    assert err is None
    for fn in (host_encode, device_encode):
        rc, msg, out = fn(ctx, 2, S.INT64, [-(1 << 63)], 1.0)
        assert rc == 0, msg
        assert_words(out[0], want, "INT64_MIN")
        rc, msg, _ = fn(ctx, 1, S.INT64, [-(1 << 63)], 1.0)
        assert (rc, msg) == (E_INVALID_ARG, "encoded value is too large")


def test_negative_wrap_on_device():
    n = 4096
    mods = R.coeff_modulus_create(n, [30, 30, 30])
    ctx = sb().Context(sb().CKKS, n, mods)
    out = ctx.ckks_encode_scalar(np.int64(-(1 << 40)), 2)
    for j, q in enumerate(mods[:2]):
        assert (out[j] == ((1 << 64) - (1 << 40)) % q).all()
        assert int(out[j, 0]) != (-(1 << 40)) % q


@pytest.mark.parametrize("kind", [S.REAL, S.COMPLEX, S.INT64])
def test_batches_and_staging_chunks(kind):
    """B = 1 and 3 through both entry points, and a host batch of 7 in chunks of 2 (4 chunks, the last one ragged), equal to the
    same plaintexts encoded one by one"""
    n = 8192
    mods = R.coeff_modulus_create(n, [60, 40, 40, 60])
    ctx = sb().Context(sb().CKKS, n, mods)
    L, scale = 3, 2.0 ** 40
    rng = np.random.default_rng(7 + kind)
    if kind == S.REAL:
        vals = rng.normal(0, 100, 7)
    elif kind == S.COMPLEX:
        vals = rng.normal(0, 100, 7) + 1j * rng.normal(0, 100, 7)
    else:
        vals = rng.integers(-(1 << 40), 1 << 40, 7)
    one = [host_encode(ctx, L, kind, [v], scale)[2][0] for v in vals]
    for B in (1, 3):
        for fn in (host_encode, device_encode):
            rc, msg, out = fn(ctx, L, kind, vals[:B], scale)
            assert rc == 0, msg
            for b in range(B):
                assert_words(out[b], one[b], f"B = {B}, member {b}")
    per_ct = (2 if kind == S.COMPLEX else 1) * 8 + L * n * 8
    ctx.set_limit(ctx.LIMIT_HOST_STAGE_BYTES, 2 * per_ct)
    rc, msg, out = host_encode(ctx, L, kind, vals, scale)
    assert rc == 0, msg
    for b in range(7):
        assert_words(out[b], one[b], f"chunked, member {b}")
    if kind != S.COMPLEX:  # a refused member in the last chunk: nothing is written, not even the earlier chunks
        bad = list(vals)
        bad[6] = math.inf if kind == S.REAL else -(1 << 63)
        sentinel = np.full((7, 1, n), 0x77, dtype=np.uint64)
        rc, msg, out = host_encode(ctx, 1, kind, bad, scale, sentinel)
        assert rc == E_INVALID_ARG and (out == 0x77).all(), msg


@needs_ref
@pytest.mark.parametrize("n", [4096, 65536])
def test_complex_is_the_vector_encode_of_copies(n):
    mods = R.coeff_modulus_create(n, [60, 40, 40, 60])
    ctx = sb().Context(sb().CKKS, n, mods)
    ref = S.RefScalar(n, mods) if n == 4096 else None
    zs = [1.5 - 0.25j, -3.0 + 0j, 0j, 1e6 + 1e-6j]
    for L in (3, 1):
        scale = 2.0 ** 40 if L == 3 else 2.0 ** 30
        for fn in (host_encode, device_encode):
            rc, msg, out = fn(ctx, L, S.COMPLEX, zs, scale)
            assert rc == 0, msg
            for b, z in enumerate(zs):
                assert_words(out[b], ctx.ckks_encode(np.full(n // 2, z), L, scale), f"complex {z}, sb200_ckks_encode of copies")
                if ref is not None:
                    assert_words(out[b], ref.encode(L, S.COMPLEX, z, scale)[0], f"complex {z}, reference")


def test_errors():
    n = 4096
    mods = R.coeff_modulus_create(n, [60, 40, 60])
    ctx = sb().Context(sb().CKKS, n, mods)
    k, L = len(mods), 2
    tb = S.total_bits(mods[:L])
    cases = [
        # (kind, L, values, scale, message)
        (S.REAL, 0, [1.0], 1.0, "parms_id is not valid for encryption parameters"),
        (S.INT64, k + 1, [1], 1.0, "parms_id is not valid for encryption parameters"),
        (S.COMPLEX, k + 1, [1j], 2.0 ** 20, "parms_id is not valid for encryption parameters"),
        (S.REAL, L, [math.inf], 1.0, "value must be finite"),
        (S.COMPLEX, L, [complex(math.nan, 0)], 2.0 ** 20, "values must be finite"),
        (S.COMPLEX, L, [1e300 + 0j], 2.0 ** 40, "encoded values are too large"),
        (S.REAL, L, [1e300], 2.0 ** 40, "encoded value is too large"),
        (S.INT64, L, [(1 << 63) - 1], 1.0, "encoded value is too large") if tb <= 65 else None,
        (S.REAL, L, [1.0], 0.0, "scale out of bounds"),
        (S.REAL, L, [1.0], math.nan, "scale out of bounds"),
        (S.REAL, L, [1.0], 2.0 ** tb, "scale out of bounds"),
        (S.COMPLEX, L, [1 + 0j], 5e-324, "scale out of bounds"),  # accepted by the real kind (below)
        (S.COMPLEX, L, [0j], 2.0 ** (tb - 1), "scale out of bounds"),  # likewise
        # the first failing member in batch order
        (S.REAL, L, [1.0, math.inf, 1e300], 2.0 ** 40, "value must be finite"),
        (S.REAL, L, [1.0, 1e300, math.inf], 2.0 ** 40, "encoded value is too large"),
    ]
    for case in [c for c in cases if c]:
        kind, lv, vals, scale, message = case
        for fn in (host_encode, device_encode):
            if lv < 1 or lv > k:
                v = np.ascontiguousarray(vals, dtype=DTYPE[kind])
                out = np.zeros((len(v), 1, n), dtype=np.uint64)
                rc = sb().lib().sb200_ckks_encode_scalar_host(ctx.h, lv, len(v), kind, v.ctypes.data, float(scale),
                                                              out.ctypes.data_as(C.POINTER(C.c_uint64)))
                msg = sb().lib().sb200_last_error().decode()
            else:
                rc, msg, _ = fn(ctx, lv, kind, vals, scale)
            assert (rc, msg) == (E_INVALID_ARG, message), case
    for kind, vals, scale in ((S.REAL, [1.0], 5e-324), (S.REAL, [2.0 ** -tb], 2.0 ** (tb - 1))):
        rc, msg, out = host_encode(ctx, L, kind, vals, scale)
        assert rc == 0, msg
    lib, out = sb().lib(), np.zeros((1, L, n), dtype=np.uint64)
    v = np.array([1.0])
    outp = out.ctypes.data_as(C.POINTER(C.c_uint64))
    assert lib.sb200_ckks_encode_scalar_host(ctx.h, L, 1, 3, v.ctypes.data, 1.0, outp) == E_INVALID_ARG
    assert lib.sb200_ckks_encode_scalar_host(ctx.h, L, 1, -1, v.ctypes.data, 1.0, outp) == E_INVALID_ARG
    assert lib.sb200_ckks_encode_scalar_host(ctx.h, L, 0, 0, v.ctypes.data, 1.0, outp) == E_INVALID_ARG
    assert lib.sb200_ckks_encode_scalar_host(ctx.h, L, 1, 0, None, 1.0, outp) == E_POINTER
    assert lib.sb200_ckks_encode_scalar_host(ctx.h, L, 1, 0, v.ctypes.data, 1.0, None) == E_POINTER
    assert lib.sb200_ckks_encode_scalar(ctx.h, L, 1, 0, None, 1.0, None, None) == E_POINTER
    t = R.plain_modulus_batching(n, 20)
    bfv = sb().Context(sb().BFV, n, mods, t)
    assert lib.sb200_ckks_encode_scalar_host(bfv.h, L, 1, 0, v.ctypes.data, 1.0, outp) == E_INVALID_ARG
    assert lib.sb200_last_error().decode() == "unsupported scheme"


def test_fill_is_profiled():
    n = 65536
    mods = R.coeff_modulus_create(n, [60] + [50] * 6 + [60])
    ctx = sb().Context(sb().CKKS, n, mods)
    L, B = 7, 5
    ctx.profile(True)
    rc, msg, _ = device_encode(ctx, L, S.REAL, np.arange(B, dtype=np.float64), 2.0 ** 40)
    assert rc == 0, msg
    rows = {name: (launches, by) for name, _, launches, by in ctx.profile_read()}
    ctx.profile(False)
    assert rows["ckks_fill"] == (1, 8.0 * B * L * n)


@needs_ref
def test_scalar_batches_through_plain_operations():
    """a shared (B = 1) and a per-member scalar batch through multiply_plain / add_plain on a batch of ciphertexts, against the
    reference's multiply_plain / add with its own scalar plaintexts"""
    n = 8192
    mods = R.coeff_modulus_create(n, [60, 40, 40, 60])
    ctx, ref, rc = sb().Context(sb().CKKS, n, mods), S.RefScalar(n, mods), R.RefContext(R.CKKS, n, mods)
    L, B, scale = 3, 4, 2.0 ** 40
    rng = np.random.default_rng(11)
    a = rand_ct(rng, mods, n, 2, L, B)
    zero = np.zeros((L, n), dtype=np.uint64)
    # shared: one real constant for the whole batch
    shared = ctx.ckks_encode_scalar(np.float64(3.14159), L, scale)
    p_ref = ref.encode(L, S.REAL, 3.14159, scale)[0]
    assert_words(shared, p_ref, "shared scalar plaintext")
    got = ctx.multiply_plain_n(a, shared)
    for i in range(B):
        assert_words(got[i], rc.multiply_plain(L, a[i], p_ref), f"multiply_plain by a shared scalar, ciphertext {i}")
    got = ctx.add_plain_ntt(a, shared)
    for i in range(B):
        assert_words(got[i], rc.linear(0, L, a[i], np.stack([p_ref, zero])), f"add_plain of a shared scalar, ciphertext {i}")
    # per member: int64 and complex constants (none zero: the reference refuses a transparent product)
    for kind, vals in ((S.INT64, np.array([-5, 3, 7, -(1 << 40)], dtype=np.int64)),
                       (S.COMPLEX, np.array([1 + 1j, -2.5j, 0.5, -0.25 + 3j]))):
        plains = ctx.ckks_encode_scalar(vals, L, scale)
        refs = [ref.encode(L, kind, v, scale)[0] for v in vals]
        got_m, got_a = ctx.multiply_plain_n(a, plains), ctx.add_plain_ntt(a, plains)
        for i in range(B):
            assert_words(plains[i], refs[i], f"kind {kind}, member {i}")
            assert_words(got_m[i], rc.multiply_plain(L, a[i], refs[i]), f"multiply_plain, kind {kind}, ciphertext {i}")
            assert_words(got_a[i], rc.linear(0, L, a[i], np.stack([refs[i], zero])), f"add_plain, kind {kind}, ciphertext {i}")


@pytest.mark.skipif(not os.path.exists(BIN), reason="oracle/_ref/bin/shim_scalar_test not built (oracle/scalar.mk, needs the reference sources)")
def test_cpp_scalar_overloads_and_example_5():
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=900)
    print(r.stdout, r.stderr)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "PASS" in r.stdout
