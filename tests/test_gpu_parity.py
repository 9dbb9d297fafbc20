"""GPU parity tests proper (-m gpu): every call goes through the C-ABI of libseal_b200.so and is compared word for
word with (i) committed golden vectors from the real reference, (ii) the plain-C oracle, (iii) the reference library
itself (oracle/_ref/libsealref.so) where it travelled to the box.  Bar: bit-exact."""
import ctypes as C

import numpy as np
import pytest

import oracle as O
import refseal as R
from common import assert_words, golden, max_ct, rand_ct

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsealref.so not present")


def sb():
    import seal_b200

    return seal_b200


@pytest.mark.parametrize("name", ["ckks_n128", "ckks_n1024", "bfv_n128"])
def test_golden_vectors(name):
    g = golden(name)
    scheme, n, mods, t = int(g["scheme"]), int(g["n"]), [int(x) for x in g["moduli"]], int(g["t"])
    k = len(mods)
    ctx = sb().Context(scheme, n, mods, t)
    for i in range(k):
        assert ctx.ntt_tables(i)[0] == int(g["roots"][i])
    rk = ctx.load_key(g["relin_key"])
    for L in range(k - 1, 0, -1):
        a, b = g[f"L{L}_a"], g[f"L{L}_b"]
        assert (ctx.transform_to_ntt(a) == g[f"L{L}_ntt_fwd_a"]).all()
        assert (ctx.transform_from_ntt(a) == g[f"L{L}_ntt_inv_a"]).all()
        m = ctx.multiply(a, b)
        assert (m == g[f"L{L}_mul"]).all()
        assert (ctx.multiply_relinearize(a, b, rk) == g[f"L{L}_relin"]).all()
        assert (ctx.relinearize(g[f"L{L}_mul"], rk) == g[f"L{L}_relin"]).all()
        if L > 1:
            ms = ctx.rescale_to_next(a) if scheme == sb().CKKS else ctx.mod_switch_to_next(a)
            assert (ms == g[f"L{L}_modswitch_a"]).all()
        for e in g["galois_elts"]:
            e = int(e)
            gk = ctx.load_key(g[f"galois_key_{e}"])
            assert (ctx.apply_galois(a, e, gk) == g[f"L{L}_galois_{e}"]).all()


def test_kat_ntt_n2():
    # native/tests/seal/util/ntt.cpp:75-100 through the CUDA path
    q = 0xFFFFFFFFFFC0001
    ctx = sb().Context(sb().CKKS, 2, [q])
    root, rp, _, irp, _ = ctx.ntt_tables(0)
    assert int(rp[1]) == 288794978602139552 and (int(rp[1]) * int(irp[1])) % q == 1
    x = np.array([[[1, 1]]], dtype=np.uint64)
    assert [int(v) for v in ctx.transform_to_ntt(x)[0, 0]] == [288794978602139553, 864126526004445282]
    z = np.array([[[1, 0]]], dtype=np.uint64)
    assert [int(v) for v in ctx.transform_to_ntt(z)[0, 0]] == [1, 1]


@pytest.mark.parametrize("logn", [3, 8, 11, 12, 13, 14, 15, 16, 17])
def test_ntt_vs_oracle_and_roundtrip(logn):
    n = 1 << logn
    bits = [50, 60, 36] if logn < 17 else [50, 60, 40]
    mods = O.coeff_modulus_create(n, bits)
    ctx = sb().Context(sb().CKKS, n, mods)
    oc = O.Oracle(O.CKKS, n, mods)
    for i in range(3):
        root, rp, _, irp, inv_n = ctx.ntt_tables(i)
        oroot, orp, oirp, oinv = oc.ntt_tables(i)
        assert root == oroot and (rp == orp).all() and (irp == oirp).all() and inv_n == oinv
    rng = np.random.default_rng(logn)
    x = rand_ct(rng, mods, n, 2, 3, batch=3)
    f = ctx.transform_to_ntt(x)
    assert (ctx.transform_from_ntt(f) == x).all()
    assert (f[1] == oc.ntt_forward(3, x[1])).all()
    assert (ctx.transform_from_ntt(x)[2] == oc.ntt_inverse(3, x[2])).all()
    # linearity: NTT(a + b) = NTT(a) + NTT(b)
    y = rand_ct(rng, mods, n, 2, 3, batch=3)
    qv = np.array(mods, dtype=np.uint64)[None, None, :, None]
    s = (x + y) % qv  # primes <= 60 bits so the sum cannot wrap
    assert (ctx.transform_to_ntt(s) == (f + ctx.transform_to_ntt(y)) % qv).all()


@pytest.mark.parametrize("fast", [True, False], ids=["q57", "q60"])
@pytest.mark.parametrize("logn", [1, 3, 6, 7, 8, 9, 11, 12, 13, 14, 15, 16, 17])
def test_ntt_butterfly_classes_vs_oracle(logn, fast):
    """transform_to_ntt / transform_from_ntt word for word against the oracle in both butterfly classes: every prime below 2^57,
    the largest 57-bit prime among them (the guard-free forward instantiations ntt_fwd_col<LOGNA, true> / ntt_fwd_local<true>), or
    a 60-bit prime in the set (guarded); every small-kernel thread count and every LOGNA; uniform words and every word q_i - 1"""
    n = 1 << logn
    mods = O.coeff_modulus_create(n, [50, 57 if fast else 60, 30])
    assert all(q < 2 ** 57 for q in mods) == fast
    ctx = sb().Context(sb().CKKS, n, mods)
    oc = O.Oracle(O.CKKS, n, mods)
    rng = np.random.default_rng(100 + logn)
    for what, x in (("uniform", rand_ct(rng, mods, n, 2, 3)), ("q - 1", max_ct(mods, n, 2, 3))):
        assert_words(ctx.transform_to_ntt(x), oc.ntt_forward(3, x), f"forward, {what} words")
        assert_words(ctx.transform_from_ntt(x), oc.ntt_inverse(3, x), f"inverse, {what} words")


@needs_ref
@pytest.mark.parametrize("n,bits,batch", [(4096, [50, 40, 45, 60], 3), (8192, [54, 54, 54, 54], 4), (16384, [40, 50, 50, 45, 50], 2)])
def test_ckks_ops_vs_reference(n, bits, batch):
    mods = R.coeff_modulus_create(n, bits)
    assert mods == sb().coeff_modulus_create(n, bits)
    k = len(mods)
    rc = R.RefContext(R.CKKS, n, mods)
    ctx = sb().Context(sb().CKKS, n, mods)
    rk = ctx.load_key(rc.relin_key())
    rng = np.random.default_rng(n)
    for L in (k - 1, k - 2, 1):
        a, b = rand_ct(rng, mods, n, 2, L, batch), rand_ct(rng, mods, n, 2, L, batch)
        m = ctx.multiply(a, b)
        r = ctx.relinearize(m, rk)
        mr = ctx.multiply_relinearize(a, b, rk)
        for i in range(batch):
            assert (m[i] == rc.multiply(L, a[i], b[i])).all()
            assert (r[i] == rc.relinearize(L, m[i])).all()
        assert (mr == r).all()
        if L > 1:
            rs = ctx.rescale_to_next(a)
            dr = ctx.mod_switch_to_next(a)
            for i in range(batch):
                assert (rs[i] == rc.rescale(L, a[i])).all()
                assert (dr[i] == rc.mod_switch(L, a[i])).all()
        for step in (1, -2):
            e = rc.galois_elt_from_step(step)
            assert e == ctx.galois_elt_from_step(step)
            gk = ctx.load_key(rc.galois_key(e))
            g = ctx.rotate(a, step, gk)
            for i in range(batch):
                assert (g[i] == rc.rotate(L, a[i], step)).all()


@needs_ref
def test_bfv_keyswitch_vs_reference():
    # BFV branches of switch_key_inplace / apply_galois / mod_switch (coefficient form)
    n = 4096
    mods = R.coeff_modulus_bfv_default(n)
    t = R.plain_modulus_batching(n, 20)
    rb = R.RefContext(R.BFV, n, mods, t)
    ctx = sb().Context(sb().BFV, n, mods, t)
    rng = np.random.default_rng(5)
    L, batch = 2, 3
    a, b = rand_ct(rng, mods, n, 2, L, batch), rand_ct(rng, mods, n, 2, L, batch)
    rk = ctx.load_key(rb.relin_key())
    m = np.stack([rb.multiply(L, a[i], b[i]) for i in range(batch)])
    r = ctx.relinearize(m, rk)
    for i in range(batch):
        assert (r[i] == rb.relinearize(L, m[i])).all()
    for step in (1, -3, 0):
        e = rb.galois_elt_from_step(step)
        gk = ctx.load_key(rb.galois_key(e))
        g = ctx.apply_galois(a, e, gk)
        for i in range(batch):
            assert (g[i] == rb.apply_galois(L, a[i], e)).all()
    ms = ctx.mod_switch_to_next(a)
    for i in range(batch):
        assert (ms[i] == rb.mod_switch(L, a[i])).all()


# The evaluator operations, encoder and decryptor each have a stream entry point sb200_<name> on device slabs and a host-buffer
# entry point sb200_<name>_host with the same arguments minus the stream.  Argument order after the context handle: a / b are the
# input slabs, out the output slab (NTT: a is transformed in place), cf host correction factors, flag the int argument.
ABI_PAIRS = {
    "ntt_forward": ("L", "size", "batch", "a"),
    "ntt_inverse": ("L", "size", "batch", "a"),
    "multiply": ("L", "batch", "a", "b", "out"),
    "multiply_sized": ("L", "size_a", "size_b", "batch", "a", "b", "out"),
    "square": ("L", "batch", "a", "out"),
    "add": ("L", "size", "batch", "a", "b", "out"),
    "sub": ("L", "size", "batch", "a", "b", "out"),
    "negate": ("L", "size", "batch", "a", "out"),
    "multiply_plain": ("L", "size", "batch", "a", "b", "out"),
    "plain_to_ntt": ("L", "batch", "a", "out"),
    "multiply_plain_coeff": ("L", "size", "batch", "flag", "a", "b", "out"),
    "add_plain_coeff": ("L", "size", "batch", "flag", "a", "b", "cf", "out"),
    "batch_encode": ("batch", "a", "out"),
    "batch_decode": ("batch", "a", "out"),
    "relinearize": ("L", "batch", "a", "key", "out"),
    "multiply_relinearize": ("L", "batch", "a", "b", "key", "out"),
    "rescale_to_next": ("L", "batch", "a", "out"),
    "mod_switch_to_next": ("L", "batch", "a", "out"),
    "rescale_to_next_sized": ("L", "size", "batch", "a", "out"),
    "mod_switch_to_next_sized": ("L", "size", "batch", "a", "out"),
    "relinearize_sized": ("L", "size", "batch", "a", "key", "out"),
    "apply_galois": ("L", "batch", "a", "elt", "key", "out"),
    "ckks_encode": ("L", "batch", "a", "count", "flag", "scale", "out"),
    "ckks_decode": ("L", "batch", "a", "scale", "out"),
    "decrypt": ("key", "L", "size", "batch", "a", "cf", "out"),
}
_ABI_SCALARS = {"L": C.c_size_t, "size": C.c_size_t, "size_a": C.c_size_t, "size_b": C.c_size_t, "batch": C.c_size_t, "count": C.c_size_t,
                "flag": C.c_int, "elt": C.c_uint32, "scale": C.c_double}
_abi_lib = None


def abi_call(ctx_h, name, v, stream=None):
    """sb200_<name>_host (stream None) or sb200_<name> on `stream`, arguments from v (pointers as c_void_p or None); returns the
    status and sb200_last_error()"""
    global _abi_lib
    if _abi_lib is None:  # a handle of its own: no argtypes, every argument is passed with its C type
        _abi_lib = C.CDLL(sb().LIB_PATH)
        _abi_lib.sb200_last_error.restype = C.c_char_p
    args = [ctx_h] + [_ABI_SCALARS[f](v[f]) if f in _ABI_SCALARS else v[f] for f in ABI_PAIRS[name]]
    fn = getattr(_abi_lib, f"sb200_{name}_host" if stream is None else f"sb200_{name}")
    rc = fn(*args) if stream is None else fn(*args, stream)
    return rc, _abi_lib.sb200_last_error().decode()


_PAIR_SCHEMES = {"plain_to_ntt": "bfv bgv", "multiply_plain_coeff": "bfv bgv", "add_plain_coeff": "bfv bgv", "batch_encode": "bfv bgv",
                 "batch_decode": "bfv bgv", "rescale_to_next": "ckks", "rescale_to_next_sized": "ckks", "ckks_encode": "ckks", "ckks_decode": "ckks"}


def _pair_inputs(name, ctx, rng, key, sk):
    """seeded inputs of one call: slabs as uint64 arrays (values and complex outputs as their words), the rest as scalars / handles"""
    n, mods, t, L, B = ctx.n, ctx.moduli, ctx.t, 2, 7
    bgv = ctx.scheme == sb().BGV

    def ct(size, lv=L):
        return rand_ct(rng, mods, n, size, lv, B)

    def zeros(*shape):
        return np.zeros((B,) + shape, dtype=np.uint64)

    def coeffs():
        return rng.integers(0, t, (B, n), dtype=np.uint64)

    cf = rng.integers(1, t, B, dtype=np.uint64) if bgv else None
    v = dict(L=L, batch=B)
    if name.startswith("ntt"):
        v.update(size=2, a=ct(2))
    elif name == "multiply":
        v.update(a=ct(2), b=ct(2), out=zeros(3, L, n))
    elif name == "multiply_sized":
        v.update(L=1, size_a=3, size_b=2, a=ct(3, 1), b=ct(2, 1), out=zeros(4, 1, n))
    elif name == "square":
        v.update(a=ct(2), out=zeros(3, L, n))
    elif name in ("add", "sub"):
        v.update(size=2, a=ct(2), b=ct(2), out=zeros(2, L, n))
    elif name == "negate":
        v.update(size=2, a=ct(2), out=zeros(2, L, n))
    elif name == "multiply_plain":
        v.update(size=2, a=ct(2), b=ct(1)[:, 0].copy(), out=zeros(2, L, n))
    elif name == "plain_to_ntt":
        v.update(a=coeffs(), out=zeros(L, n))
    elif name == "multiply_plain_coeff":
        v.update(size=2, flag=int(bgv), a=ct(2), b=coeffs(), out=zeros(2, L, n))
    elif name == "add_plain_coeff":
        v.update(size=2, flag=1, a=ct(2), b=coeffs(), cf=cf, out=zeros(2, L, n))
    elif name.startswith("batch_"):
        v.update(a=coeffs(), out=zeros(n))
    elif name == "relinearize":
        v.update(a=ct(3), key=key, out=zeros(2, L, n))
    elif name == "multiply_relinearize":
        v.update(a=ct(2), b=ct(2), key=key, out=zeros(2, L, n))
    elif name in ("rescale_to_next", "mod_switch_to_next"):
        v.update(a=ct(2), out=zeros(2, L - 1, n))
    elif name in ("rescale_to_next_sized", "mod_switch_to_next_sized"):
        v.update(size=3, a=ct(3), out=zeros(3, L - 1, n))
    elif name == "relinearize_sized":
        v.update(size=4, a=ct(4), key=key, out=zeros(4, L, n))
    elif name == "apply_galois":
        v.update(a=ct(2), elt=3, key=key, out=zeros(2, L, n))
    elif name == "ckks_encode":
        count = n // 2 - 3
        vals = (rng.standard_normal((B, count)) + 1j * rng.standard_normal((B, count))) * 100.0
        v.update(a=np.ascontiguousarray(vals).view(np.uint64), count=count, flag=1, scale=2.0 ** 20, out=zeros(L, n))
    elif name == "ckks_decode":
        v.update(a=ct(1)[:, 0].copy(), scale=2.0 ** 20, out=zeros(n))  # n / 2 complex values: n words
    elif name == "decrypt":
        v.update(key=sk, size=3, a=ct(3), cf=cf, out=zeros(L, n) if ctx.scheme == sb().CKKS else zeros(n))
    return v


def test_device_api_matches_host_api():
    import torch

    n, bits = 4096, [50, 50, 50, 50]
    mods = O.coeff_modulus_create(n, bits)
    ctx = sb().Context(sb().CKKS, n, mods)
    rng = np.random.default_rng(9)
    L, batch = 3, 5
    a, b = rand_ct(rng, mods, n, 2, L, batch), rand_ct(rng, mods, n, 2, L, batch)
    key = rng.integers(0, 1 << 40, (L, 2, 4, n), dtype=np.uint64)  # any residues < q work as a "key" for parity
    rk = ctx.load_key(key)
    da = torch.from_numpy(a.view(np.int64)).cuda()
    db = torch.from_numpy(b.view(np.int64)).cuda()
    out = torch.empty((batch, 2, L, n), dtype=torch.int64, device="cuda")
    before = ctx.launch_count
    ctx.d_multiply_relinearize(da, db, rk, out, L, batch)
    torch.cuda.synchronize()
    assert ctx.launch_count > before
    host = ctx.multiply_relinearize(a, b, rk)
    assert (out.cpu().numpy().view(np.uint64) == host).all()
    oc = O.Oracle(O.CKKS, n, mods)
    assert (host[0] == oc.multiply_relin(L, a[0], b[0], key)).all()


@pytest.mark.parametrize("name", list(ABI_PAIRS))
def test_stream_and_host_entry_points_agree(name):
    """both entry points of every pair produce the same words: the host one through its chunked pipeline (batch 7 at a 64 KiB
    staging limit: several chunks, most operations with a ragged last one), the stream one in one call on torch slabs"""
    import torch

    S = sb()
    n, t = 256, 65537
    mods = S.coeff_modulus_create(n, [40, 40, 40])
    schemes = _PAIR_SCHEMES.get(name, "ckks bfv bgv").split()
    for scheme in schemes:
        sid = {"ckks": S.CKKS, "bfv": S.BFV, "bgv": S.BGV}[scheme]
        ctx = S.Context(sid, n, mods, 0 if scheme == "ckks" else t)
        ctx.set_limit(ctx.LIMIT_HOST_STAGE_BYTES, 1 << 16)
        rng = np.random.default_rng((list(ABI_PAIRS).index(name), schemes.index(scheme)))
        key = ctx.load_key(rng.integers(0, 1 << 39, (2, 2, 3, n), dtype=np.uint64))  # any residues < q work as a key for parity
        sk = ctx.load_secret_key(rng.integers(0, 1 << 39, (3, n), dtype=np.uint64))
        v = _pair_inputs(name, ctx, rng, key.h, sk.h)
        outs = [f for f in ("a", "out") if f in ABI_PAIRS[name]][-1:]  # the NTT overwrites a
        host = {f: v[f].copy() for f in ("a", "b", "out") if f in v}
        dev = {f: torch.from_numpy(x.view(np.int64)).cuda() for f, x in host.items()}
        cf = None if v.get("cf") is None else v["cf"].ctypes.data_as(C.c_void_p)
        hv = dict(v, cf=cf, **{f: x.ctypes.data_as(C.c_void_p) for f, x in host.items()})
        dv = dict(v, cf=cf, **{f: C.c_void_p(x.data_ptr()) for f, x in dev.items()})
        before = ctx.launch_count
        assert abi_call(ctx.h, name, dv, C.c_void_p(torch.cuda.current_stream().cuda_stream))[0] == 0, (name, scheme)
        torch.cuda.synchronize()
        # (the CKKS modulus switch drops the last prime with a device copy: no kernel)
        assert ctx.launch_count > before or (name.startswith("mod_switch") and scheme == "ckks"), (name, scheme)
        assert abi_call(ctx.h, name, hv)[0] == 0, (name, scheme)
        for f in outs:
            got = dev[f].cpu().numpy().view(np.uint64)
            assert (host[f] != v[f]).any() if f == "a" else (host[f] != 0).any(), (name, scheme, "host output unchanged")
            assert (got == host[f]).all(), (name, scheme)


def test_one_context_on_two_streams():
    # calls of one context share its scratch arenas: a call on another stream must wait for the previous call's kernels
    import torch

    n, bits = 8192, [50, 50, 50, 50, 50]
    mods = O.coeff_modulus_create(n, bits)
    ctx = sb().Context(sb().CKKS, n, mods)
    rng = np.random.default_rng(10)
    L, batch = 4, 24
    key = rng.integers(0, 1 << 40, (L, 2, 5, n), dtype=np.uint64)
    rk = ctx.load_key(key)
    ins = [(rand_ct(rng, mods, n, 2, L, batch), rand_ct(rng, mods, n, 2, L, batch)) for _ in range(2)]
    want = [ctx.multiply_relinearize(a, b, rk) for a, b in ins]
    dev = [(torch.from_numpy(a.view(np.int64)).cuda(), torch.from_numpy(b.view(np.int64)).cuda()) for a, b in ins]
    outs = [torch.empty((batch, 2, L, n), dtype=torch.int64, device="cuda") for _ in range(2)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for rep in range(3):
        for i in range(2):
            with torch.cuda.stream(streams[i]):
                ctx.d_multiply_relinearize(dev[i][0], dev[i][1], rk, outs[i], L, batch)
        torch.cuda.synchronize()
        for i in range(2):
            assert (outs[i].cpu().numpy().view(np.uint64) == want[i]).all()


def test_error_codes():
    s = sb()
    with pytest.raises(ValueError):
        s.Context(s.CKKS, 1000, [1099511480321])  # not a power of two
    with pytest.raises(ValueError):
        s.Context(s.CKKS, 1024, [1099511480321 + 2])  # no primitive 2n-th root
    n = 1024
    mods = O.coeff_modulus_create(n, [40, 40, 40])
    ctx = s.Context(s.CKKS, n, mods)
    key = ctx.load_key(np.zeros((1, 2, 3, n), dtype=np.uint64))
    a = np.zeros((1, 3, 2, n), dtype=np.uint64)
    with pytest.raises(ValueError):  # key with too few digits: evaluator.cpp:2635
        ctx.relinearize(a, key)
    with pytest.raises(ValueError):  # rescale at the last level: evaluator.cpp:1521
        ctx.rescale_to_next(np.zeros((1, 2, 1, n), dtype=np.uint64))
    bad = np.zeros((2, 2, 3, n), dtype=np.uint64)
    bad[1, 1, 2, 5] = mods[2]  # one residue == its modulus: is_data_valid_for fails (valcheck.cpp:412-456)
    with pytest.raises(ValueError):
        ctx.load_key(bad)


@needs_ref
@pytest.mark.parametrize("n,mods_fn,t_bits,batch", [
    (4096, lambda: R.coeff_modulus_bfv_default(4096), 20, 3),            # BASELINE.json configs[0]
    (16384, lambda: R.coeff_modulus_create(16384, [54] * 8), 20, 2),     # configs[3] shape (BFV n=16384, 8 primes)
    (8192, lambda: R.coeff_modulus_create(8192, [60, 60, 60]), 30, 2),   # 60-bit primes: |B| grows to L+1 (rns.cpp:607-612)
])
def test_bfv_multiply_vs_reference(n, mods_fn, t_bits, batch):
    mods = mods_fn()
    t = R.plain_modulus_batching(n, t_bits)
    rb = R.RefContext(R.BFV, n, mods, t)
    ctx = sb().Context(sb().BFV, n, mods, t)
    rng = np.random.default_rng(n + 1)
    rk = ctx.load_key(rb.relin_key())
    for L in (len(mods) - 1, 1):
        assert ctx.base_bsk(L) == rb.base_bsk(L)
        a, b = rand_ct(rng, mods, n, 2, L, batch), rand_ct(rng, mods, n, 2, L, batch)
        m = ctx.multiply(a, b)
        mr = ctx.multiply_relinearize(a, b, rk)
        for i in range(batch):
            want = rb.multiply(L, a[i], b[i])
            assert (m[i] == want).all()
            assert (mr[i] == rb.relinearize(L, want)).all()


@needs_ref
def test_bfv_semantic_roundtrip():
    # the reference's own style of integration test (native/tests/seal/evaluator.cpp:1356 BFVEncryptMultiplyDecrypt,
    # :5670 BFVEncryptRotateMatrixDecrypt): encrypt with the reference, evaluate on the GPU, decrypt with the reference
    n = 4096
    mods = R.coeff_modulus_bfv_default(n)
    t = R.plain_modulus_batching(n, 20)
    rb = R.RefContext(R.BFV, n, mods, t)
    ctx = sb().Context(sb().BFV, n, mods, t)
    L = 2
    rng = np.random.default_rng(77)
    x, y = rng.integers(0, 1000, n, dtype=np.uint64), rng.integers(0, 1000, n, dtype=np.uint64)
    cx, cy = rb.bfv_encrypt(x), rb.bfv_encrypt(y)
    prod = ctx.multiply_relinearize(cx, cy, ctx.load_key(rb.relin_key()))
    got, budget = rb.bfv_decrypt(L, prod)
    assert budget > 0 and (got == (x * y) % np.uint64(t)).all()
    e = rb.galois_elt_from_step(3)
    rot = ctx.apply_galois(cx, e, ctx.load_key(rb.galois_key(e)))
    got, _ = rb.bfv_decrypt(L, rot)
    rows = x.reshape(2, n // 2)
    assert (got.reshape(2, n // 2) == np.roll(rows, -3, axis=1)).all()


@needs_ref
@pytest.mark.parametrize("scheme", ["ckks", "bfv"])
def test_linear_ops_and_square_vs_reference(scheme):
    # SURVEY 8(f) rank 1: add / sub / negate / square
    n, batch = 4096, 3
    mods = R.coeff_modulus_create(n, [50, 45, 60])
    t = R.plain_modulus_batching(n, 20) if scheme == "bfv" else 0
    sid = sb().BFV if scheme == "bfv" else sb().CKKS
    rc = R.RefContext(sid, n, mods, t)
    ctx = sb().Context(sid, n, mods, t)
    rng = np.random.default_rng(31)
    L = 2
    a, b = rand_ct(rng, mods, n, 2, L, batch), rand_ct(rng, mods, n, 2, L, batch)
    add, sub, neg, sq = ctx.add(a, b), ctx.sub(a, b), ctx.negate(a), ctx.square(a)
    for i in range(batch):
        assert (add[i] == rc.linear(0, L, a[i], b[i])).all()
        assert (sub[i] == rc.linear(1, L, a[i], b[i])).all()
        assert (neg[i] == rc.linear(2, L, a[i])).all()
        assert (sq[i] == rc.square(L, a[i])).all()
    # size-3 operands
    a3 = rand_ct(rng, mods, n, 3, L, batch)
    assert (ctx.add(a3, a3)[1] == rc.linear(0, L, a3[1], a3[1])).all()


@needs_ref
@pytest.mark.parametrize("scheme", ["ckks", "bfv"])
def test_multiply_plain_vs_reference(scheme):
    # SURVEY 8(f) rank 1: multiply_plain, NTT path (evaluator.cpp:2157-2195); one plaintext per ciphertext
    n, batch = 4096, 5
    mods = R.coeff_modulus_create(n, [50, 45, 60])
    t = R.plain_modulus_batching(n, 20) if scheme == "bfv" else 0
    sid = sb().BFV if scheme == "bfv" else sb().CKKS
    rc = R.RefContext(sid, n, mods, t)
    ctx = sb().Context(sid, n, mods, t)
    rng = np.random.default_rng(37)
    for L, size in ((2, 2), (2, 3), (1, 2)):
        a = rand_ct(rng, mods, n, size, L, batch)
        plain = rand_ct(rng, mods, n, 1, L, batch)[:, 0]
        got = ctx.multiply_plain(a, plain)
        for i in range(batch):
            assert (got[i] == rc.multiply_plain(L, a[i], plain[i])).all()
    # device entry point, in place
    import torch

    da = torch.from_numpy(a.view(np.int64)).cuda()
    dp = torch.from_numpy(np.ascontiguousarray(plain).view(np.int64)).cuda()
    ctx.d_multiply_plain(da, dp, da, L, size, batch)
    torch.cuda.synchronize()
    assert (da.cpu().numpy().view(np.uint64) == got).all()


@needs_ref
def test_dyadic_kernels_accept_unreduced_words_like_the_reference():
    """the reference's dyadic products (multiply_uint64 + barrett_reduce_128, util/uintarithsmallmod.h) accept any 64-bit operand
    words; a ciphertext or plaintext whose words are congruent but not reduced must give the reference's words here too (the
    kernels use a one-word Barrett step that presumes reduced operands, and reduce anything else on the way in)"""
    n, batch, L = 4096, 3, 2
    mods = R.coeff_modulus_create(n, [50, 45, 60])
    rc = R.RefContext(sb().CKKS, n, mods)
    ctx = sb().Context(sb().CKKS, n, mods)
    rng = np.random.default_rng(41)
    a, b = rand_ct(rng, mods, n, 2, L, batch), rand_ct(rng, mods, n, 2, L, batch)
    plain = rand_ct(rng, mods, n, 1, L, batch)[:, 0]
    ua, ub, up = a.copy(), b.copy(), plain.copy()
    for i in range(L):  # add multiples of the prime (still below 2^64) to a third of the words
        q = np.uint64(mods[i])
        for arr in (ua[:, :, i, :], ub[:, :, i, :], up[:, i, :]):
            mask = rng.integers(0, 3, arr.shape) == 0
            arr[mask] += q * np.uint64((2 ** 63 // mods[i]) - 1)
    assert (ua >= a).all() and (ua != a).any()
    got_m, got_s, got_p = ctx.multiply(ua, ub), ctx.square(ua), ctx.multiply_plain(ua, up)
    for i in range(batch):
        assert (got_m[i] == rc.multiply(L, a[i], b[i])).all()
        assert (got_m[i] == rc.multiply(L, ua[i], ub[i])).all(), "the reference itself is insensitive to the representative"
        assert (got_s[i] == rc.square(L, a[i])).all()
        assert (got_p[i] == rc.multiply_plain(L, a[i], plain[i])).all()


@needs_ref
@pytest.mark.parametrize("n,bits,t_bits,batch", [(4096, [50, 36, 45, 60], 20, 3), (4096, [50, 36, 45, 60], 38, 2),
                                                  (256, [40, 36, 42, 43], 17, 3), (16384, [54, 54, 54, 54, 54], 20, 2)])
def test_bgv_ops_vs_reference(n, bits, t_bits, batch):
    # SURVEY 8(f) rank 2: BGV -- bgv_multiply (evaluator.cpp:710-841), BGV mod-down of switch_key_inplace (:2762-2805),
    # mod_t_and_divide_q_last_ntt_inplace (rns.cpp:1193-1236); plain modulus below and above the smallest coefficient prime
    mods = R.coeff_modulus_create(n, bits)
    k = len(mods)
    t = R.plain_modulus_batching(n, t_bits)
    rc = R.RefContext(R.BGV, n, mods, t)
    ctx = sb().Context(sb().BGV, n, mods, t)
    rk = ctx.load_key(rc.relin_key())
    rng = np.random.default_rng(n + t_bits)
    for L in (k - 1, 2, 1):
        a, b = rand_ct(rng, mods, n, 2, L, batch), rand_ct(rng, mods, n, 2, L, batch)
        m = ctx.multiply(a, b)
        r = ctx.relinearize(m, rk)
        mr = ctx.multiply_relinearize(a, b, rk)
        for i in range(batch):
            assert (m[i] == rc.multiply(L, a[i], b[i])).all()
            assert (r[i] == rc.relinearize(L, m[i])).all()
        assert (mr == r).all()
        if L > 1:
            ms = ctx.mod_switch_to_next(a)
            for i in range(batch):
                assert (ms[i] == rc.mod_switch(L, a[i])).all()
            with pytest.raises(ValueError):
                ctx.rescale_to_next(a)  # evaluator.cpp:1533: unsupported operation for scheme type
        for step in (1, -2):
            e = rc.galois_elt_from_step(step)
            gk = ctx.load_key(rc.galois_key(e))
            g = ctx.rotate(a, step, gk)
            for i in range(batch):
                assert (g[i] == rc.rotate(L, a[i], step)).all()


@needs_ref
@pytest.mark.parametrize("scheme", ["ckks", "bfv", "bgv"])
def test_general_size_multiply_vs_reference(scheme):
    # SURVEY 8(a) a9/a10: the general-size branches of multiply (evaluator.cpp:524-560, :664-700, :796-833)
    n, batch = 4096, 3
    mods = R.coeff_modulus_create(n, [50, 45, 60, 55])
    sid = {"ckks": R.CKKS, "bfv": R.BFV, "bgv": R.BGV}[scheme]
    t = 0 if scheme == "ckks" else R.plain_modulus_batching(n, 20)
    rc = R.RefContext(sid, n, mods, t)
    ctx = sb().Context(sid, n, mods, t)
    rng = np.random.default_rng(43)
    for L, sa, sb_ in ((3, 3, 2), (2, 2, 3), (1, 3, 3), (2, 4, 2)):
        a, b = rand_ct(rng, mods, n, sa, L, batch), rand_ct(rng, mods, n, sb_, L, batch)
        got = ctx.multiply(a, b)
        assert got.shape == (batch, sa + sb_ - 1, L, n)
        for i in range(batch):
            assert (got[i] == rc.multiply(L, a[i], b[i])).all()
    with pytest.raises(ValueError):
        ctx.multiply(rand_ct(rng, mods, n, 9, 1, 1), rand_ct(rng, mods, n, 9, 1, 1))  # 17 polynomials > SEAL_CIPHERTEXT_SIZE_MAX


@needs_ref
@pytest.mark.parametrize("scheme", ["ckks", "bfv"])
def test_wire_format_vs_reference(scheme):
    # SURVEY 8(f) rank 3: Ciphertext::save / load (compr_mode none) between byte streams and device slabs
    import torch

    n, batch, L, size = 4096, 3, 2, 2
    mods = R.coeff_modulus_create(n, [50, 45, 60])
    sid = R.CKKS if scheme == "ckks" else R.BFV
    t = 0 if scheme == "ckks" else R.plain_modulus_batching(n, 20)
    rc = R.RefContext(sid, n, mods, t)
    ctx = sb().Context(sid, n, mods, t)
    for lv in (3, 2, 1):
        assert ctx.parms_id(lv) == rc.parms_id(lv)
    rng = np.random.default_rng(47)
    data = rand_ct(rng, mods, n, size, L, batch)
    ntt, scale = scheme == "ckks", (2.0 ** 40 if scheme == "ckks" else 1.0)
    streams = [rc.ct_save(L, data[i], ntt, scale) for i in range(batch)]
    dev = torch.zeros((batch, size, L, n), dtype=torch.int64, device="cuda")
    infos = ctx.d_load_ciphertexts(streams, dev, L, size)
    torch.cuda.synchronize()
    assert (dev.cpu().numpy().view(np.uint64) == data).all()
    assert all(i.is_ntt_form == int(ntt) and i.scale == scale for i in infos)
    # save: byte-identical to the reference's own stream, and the reference loads it back
    saved = ctx.d_save_ciphertexts(dev, L, size, batch, ntt, scale)
    assert saved == streams
    back, b_ntt, b_scale, b_cf = rc.ct_load(saved[1])
    assert (back == data[1]).all() and b_ntt == ntt and b_scale == scale and b_cf == 1
    # a pipeline that never leaves the device between load and save
    if scheme == "ckks":
        rk = ctx.load_key(rc.relin_key())
        out = torch.empty_like(dev)
        ctx.d_multiply_relinearize(dev, dev, rk, out, L, batch)
        res = ctx.d_save_ciphertexts(out, L, size, batch, True, scale * scale)
        got, _, g_scale, _ = rc.ct_load(res[0])
        assert (got == rc.multiply_relin(L, data[0], data[0])).all() and g_scale == scale * scale
    # keys from a serialized RelinKeys / GaloisKeys object (KSwitchKeys::load of one entry)
    m = ctx.multiply(data, data)
    rk_s = ctx.load_key_stream(rc.kswitch_keys_stream(0), 0)
    assert (ctx.relinearize(m, rk_s) == ctx.relinearize(m, ctx.load_key(rc.relin_key()))).all()
    e = rc.galois_elt_from_step(1)
    gk_s = ctx.load_key_stream(rc.kswitch_keys_stream(e), (e - 1) // 2)
    assert (ctx.apply_galois(data, e, gk_s)[0] == rc.apply_galois(L, data[0], e)).all()
    with pytest.raises(ValueError):
        ctx.load_key_stream(rc.kswitch_keys_stream(e), 0)  # empty slot
    with pytest.raises(IndexError):
        ctx.load_key_stream(rc.kswitch_keys_stream(0), 5)
    # KSwitchKeys::load ends in is_valid_for (kswitchkeys.cpp:149-153): one word >= its modulus makes the stream invalid
    ks = bytearray(rc.kswitch_keys_stream(0))
    words = np.frombuffer(bytes(ks), dtype=np.uint8)
    kdata = rc.relin_key()
    needle = kdata[0, 1, 0, :4].tobytes()  # the first words of digit 0, component 1, prime 0
    pos = bytes(ks).find(needle)
    assert pos > 0
    ks[pos:pos + 8] = int(mods[0]).to_bytes(8, "little")
    with pytest.raises(RuntimeError):
        ctx.load_key_stream(bytes(ks), 0)
    # Ciphertext::load rejects residues >= q_i (is_data_valid_for); unsafe_load does not look
    bad = bytearray(streams[0])
    off = infos[0].data_offset
    bad[off:off + 8] = int(mods[0]).to_bytes(8, "little")
    with pytest.raises(RuntimeError):
        ctx.d_load_ciphertexts([bytes(bad)], dev, L, size)
    ctx.d_load_ciphertexts([bytes(bad)], dev, L, size, validate=False)
    # a stream of another level / another context
    with pytest.raises(RuntimeError):
        ctx.d_load_ciphertexts([rc.ct_save(1, data[0][:, :1], ntt, scale)], dev, L, size)
    # a seed-compressed fresh ciphertext lives at the first data level (2 primes here): loads there, not at level 1
    one = torch.zeros((1, 2, 2, n), dtype=torch.int64, device="cuda")
    ctx.d_load_ciphertexts([rc.seeded_ct_stream()], one, 2, 2)
    torch.cuda.synchronize()
    assert (one.cpu().numpy().view(np.uint64)[0] == rc.ct_load(rc.seeded_ct_stream())[0]).all()
    with pytest.raises(RuntimeError):
        ctx.d_load_ciphertexts([rc.seeded_ct_stream()], torch.zeros((1, 2, 1, n), dtype=torch.int64, device="cuda"), 1, 2)


@needs_ref
@pytest.mark.parametrize("scheme,n,bits", [("ckks", 8192, [55, 55, 55, 55]), ("ckks", 4096, [60, 60, 60]), ("bfv", 4096, [36, 36, 37]),
                                          ("ckks", 32768, [55] * 4)])
def test_seeded_ciphertext_expansion_vs_reference(scheme, n, bits):
    """Ciphertext::load of seed-compressed streams (symmetric-key encryptions saved with their second polynomial as a PRNG seed):
    c_0 is uploaded, c_1 is re-created on the device (BLAKE2Xb stream + sample_poly_uniform's rejection sampling, sb_prng.cu) and
    must equal what the reference's own load produces, word for word; 60-bit primes make rejections frequent (~2^-4 per word)"""
    import torch

    mods = R.coeff_modulus_create(n, bits)
    t = R.plain_modulus_batching(n, 20) if scheme == "bfv" else 0
    sid = R.BFV if scheme == "bfv" else R.CKKS
    rc = R.RefContext(sid, n, mods, t)
    ctx = sb().Context(sid, n, mods, t)
    oc = O.Oracle(O.BFV if scheme == "bfv" else O.CKKS, n, mods, t)
    L = len(mods) - 1 if len(mods) > 1 else 1
    seeded = [rc.seeded_ct_stream() for _ in range(3)]
    full = [rc.ct_load(s)[0] for s in seeded]
    assert full[0].shape == (2, L, n)
    # a mixed batch: seeded, plain (re-saved by the reference), seeded, seeded
    plain_stream = rc.ct_save(L, full[1], scheme != "bfv", 1.0)
    streams = [seeded[0], plain_stream, seeded[1], seeded[2]]
    want = [full[0], full[1], full[1], full[2]]
    dev = torch.zeros((4, 2, L, n), dtype=torch.int64, device="cuda")
    infos = ctx.d_load_ciphertexts(streams, dev, L, 2)
    torch.cuda.synchronize()
    got = dev.cpu().numpy().view(np.uint64)
    assert [i.seeded for i in infos] == [1, 0, 1, 1]
    for g, w in zip(got, want):
        assert (g == w).all()
    seed = np.frombuffer(seeded[0], dtype=np.uint64, count=8, offset=infos[0].seed_offset)
    assert (oc.expand_seed(L, seed) == got[0][1]).all()  # and the oracle's restatement agrees
    # the same objects saved with compr_mode_type::zlib (the reference's default when it is built with zlib): inflated on the host,
    # then the same path; a key-switching key object too
    zstreams = [rc.seeded_ct_stream(compr=1), rc.ct_save(L, full[1], scheme != "bfv", 1.0, compr=1)]
    zwant = [rc.ct_load(zstreams[0])[0], full[1]]
    zdev = torch.zeros((2, 2, L, n), dtype=torch.int64, device="cuda")
    zinfos = ctx.d_load_ciphertexts(zstreams, zdev, L, 2)
    torch.cuda.synchronize()
    assert [(i.compr_mode, i.seeded) for i in zinfos] == [(1, 1), (1, 0)]
    for g, w in zip(zdev.cpu().numpy().view(np.uint64), zwant):
        assert (g == w).all()
    if scheme == "ckks" and n == 8192:
        m = ctx.multiply(full[:1], full[:1])
        rk_z = ctx.load_key_stream(rc.kswitch_keys_stream(0, compr=1), 0)
        assert (ctx.relinearize(m, rk_z) == ctx.relinearize(m, ctx.load_key(rc.relin_key()))).all()


@needs_ref
@pytest.mark.parametrize("scheme,t_bits,n", [("bfv", 20, 4096), ("bfv", 38, 4096), ("bgv", 20, 4096), ("bgv", 38, 256)])
def test_coeff_plain_ops_vs_reference(scheme, t_bits, n):
    # coefficient-form plaintexts (BFV / BGV): transform_to_ntt(Plaintext), multiply_plain, add_plain, sub_plain
    batch = 3
    mods = R.coeff_modulus_create(n, [50, 36, 45, 60])
    t = R.plain_modulus_batching(n, t_bits)
    sid = R.BFV if scheme == "bfv" else R.BGV
    rc = R.RefContext(sid, n, mods, t)
    ctx = sb().Context(sid, n, mods, t)
    rng = np.random.default_rng(59)
    ntt = scheme == "bgv"
    for L, size in ((3, 2), (1, 3)):
        plain = rng.integers(0, t, (batch, n), dtype=np.uint64)
        plain[:, :4] = [0, t - 1, (t + 1) // 2, (t + 1) // 2 - 1]
        a = rand_ct(rng, mods, n, size, L, batch)
        pn = ctx.plain_to_ntt(plain, L)
        mp = ctx.multiply_plain_coeff(a, plain, ntt)
        cf = None if scheme == "bfv" else np.array([1, 12345 % t, t - 1], dtype=np.uint64)
        ap = ctx.add_plain_coeff(a, plain, False, cf)
        sp = ctx.add_plain_coeff(a, plain, True, cf)
        for i in range(batch):
            f = 1 if cf is None else int(cf[i])
            assert (pn[i] == rc.plain_to_ntt(L, plain[i])).all()
            assert (mp[i] == rc.plain_op_coeff(0, L, a[i], plain[i], ntt)).all()
            assert (ap[i] == rc.plain_op_coeff(1, L, a[i], plain[i], ntt, f)).all()
            assert (sp[i] == rc.plain_op_coeff(2, L, a[i], plain[i], ntt, f)).all()
        if scheme == "bfv":  # transformed BFV ciphertext: the NTT branch of multiply_plain
            mn = ctx.multiply_plain_coeff(a, plain, True)
            assert (mn[0] == rc.plain_op_coeff(0, L, a[0], plain[0], True)).all()


@needs_ref
@pytest.mark.parametrize("n,t_bits", [(256, 20), (4096, 20), (8192, 44)])
def test_batch_codec_vs_reference(n, t_bits):
    # SURVEY 8(f) rank 4: BatchEncoder::encode / decode (batchencoder.cpp:84-330) as a transform modulo t
    batch = 3
    mods = R.coeff_modulus_create(n, [50, 45, 60])
    t = R.plain_modulus_batching(n, t_bits)
    rc = R.RefContext(R.BFV, n, mods, t)
    ctx = sb().Context(sb().BFV, n, mods, t)
    rng = np.random.default_rng(67)
    v = rng.integers(0, t, (batch, n), dtype=np.uint64)
    p = ctx.batch_encode(v)
    w = rng.integers(0, t, (batch, n), dtype=np.uint64)
    d = ctx.batch_decode(w)
    for i in range(batch):
        assert (p[i] == rc.batch_codec(v[i], False)).all()
        assert (d[i] == rc.batch_codec(w[i], True)).all()
    assert (ctx.batch_decode(p) == v).all()
    # a plain modulus that does not support batching
    ctx2 = sb().Context(sb().BFV, n, mods, 1 << 20)
    with pytest.raises(ValueError):
        ctx2.batch_encode(v % (1 << 20))


@needs_ref
@pytest.mark.parametrize("scheme,n", [("ckks", 4096), ("bfv", 4096), ("bgv", 4096), ("bfv", 256), ("bgv", 256)])
def test_decrypt_vs_reference(scheme, n):
    # SURVEY 8(f) rank 4: Decryptor::decrypt (decryptor.cpp:62-197) -- phase, then scale-and-round (BFV), exact base
    # conversion in IEEE doubles (BGV) or nothing (CKKS); uniform-random ciphertexts reach every branch
    batch = 3
    mods = R.coeff_modulus_create(n, [50, 45, 60, 55])
    sid = {"ckks": R.CKKS, "bfv": R.BFV, "bgv": R.BGV}[scheme]
    t = 0 if scheme == "ckks" else R.plain_modulus_batching(n, 20)
    rc = R.RefContext(sid, n, mods, t)
    ctx = sb().Context(sid, n, mods, t)
    sk = ctx.load_secret_key(rc.secret_key())
    rng = np.random.default_rng(73)
    ntt = scheme != "bfv"
    for L, size in ((3, 2), (2, 3), (1, 2), (3, 4)):
        ct = rand_ct(rng, mods, n, size, L, batch)
        cf = np.array([1, 12345, t - 1], dtype=np.uint64) if scheme == "bgv" else None
        got = ctx.decrypt(ct, sk, cf)
        for i in range(batch):
            f = 1 if cf is None else int(cf[i])
            assert (got[i] == rc.decrypt(L, ct[i], ntt, f)).all()
    if scheme == "bfv":  # a real encryption comes back: decrypt + decode on the device
        slots = rng.integers(0, t, n, dtype=np.uint64)
        p = ctx.decrypt(rc.bfv_encrypt(slots), sk)
        assert (ctx.batch_decode(p) == slots).all()


_INVALID, _BATCH = "encrypted is not valid for encryption parameters", "batch must be positive"
# status and sb200_last_error() text of both entry points of a pair, per bad argument (pointer errors: the status only)
_ABI_ERRORS = {
    "null context": (-6, None),
    "null a": (-6, None),
    "null b": (-6, None),
    "null out": (-6, None),
    "null key": (-6, None),
    "L = 0": (-1, _INVALID),
    "L = k + 1": (-1, _INVALID),
    "L = k": (-1, _INVALID),  # key switching: the key level carries no data
    "batch = 0": (-1, _BATCH),
}
_ABI_BAD_SIZE = {  # the invalid size of each pair that takes one (the NTT transforms any number of polynomials)
    "multiply_sized": ({"size_a": 1}, "invalid ciphertext sizes"),
    "add": ({"size": 0}, _INVALID), "sub": ({"size": 0}, _INVALID), "negate": ({"size": 0}, _INVALID),
    "multiply_plain": ({"size": 0}, _INVALID), "multiply_plain_coeff": ({"size": 0}, _INVALID),
    "add_plain_coeff": ({"size": 0}, _INVALID), "decrypt": ({"size": 0}, _INVALID),
    "rescale_to_next_sized": ({"size": 0}, "invalid ciphertext size"), "mod_switch_to_next_sized": ({"size": 0}, "invalid ciphertext size"),
    "relinearize_sized": ({"size": 0}, "invalid ciphertext size"),
}
_ABI_ALIAS = {  # stream entry points that refuse an output slab aliasing an input slab (host buffers are staged apart)
    "multiply_sized": "multiply: the output slab must not alias an input slab",
    "relinearize": "relinearize: input and output slabs must not alias (different layouts)",
    "relinearize_sized": "relinearize: input and output slabs must not alias",
    "rescale_to_next": "rescale_to_next: input and output slabs must not alias (different layouts)",
    "rescale_to_next_sized": "rescale_to_next: input and output slabs must not alias (different layouts)",
    "mod_switch_to_next": "mod_switch_to_next: input and output slabs must not alias (different layouts)",
    "mod_switch_to_next_sized": "mod_switch_to_next: input and output slabs must not alias (different layouts)",
    "apply_galois": "apply_galois: in and out must not alias",
    "batch_encode": "batch_encode: input and output must not alias",
    "batch_decode": "batch_decode: input and output must not alias",
}
_END_OF_CHAIN = "end of modulus switching chain reached"


def _abi_error_cases(name, k):
    """(case, argument changes, expected status, expected text, variants) of one pair"""
    order = ABI_PAIRS[name]
    ks = name in ("relinearize", "multiply_relinearize", "relinearize_sized", "apply_galois")
    cases = [("null context", {}, "both")]
    cases += [(f"null {p}", {p: None}, "both") for p in ("a", "b", "out", "key") if p in order]
    if "L" in order:
        cases += [("L = 0", {"L": 0}, "both"), ("L = k", {"L": k}, "both") if ks else ("L = k + 1", {"L": k + 1}, "both")]
    cases.append(("batch = 0", {"batch": 0}, "both"))
    out = []
    for case, change, variants in cases:
        status, text = _ABI_ERRORS[case]
        if name == "ckks_encode" and case == "null a":  # values may be null for an empty vector: not a pointer error
            status, text = -1, "values cannot be null"
        out.append((case, change, status, text, variants))
    if name in _ABI_BAD_SIZE:
        out.append(("invalid size", _ABI_BAD_SIZE[name][0], -1, _ABI_BAD_SIZE[name][1], "both"))
    if name in _ABI_ALIAS:
        out.append(("aliased slabs", {"out": "a"}, -1, _ABI_ALIAS[name], "stream"))
    if name == "ckks_encode":
        out.append(("count = 0, null values", {"count": 0, "a": None}, 0, None, "both"))
    if name in ("rescale_to_next", "mod_switch_to_next", "rescale_to_next_sized", "mod_switch_to_next_sized"):
        out.append(("L = 1", {"L": 1}, -1, _END_OF_CHAIN, "both"))
    return out


@pytest.mark.parametrize("name", list(ABI_PAIRS))
def test_c_abi_argument_errors_of_every_pair(name):
    """the table above for both entry points of `name`: every bad argument gets the same status (and text) from both"""
    import torch

    S = sb()
    n, k = 256, 3
    mods = S.coeff_modulus_create(n, [40, 40, 40])
    scheme = S.BFV if _PAIR_SCHEMES.get(name, "ckks").split()[0] == "bfv" else S.CKKS
    ctx = S.Context(scheme, n, mods, 65537 if scheme == S.BFV else 0)
    rng = np.random.default_rng(3)
    key = ctx.load_key(rng.integers(0, 1 << 39, (2, 2, k, n), dtype=np.uint64))
    sk = ctx.load_secret_key(rng.integers(0, 1 << 39, (k, n), dtype=np.uint64))
    words = 2 * 16 * k * n
    host = {f: np.zeros(words, dtype=np.uint64) for f in ("a", "b", "out")}
    dev = {f: torch.zeros(words, dtype=torch.int64, device="cuda") for f in ("a", "b", "out")}
    base = dict(L=2, size=3 if name == "relinearize_sized" else 2, size_a=2, size_b=2, batch=1, flag=1, elt=3, count=4, scale=2.0 ** 20,
                cf=None, key=sk.h if name == "decrypt" else key.h)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    bad = []
    for case, change, status, text, variants in _abi_error_cases(name, k):
        for variant in ("host", "stream") if variants == "both" else (variants,):
            bufs = host if variant == "host" else dev
            v = dict(base, **{f: C.c_void_p(x.ctypes.data if variant == "host" else x.data_ptr()) for f, x in bufs.items()})
            v.update({f: (v[x] if x in ("a", "b", "out") else x) if isinstance(x, str) else x for f, x in change.items()})
            ctx_h = None if case == "null context" else ctx.h
            got = abi_call(ctx_h, name, v, None if variant == "host" else stream)
            torch.cuda.synchronize()
            if got[0] != status or (text is not None and got[1] != text):
                bad.append(f"{name} {variant} [{case}]: got {got}, want ({status}, {text!r})")
    assert not bad, "\n".join(bad)


def test_rescale_at_the_last_level_of_a_bfv_context():
    """both entry points report the end of the modulus switching chain before the scheme (evaluator.cpp:1521 precedes :1533)"""
    import torch

    S = sb()
    n = 256
    ctx = S.Context(S.BFV, n, S.coeff_modulus_create(n, [40, 40, 40]), 65537)
    a, out = np.zeros(2 * n, dtype=np.uint64), np.zeros(2 * n, dtype=np.uint64)
    da, dout = torch.zeros(2 * n, dtype=torch.int64, device="cuda"), torch.zeros(2 * n, dtype=torch.int64, device="cuda")
    for name in ("rescale_to_next", "rescale_to_next_sized"):
        v = dict(L=1, size=2, batch=1, a=a.ctypes.data_as(C.c_void_p), out=out.ctypes.data_as(C.c_void_p))
        assert abi_call(ctx.h, name, v) == (-1, _END_OF_CHAIN)
        v.update(a=C.c_void_p(da.data_ptr()), out=C.c_void_p(dout.data_ptr()))
        rc, text = abi_call(ctx.h, name, v, C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == -1 and text in (_END_OF_CHAIN, "unsupported operation for scheme type")


def test_c_abi_pointer_and_argument_errors():
    # the reference's C layer rejects null handles with E_POINTER (native/tests/seal/cabi.cpp:339-425); same here
    s = sb()
    lib = s.lib()
    null = C.c_void_p(None)
    buf = np.zeros(8, dtype=np.uint64)
    assert lib.sb200_ntt_forward_host(null, 1, 1, 1, s._hp(buf)) == -6
    h = C.c_void_p()
    assert lib.sb200_context_create(2, 1024, None, 1, 0, 0, C.byref(h)) == -6
    n = 1024
    mods = O.coeff_modulus_create(n, [40, 40])
    ctx = s.Context(s.CKKS, n, mods)
    assert lib.sb200_multiply_host(ctx.h, 1, 1, None, s._hp(buf), s._hp(buf)) == -6
    assert lib.sb200_ntt_forward_host(ctx.h, 5, 1, 1, s._hp(buf)) == -1       # no such level
    assert b"not valid" in lib.sb200_last_error()
    assert lib.sb200_ntt_forward_host(ctx.h, 1, 1, 0, s._hp(buf)) == -1       # empty batch
    with pytest.raises(ValueError):
        s.Context(s.CKKS, n, mods, device=99)
    # BEHZ queries on a CKKS context are a logic error, like RNSTool without a plain modulus
    cnt = C.c_size_t(0)
    assert lib.sb200_get_base_bsk(ctx.h, 1, s._hp(buf), 8, C.byref(cnt)) == -2


@pytest.mark.parametrize("logn,scheme", [(17, "ckks"), (15, "bfv"), (11, "ckks")])
def test_keyswitch_extreme_sizes_vs_oracle(logn, scheme):
    # n = 131072 is SEAL_POLY_MOD_DEGREE_MAX (util/defines.h:52); n = 2048 is the largest size on the one-CTA-per-row path
    n = 1 << logn
    bits = [50, 45, 55] if scheme == "ckks" else [48, 48, 49]
    mods = O.coeff_modulus_create(n, bits)
    t = 0
    if scheme == "bfv":
        t = next(p for p in range((1 << 20) + 1, 1 << 21, 2 * n) if O.lib().orc_is_prime(p))  # prime = 1 mod 2n
    sid = sb().BFV if scheme == "bfv" else sb().CKKS
    ctx = sb().Context(sid, n, mods, t)
    oc = O.Oracle(sid, n, mods, t)
    rng = np.random.default_rng(logn)
    L, k = 2, 3
    key = np.stack([np.stack([np.stack([rng.integers(0, mods[i], n, dtype=np.uint64) for i in range(k)]) for _ in range(2)]) for _ in range(L)])
    rk = ctx.load_key(key)
    a, b = rand_ct(rng, mods, n, 2, L, 2), rand_ct(rng, mods, n, 2, L, 2)
    got = ctx.multiply_relinearize(a, b, rk)
    assert (got[1] == oc.multiply_relin(L, a[1], b[1], key)).all()
    e = O.galois_elt_from_step(n, 1)
    assert (ctx.apply_galois(a, e, rk)[0] == oc.apply_galois(L, a[0], e, key)).all()
    if scheme == "ckks":
        assert (ctx.rescale_to_next(a)[1] == oc.rescale(L, a[1])).all()
    else:
        assert (ctx.mod_switch_to_next(a)[1] == oc.bfv_mod_switch(L, a[1])).all()


@needs_ref
@pytest.mark.parametrize("scheme,n,bits", [("ckks", 8192, [50, 50, 50, 51]), ("bfv", 4096, [36, 36, 37]), ("bgv", 4096, [40, 40, 40]),
                                          ("ckks", 2048, [54])])
def test_encrypt_zero_symmetric_vs_reference(scheme, n, bits):
    """sb200_encrypt_zero_symmetric against Encryptor::encrypt_zero_symmetric of the reference with the same bootstrap seed (the
    reference context's generator factory is seeded): the plain variant, the seed-keeping variant (the reference's seeded stream,
    loaded by the reference), a lower level, and other seeds of the batch against the oracle; the ciphertexts decrypt to the noise"""
    import torch

    def to_np(x):
        return x.cpu().numpy().view(np.uint64)

    S = sb()
    sid = {"ckks": (R.CKKS, S.CKKS, O.CKKS), "bfv": (R.BFV, S.BFV, O.BFV), "bgv": (R.BGV, S.BGV, O.BGV)}[scheme]
    mods = R.coeff_modulus_create(n, bits)
    t = R.plain_modulus_batching(n, 20) if scheme != "ckks" else 0
    seed0 = 0xC0FFEE
    rc = R.RefContext(sid[0], n, mods, t, seed=seed0)
    oc = O.Oracle(sid[2], n, mods, t)
    ctx = S.Context(sid[1], n, mods, t)
    sk_host = rc.secret_key()
    sk = ctx.load_secret_key(sk_host)
    k = len(mods)
    L = k - 1 if k > 1 else 1
    batch = 3
    seeds = np.zeros((batch, 8), dtype=np.uint64)
    seeds[0, 0] = seed0
    seeds[1] = np.arange(1, 9, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    seeds[2, 7] = 5
    for save_seed in (False, True):
        out = torch.zeros((batch, 2, L, n), dtype=torch.int64, device="cuda")
        pub = ctx.d_encrypt_zero_symmetric(sk, out, L, batch, seeds, save_seed=save_seed, want_public_seeds=True)
        torch.cuda.synchronize()
        got = to_np(out)
        if save_seed:
            want0, _, _, _ = rc.ct_load(rc.seeded_ct_stream())
        else:
            want0 = rc.encrypt_zero_symmetric()
        assert (got[0] == want0).all(), f"ciphertext 0 vs the reference, save_seed={save_seed}"
        for b in range(batch):
            assert (got[b] == oc.encrypt_zero_symmetric(sk_host, seeds[b], save_seed)).all(), f"ciphertext {b} vs the oracle"
            assert (pub[b] == oc.blake2xb_stream(seeds[b], 8)).all()
    if k > 2:
        out = torch.zeros((1, 2, 1, n), dtype=torch.int64, device="cuda")
        ctx.d_encrypt_zero_symmetric(sk, out, 1, 1, seeds[:1])
        torch.cuda.synchronize()
        assert (to_np(out)[0] == rc.encrypt_zero_symmetric(L=1)).all()
    # fresh seeds: two calls differ, and c_0 + c_1 s is small (the noise) -- checked through the library's own decryption
    a = torch.zeros((2, 2, L, n), dtype=torch.int64, device="cuda")
    ctx.d_encrypt_zero_symmetric(sk, a, L, 2)
    torch.cuda.synchronize()
    ha = to_np(a)
    assert not (ha[0] == ha[1]).all()
    if scheme == "bfv":
        assert (ctx.decrypt(ha, sk) == 0).all()


@pytest.mark.parametrize("n,bits", [(8192, [60, 60, 60, 60]), (4096, [40, 40, 40]), (1024, [27]), (65536, [55] * 5)])
def test_ckks_encoder_vs_reference(n, bits):
    """sb200_ckks_encode / sb200_ckks_decode BIT-exact against CKKSEncoder of the reference (or the oracle pinned to it, where the
    reference library is absent): batches, partial vectors, real input, every decomposition branch (coefficients below 2^64, below
    2^128, multi-precision), a lower level, the reference's error cases, and decode of encoded and of arbitrary plaintexts"""
    S = sb()
    mods = O.coeff_modulus_create(n, bits)
    oc = O.Oracle(O.CKKS, n, mods)
    rc = R.RefContext(R.CKKS, n, mods) if R.available() else oc
    ctx = S.Context(S.CKKS, n, mods)
    k = len(mods)
    Lmax = k - 1 if k > 1 else 1
    rng = np.random.default_rng(11)
    slots = n // 2
    total = sum(bits[:Lmax])
    cases = [(Lmax, slots, 2.0 ** 20, 1.0), (Lmax, slots // 3, 2.0 ** 30, 100.0), (1, slots, 2.0 ** 10, 1e-3), (Lmax, 1, 3.7e5, 1.0)]
    if total > 70:
        cases.append((Lmax, slots, 2.0 ** 62, 50.0))
    if total > 140:
        cases.append((Lmax, slots, 2.0 ** 120, 1000.0))
    B = 3
    for L, count, scale, mag in cases:
        v = (rng.standard_normal((B, count)) + 1j * rng.standard_normal((B, count))) * mag
        if rc.ckks_encode(L, v[0], scale) is None:
            # the reference rejects the case (a scale wider than the level's modulus): the same error, not a result
            with pytest.raises(ValueError, match="scale out of bounds|encoded values are too large"):
                ctx.ckks_encode(v, L, scale)
            continue
        got = ctx.ckks_encode(v, L, scale)
        for b in range(B):
            want = rc.ckks_encode(L, v[b], scale)
            assert want is not None
            assert (got[b] == want).all(), ("encode", L, count, scale, b)
        dec = ctx.ckks_decode(got, scale)
        for b in (0, B - 1):
            want = rc.ckks_decode(L, got[b], scale)
            assert (dec[b].view(np.uint64) == want.view(np.uint64)).all(), ("decode", L, count, scale, b)
    # real input = complex input with zero imaginary parts
    r = rng.standard_normal(slots)
    assert (ctx.ckks_encode(r, Lmax, 2.0 ** 20) == rc.ckks_encode(Lmax, r + 0j, 2.0 ** 20)).all()
    # empty vector: the zero plaintext
    assert (ctx.ckks_encode(np.zeros((1, 0), dtype=np.complex128), Lmax, 2.0 ** 20) == 0).all()
    # decode of arbitrary plaintexts (uniform residues: coefficients in both halves of [0, Q))
    for L in sorted({1, Lmax}):
        p = np.stack([rng.integers(0, mods[j], n, dtype=np.uint64) for j in range(L)])
        for scale in (2.0 ** 12, 2.0 ** 30):
            want = rc.ckks_decode(L, p, scale)
            if want is None:
                with pytest.raises(ValueError, match="scale out of bounds"):
                    ctx.ckks_decode(p, scale)
            else:
                assert (ctx.ckks_decode(p, scale).view(np.uint64) == want.view(np.uint64)).all(), ("decode random", L, scale)
    # the reference's invalid_argument cases
    with pytest.raises(ValueError, match="encoded values are too large"):
        ctx.ckks_encode(np.full(slots, 1e30 + 0j), 1, 2.0 ** 20)
    with pytest.raises(ValueError, match="values must be finite"):
        ctx.ckks_encode(np.array([np.inf + 0j]), 1, 2.0 ** 20)
    with pytest.raises(ValueError, match="scale out of bounds"):
        ctx.ckks_encode(np.ones(4) + 0j, 1, 2.0 ** 200)
    with pytest.raises(ValueError, match="values_size is too large"):
        ctx.ckks_encode(np.ones(slots + 1) + 0j, 1, 2.0 ** 20)
    bfv = S.Context(S.BFV, 4096, O.coeff_modulus_create(4096, [36, 36, 37]), 65537)
    with pytest.raises(ValueError, match="unsupported scheme"):
        bfv.ckks_encode(np.ones(4) + 0j, 1, 2.0 ** 20)


@needs_ref
@pytest.mark.parametrize("scheme,n,bits", [("ckks", 8192, [50, 50, 50, 51]), ("bfv", 4096, [36, 36, 37]), ("bgv", 4096, [40, 40, 40]),
                                          ("ckks", 2048, [54])])
def test_encrypt_zero_asymmetric_vs_reference(scheme, n, bits):
    """sb200_encrypt_zero_asymmetric against Encryptor(public key)::encrypt_zero of the reference with the same PRNG seed: first data
    level, the lowest level, the key level; other seeds of the batch against the oracle (incl. a stream whose ternary words contain
    a zero word is covered by the oracle-level restatement only: probability 2^-32 per coefficient); decrypts to zero"""
    import torch

    def to_np(x):
        return x.cpu().numpy().view(np.uint64)

    S = sb()
    sid = {"ckks": (R.CKKS, S.CKKS, O.CKKS), "bfv": (R.BFV, S.BFV, O.BFV), "bgv": (R.BGV, S.BGV, O.BGV)}[scheme]
    mods = R.coeff_modulus_create(n, bits)
    t = R.plain_modulus_batching(n, 20) if scheme != "ckks" else 0
    seed0 = 0xC0FFEE
    rc = R.RefContext(sid[0], n, mods, t, seed=seed0)
    oc = O.Oracle(sid[2], n, mods, t)
    ctx = S.Context(sid[1], n, mods, t)
    pk_host = rc.public_key()
    pk = ctx.load_public_key(pk_host)
    k = len(mods)
    batch = 3
    seeds = np.zeros((batch, 8), dtype=np.uint64)
    seeds[0, 0] = seed0
    seeds[1] = np.arange(1, 9, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    seeds[2, 3] = 77
    for L in sorted({k - 1 if k > 1 else 1, 1, k}):
        out = torch.zeros((batch, 2, L, n), dtype=torch.int64, device="cuda")
        ctx.d_encrypt_zero_asymmetric(pk, out, L, batch, seeds)
        torch.cuda.synchronize()
        got = to_np(out)
        assert (got[0] == rc.encrypt_zero_asymmetric(L=L)).all(), f"level {L} vs the reference"
        for b in range(1, batch):
            assert (got[b] == oc.encrypt_zero_asymmetric(pk_host, seeds[b], L=L)).all(), f"level {L}, ciphertext {b} vs the oracle"
    L = k - 1 if k > 1 else 1
    a = torch.zeros((2, 2, L, n), dtype=torch.int64, device="cuda")
    ctx.d_encrypt_zero_asymmetric(pk, a, L, 2)
    torch.cuda.synchronize()
    ha = to_np(a)
    assert not (ha[0] == ha[1]).all()
    if scheme == "bfv":
        sk = ctx.load_secret_key(rc.secret_key())
        assert (ctx.decrypt(ha, sk) == 0).all()
    bad = pk_host.copy()
    bad[1, 0, 5] = mods[0]
    with pytest.raises(ValueError, match="public key is not valid"):
        ctx.load_public_key(bad)
