"""Seed-compressed streams written on an H100 (-m gpu): sb200_public_key_generate_seeded, sb200_kswitch_keys_generate_seeded and
sb200_ciphertext_save_seeded against the bytes the reference's Serializable<...>::save(compr_mode_type::none) writes under seeded
Blake2xb / Shake256 factories (oracle/ref_serial.cpp); the size functions; chunking; round trips through the device's and the
reference's loaders; ciphertext_prng = 2 against tests/refprng.py; the argument errors; and the C++ Serializable overloads
(tests/cpp/shim_serial_test.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import keygen_ref as K
import oracle as O
import refprng as P
import refseal as R

pytestmark = pytest.mark.gpu
_REF = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref", "libsealref_serial.so")
needs_ref = pytest.mark.skipif(not os.path.exists(_REF), reason="oracle/_ref/libsealref_serial.so not present (oracle/serial.mk)")
_u64p = C.POINTER(C.c_uint64)
_lib = None


def ref():
    global _lib
    if _lib is None:
        L = C.CDLL(_REF)
        vp, sz, u8p = C.c_void_p, C.c_size_t, C.c_char_p
        L.refser_last_error.restype = C.c_char_p
        L.refser_create.restype = vp
        L.refser_create.argtypes = [C.c_int, sz, _u64p, sz, C.c_uint64, C.c_uint64, C.c_int]
        L.refser_destroy.argtypes = [vp]
        L.refser_secret_key.argtypes = [vp, _u64p]
        for f in ("refser_public_key", "refser_relin_keys"):
            getattr(L, f).restype = C.c_long
            getattr(L, f).argtypes = [vp, vp, sz]
        L.refser_galois_keys.restype = C.c_long
        L.refser_galois_keys.argtypes = [vp, C.POINTER(C.c_uint32), sz, C.c_int, vp, sz]
        L.refser_encrypt_symmetric.restype = C.c_long
        L.refser_encrypt_symmetric.argtypes = [vp, sz, _u64p, C.c_double, vp, sz]
        L.refser_encrypt_zero_symmetric.restype = C.c_long
        L.refser_encrypt_zero_symmetric.argtypes = [vp, sz, vp, sz]
        L.refser_load_ciphertext.restype = C.c_long
        L.refser_load_ciphertext.argtypes = [vp, u8p, sz, _u64p, sz]
        L.refser_load_public_key.restype = C.c_long
        L.refser_load_public_key.argtypes = [vp, u8p, sz, _u64p]
        L.refser_load_kswitch.restype = C.c_long
        L.refser_load_kswitch.argtypes = [vp, u8p, sz, C.c_uint32, _u64p]
        _lib = L
    return _lib


def _p(a):
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(_u64p)


class Ref:
    """the reference's KeyGenerator and symmetric Encryptor under a fixed-seed factory: every bootstrap seed is {seed, 0, ...}"""

    def __init__(self, scheme, n, mods, t, prng, seed=0x5E71A1):
        self.n, self.k, self.mods, self.seed = n, len(mods), list(mods), seed
        m = np.array(mods, dtype=np.uint64)
        self.h = ref().refser_create(scheme, n, _p(m), self.k, t, seed, prng)
        assert self.h, ref().refser_last_error().decode()

    def __del__(self):
        if getattr(self, "h", None):
            ref().refser_destroy(self.h)

    def _bytes(self, fn, *args):
        size = fn(self.h, *args, None, 0)
        assert size >= 0, ref().refser_last_error().decode()
        buf = C.create_string_buffer(size)
        got = fn(self.h, *args, C.addressof(buf), size)
        assert got == size, ref().refser_last_error().decode()
        return buf.raw

    def secret_key(self):
        out = np.zeros((self.k, self.n), dtype=np.uint64)
        assert ref().refser_secret_key(self.h, _p(out)) == 0
        return out

    def seeds(self, count):
        s = np.zeros((count, 8), dtype=np.uint64)
        s[:, 0] = self.seed
        return s

    # every call below draws from the factory; with a fixed seed each draw is the same, so calls may come in any order
    def public_key(self):
        return self._bytes(ref().refser_public_key)

    def relin_keys(self):
        return self._bytes(ref().refser_relin_keys)

    def galois_keys(self, elts=None):
        e = (C.c_uint32 * max(len(elts or []), 1))(*(elts or []))
        return self._bytes(ref().refser_galois_keys, e, len(elts or []), int(elts is None))

    def encrypt_symmetric(self, L, plain, scale=1.0):
        return self._bytes(ref().refser_encrypt_symmetric, L, _p(np.ascontiguousarray(plain, dtype=np.uint64)), scale)

    def encrypt_zero_symmetric(self, L):
        return self._bytes(ref().refser_encrypt_zero_symmetric, L)

    def load_ciphertext(self, stream, L):
        out = np.zeros(2 * L * self.n, dtype=np.uint64)
        got = ref().refser_load_ciphertext(self.h, stream, len(stream), _p(out), out.size)
        assert got == out.size, ref().refser_last_error().decode()
        return out.reshape(2, L, self.n)

    def load_kswitch(self, stream, elt):
        out = np.zeros((self.k - 1, 2, self.k, self.n), dtype=np.uint64)
        assert ref().refser_load_kswitch(self.h, stream, len(stream), elt, _p(out)) == self.k - 1, ref().refser_last_error().decode()
        return out


def sb():
    import seal_b200

    return seal_b200


def make(scheme, n, bits, prng=P.BLAKE2XB, t_bits=20):
    S = sb()
    mods = R.coeff_modulus_create(n, bits)
    t = R.plain_modulus_batching(n, t_bits) if scheme != O.CKKS else 0
    r = Ref(scheme, n, mods, t, prng)
    ctx = S.Context(scheme, n, mods, t)
    return r, ctx, ctx.load_secret_key(r.secret_key()), mods, t


def keys_match(r, ctx, skd, prng, elts):
    """every key stream of the device equals the reference's; the _size functions give the lengths"""
    k, n = ctx.k, ctx.n
    pk, _ = ctx.generate_public_key_seeded(skd, r.seeds(1)[0], bootstrap_prng=prng)
    assert pk == r.public_key()
    assert len(pk) == sb().lib().sb200_ciphertext_save_seeded_size(ctx.h, k)
    rk = ctx.generate_kswitch_keys_seeded(skd, [0], r.seeds(k - 1), bootstrap_prng=prng)
    assert rk == r.relin_keys() and len(rk) == ctx.kswitch_keys_seeded_size([0])
    distinct = list(dict.fromkeys(elts))
    gk = ctx.generate_kswitch_keys_seeded(skd, elts, r.seeds(len(distinct) * (k - 1)), bootstrap_prng=prng)
    assert gk == r.galois_keys(elts) and len(gk) == ctx.kswitch_keys_seeded_size(elts)
    return pk, rk, gk


@needs_ref
@pytest.mark.parametrize("prng", [P.BLAKE2XB, P.SHAKE256])
@pytest.mark.parametrize("scheme,n,bits", [(O.CKKS, 1024, [40, 40, 50]), (O.BFV, 2048, [36, 36, 37]), (O.BGV, 2048, [40, 40, 50, 50])])
def test_keys_vs_reference(scheme, n, bits, prng):
    """public key, relinearization key, Galois keys with unordered and duplicated elements, and the default Galois set"""
    r, ctx, skd, mods, t = make(scheme, n, bits, prng)
    elts = [2 * n - 1, ctx.galois_elt_from_step(3), 3, ctx.galois_elt_from_step(3), 5]
    keys_match(r, ctx, skd, prng, elts)
    all_elts = K.RefKeygen(scheme, n, mods, t).galois_elts_all()
    gk = ctx.generate_kswitch_keys_seeded(skd, all_elts, r.seeds(len(all_elts) * (ctx.k - 1)), bootstrap_prng=prng)
    assert gk == r.galois_keys(None)
    assert ctx.generate_kswitch_keys_seeded(skd, []) == r.galois_keys([])  # an empty GaloisKeys object: n bare slots


@needs_ref
@pytest.mark.parametrize("n,bits", [(4096, [60, 60, 60]), (32768, [60] * 4)])
def test_keys_60_bit_primes(n, bits):
    r, ctx, skd, mods, t = make(O.CKKS, n, bits)
    keys_match(r, ctx, skd, P.BLAKE2XB, [ctx.galois_elt_from_step(1), 2 * n - 1])


@needs_ref
def test_relin_key_headline_shape():
    """the relinearization key at n = 65536, k = 32 (31 digits): the reference's bytes, and what the reference loads from it"""
    r, ctx, skd, mods, t = make(O.CKKS, 65536, [30] * 32)
    rk = ctx.generate_kswitch_keys_seeded(skd, [0], r.seeds(31))
    assert rk == r.relin_keys()
    words, _ = ctx.generate_kswitch_key(skd, 0, r.seeds(31), device=False)
    assert (r.load_kswitch(rk, 0) == words).all()


def _plain(ctx, scheme, L, t, rng):
    if scheme == O.CKKS:
        return np.stack([rng.integers(0, q, ctx.n, dtype=np.uint64) for q in ctx.moduli[:L]])
    p = rng.integers(0, t, ctx.n, dtype=np.uint64)
    p[:4] = [0, t - 1, t // 2, (t + 1) // 2]  # the lift edges
    return p


def _seeded_ct(ctx, skd, scheme, L, plain, seed, prng, ct_prng=1, scale=1.0):
    """a device seeded symmetric encryption (of plain, or of zero when plain is None) and its stream"""
    import torch

    out = torch.zeros((1, 2, L, ctx.n), dtype=torch.int64, device="cuda")
    if plain is None:
        pub = ctx.d_encrypt_zero_symmetric(skd, out, L, 1, seed, save_seed=True, want_public_seeds=True, bootstrap_prng=prng,
                                           ciphertext_prng=ct_prng)
    else:
        d_plain = torch.from_numpy(np.ascontiguousarray(plain[None]).view(np.int64)).cuda()
        pub = ctx.d_encrypt_symmetric(skd, d_plain, out, L, 1, seed, save_seed=True, want_public_seeds=True, bootstrap_prng=prng,
                                      ciphertext_prng=ct_prng)
    torch.cuda.synchronize()
    stream = ctx.d_save_ciphertexts_seeded(out, L, 1, pub, ct_prng, scheme != O.BFV, scale)[0]
    return out, stream


@needs_ref
@pytest.mark.parametrize("prng", [P.BLAKE2XB, P.SHAKE256])
@pytest.mark.parametrize("scheme,n,bits,t_bits", [(O.CKKS, 4096, [40, 30, 30, 40], 0), (O.BFV, 4096, [36, 36, 37], 20),
                                                  (O.BGV, 4096, [40, 40, 50], 20), (O.BFV, 4096, [30, 30, 30], 40),
                                                  (O.CKKS, 32768, [60] * 4, 0), (O.BFV, 32768, [60] * 3, 30)])
def test_symmetric_ciphertexts_vs_reference(scheme, n, bits, t_bits, prng):
    """encrypt_symmetric(plain) / encrypt_zero_symmetric at two CKKS levels, BFV (seeding changes c_0), BGV, t above every q_j;
    round trips through the device's and the reference's loaders"""
    r, ctx, skd, mods, t = make(scheme, n, bits, prng, t_bits)
    assert scheme == O.CKKS or t_bits < 40 or t > max(mods)
    rng = np.random.default_rng(n + scheme)
    seed = r.seeds(1)
    levels = [ctx.k - 1, ctx.k - 2] if scheme == O.CKKS else [ctx.k - 1]
    for L in levels:
        plain = _plain(ctx, scheme, L, t, rng)
        scale = 2.0 ** 30 if scheme == O.CKKS else 1.0
        ct, stream = _seeded_ct(ctx, skd, scheme, L, plain, seed, prng, scale=scale)
        assert stream == r.encrypt_symmetric(L, plain, scale), f"L={L}"
        assert len(stream) == sb().lib().sb200_ciphertext_save_seeded_size(ctx.h, L)
        words = ct.cpu().numpy().view(np.uint64)[0]
        assert (r.load_ciphertext(stream, L) == words).all()
        import torch

        back = torch.zeros_like(ct)
        info = ctx.d_load_ciphertexts([stream], back, L, 2)[0]
        assert info.seeded == 1 and (back.cpu().numpy().view(np.uint64)[0] == words).all()
        _, zstream = _seeded_ct(ctx, skd, scheme, L, None, seed, prng)
        assert zstream == r.encrypt_zero_symmetric(L)


@needs_ref
@pytest.mark.parametrize("scheme", [O.CKKS, O.BFV, O.BGV])
def test_ciphertext_prng_shake256(scheme):
    """ciphertext_prng = 2: the streams name shake256, carry the restatement's c_0 and public seed, and the device's loaders expand
    them back to the generated words"""
    n, bits = 1024, [40, 40, 50]
    r, ctx, skd, mods, t = make(scheme, n, bits, P.SHAKE256)
    sk = r.secret_key()
    ko = K.KeygenOracle(scheme, n, mods, t)
    seeds = np.arange(8 * (ctx.k - 1), dtype=np.uint64).reshape(ctx.k - 1, 8) * np.uint64(0x9E3779B97F4A7C15)
    words, _ = ctx.generate_kswitch_key(skd, 0, seeds, ciphertext_prng=P.SHAKE256, device=False)
    assert (words == ko.kswitch_key(sk, 0, seeds, P.BLAKE2XB, P.SHAKE256)).all()
    stream = ctx.generate_kswitch_keys_seeded(skd, [0], seeds, ciphertext_prng=P.SHAKE256)
    pk_stream, _ = ctx.generate_public_key_seeded(skd, seeds[0], ciphertext_prng=P.SHAKE256)
    info = sb().ciphertext_inspect(pk_stream)
    assert info.seeded == P.SHAKE256
    pk_words = np.frombuffer(pk_stream, dtype=np.uint64, count=ctx.k * n, offset=info.data_offset).reshape(ctx.k, n)
    assert (pk_words == ko.public_key(sk, seeds[0], P.BLAKE2XB, P.SHAKE256)[0]).all()
    # the stream's relinearization key and the uploaded words relinearize alike
    L = ctx.k - 1
    rng = np.random.default_rng(2)
    c3 = np.stack([np.stack([rng.integers(0, q, n, dtype=np.uint64) for q in mods[:L]]) for _ in range(3)])[None]
    assert (ctx.relinearize(c3, ctx.load_key_stream(stream, 0)) == ctx.relinearize(c3, ctx.load_key(words))).all()
    # symmetric ciphertexts: c_1 of the seeded stream expands with SHAKE256 on load
    seed = seeds[:1]
    ct, cstream = _seeded_ct(ctx, skd, scheme, L, None, seed, P.BLAKE2XB, ct_prng=P.SHAKE256)
    import torch

    back = torch.zeros_like(ct)
    assert ctx.d_load_ciphertexts([cstream], back, L, 2)[0].seeded == P.SHAKE256
    assert (back.cpu() == ct.cpu()).all()


@needs_ref
def test_round_trips_and_key_switching():
    """the key streams load through the reference and through sb200_kswitch_key_load; relinearize / rotate with the loaded keys
    equal those with the generated handles"""
    n = 4096
    r, ctx, skd, mods, t = make(O.CKKS, n, [30] * 8)
    k, L, B = ctx.k, ctx.k - 1, 16
    elt = ctx.galois_elt_from_step(5)
    seeds = r.seeds(k - 1)
    rk = ctx.generate_kswitch_keys_seeded(skd, [0], seeds)
    gk = ctx.generate_kswitch_keys_seeded(skd, [elt, 3], r.seeds(2 * (k - 1)))
    rw, rh = ctx.generate_kswitch_key(skd, 0, seeds)
    gw, gh = ctx.generate_kswitch_key(skd, elt, seeds)
    assert (r.load_kswitch(rk, 0) == rw).all() and (r.load_kswitch(gk, elt) == gw).all()
    pk, pkh = ctx.generate_public_key_seeded(skd, seeds[0], device=True)
    pw, _ = ctx.generate_public_key(skd, seeds[0], device=False)
    assert pkh is not None
    out = np.zeros(2 * k * n, dtype=np.uint64)
    assert ref().refser_load_public_key(r.h, pk, len(pk), _p(out)) == 0 and (out.reshape(2, k, n) == pw).all()
    rng = np.random.default_rng(9)

    def rnd(size):
        return np.stack([np.stack([np.stack([rng.integers(0, q, n, dtype=np.uint64) for q in mods[:L]]) for _ in range(size)])
                         for _ in range(B)])

    a, c3 = rnd(2), rnd(3)
    assert (ctx.relinearize(c3, ctx.load_key_stream(rk, 0)) == ctx.relinearize(c3, rh)).all()
    assert (ctx.apply_galois(a, elt, ctx.load_key_stream(gk, (elt - 1) // 2)) == ctx.apply_galois(a, elt, gh)).all()


def test_chunked_generation_gives_the_same_bytes():
    """a 1 MiB scratch budget cuts the 7 digits of n = 2048, k = 8 into chunks of 3, 3 and 1: the streams of two keys equal those
    of one chunk per key"""
    S = sb()
    n = 2048
    mods = O.coeff_modulus_create(n, [30] * 8)
    ctx = S.Context(S.BGV, n, mods, R.plain_modulus_batching(n, 20))
    rng = np.random.default_rng(5)
    skd = ctx.load_secret_key(np.stack([rng.integers(0, q, n, dtype=np.uint64) for q in mods]))
    elts = [2 * n - 1, 5]
    seeds = rng.integers(0, 2 ** 63, (2, 7, 8), dtype=np.uint64)
    whole = ctx.generate_kswitch_keys_seeded(skd, elts, seeds)
    ctx.set_limit(ctx.LIMIT_SCRATCH_BYTES, 1 << 20)
    ctx.profile(True)
    cut = ctx.generate_kswitch_keys_seeded(skd, elts, seeds)
    launches = {name: cnt for name, _, cnt, _ in ctx.profile_read()}
    ctx.profile(False)
    ctx.set_limit(ctx.LIMIT_SCRATCH_BYTES, 8 << 30)
    assert launches.get("enc_combine:kswitch") == 6, launches
    assert cut == whole
    # the key behind the stream is the generator's: element 5 sits in slot 2
    words, _ = ctx.generate_kswitch_key(skd, 5, seeds[1], device=False)
    c3 = np.stack([np.stack([rng.integers(0, q, n, dtype=np.uint64) for q in mods[:7]]) for _ in range(3)])[None]
    assert (ctx.relinearize(c3, ctx.load_key_stream(cut, 2)) == ctx.relinearize(c3, ctx.load_key(words))).all()


def test_errors_leave_the_output_untouched():
    S = sb()
    n = 1024
    mods = O.coeff_modulus_create(n, [40, 40, 40])
    ctx, other = S.Context(S.CKKS, n, mods), S.Context(S.CKKS, n, mods)
    rng = np.random.default_rng(1)
    sk = np.stack([rng.integers(0, q, n, dtype=np.uint64) for q in mods])
    skd, foreign = ctx.load_secret_key(sk), other.load_secret_key(sk)
    L = S.lib()
    size = ctx.kswitch_keys_seeded_size([3])
    assert size > 0 and ctx.kswitch_keys_seeded_size([2]) == 0 and ctx.kswitch_keys_seeded_size([0, 3]) == 0

    def ks(elts, key=skd, bp=1, cp=1, cap=size):
        buf = C.create_string_buffer(b"\xAB" * size, size)
        e = (C.c_uint32 * max(len(elts), 1))(*elts)
        rc = L.sb200_kswitch_keys_generate_seeded(ctx.h, key.h, e, len(elts), bp, cp, None, C.addressof(buf), cap)
        assert buf.raw == b"\xAB" * size, "output written on error"
        return rc, L.sb200_last_error().decode()

    assert ks([2]) == (-1, "Galois element is not valid")
    assert ks([2 * n + 1])[0] == -1
    assert ks([0, 3]) == (-1, "galois_elts: 0 (relinearization) cannot be mixed with Galois elements")
    assert ks([3], key=foreign) == (-1, "secret key is not valid for encryption parameters")
    assert ks([3], bp=3) == (-1, "prng_type is invalid") and ks([3], cp=0) == (-1, "prng_type is invalid")
    assert ks([3], cap=size - 1) == (-1, "insufficient size")
    one = S.Context(S.CKKS, n, mods[:1])
    sk1 = one.load_secret_key(sk[:1].copy())
    with pytest.raises(RuntimeError, match="keyswitching is not supported by the context"):
        one.generate_kswitch_keys_seeded(sk1, [0], capacity=64)
    # the public key
    cap = L.sb200_ciphertext_save_seeded_size(ctx.h, ctx.k)
    for kw, msg in ((dict(key=foreign), "secret key is not valid"), (dict(bp=0), "prng_type"), (dict(cap=cap - 1), "insufficient size")):
        buf = C.create_string_buffer(b"\xCD" * cap, cap)
        rc = L.sb200_public_key_generate_seeded(ctx.h, kw.get("key", skd).h, kw.get("bp", 1), 1, None, C.addressof(buf), kw.get("cap", cap), None)
        assert rc == -1 and msg in L.sb200_last_error().decode() and buf.raw == b"\xCD" * cap
    assert L.sb200_public_key_generate_seeded(ctx.h, skd.h, 1, 1, None, None, cap, None) == -6
    # ciphertexts
    import torch

    Lv = ctx.k - 1
    ct = torch.zeros((2, 2, Lv, n), dtype=torch.int64, device="cuda")
    pub = ctx.d_encrypt_zero_symmetric(skd, ct, Lv, 2, save_seed=True, want_public_seeds=True)
    torch.cuda.synchronize()
    cap = L.sb200_ciphertext_save_seeded_size(ctx.h, Lv)
    meta = (S.CtInfo * 2)()

    def save(prng=1, capacity=cap, null_second=False, level=Lv, seeds=pub):
        bufs = [C.create_string_buffer(b"\xEF" * cap, cap) for _ in range(2)]
        outs = (C.c_void_p * 2)(C.addressof(bufs[0]), None if null_second else C.addressof(bufs[1]))
        rc = L.sb200_ciphertext_save_seeded(ctx.h, 2, level, C.c_void_p(ct.data_ptr()), meta,
                                            None if seeds is None else seeds.ctypes.data_as(_u64p), prng, outs, capacity, None)
        assert all(b.raw == b"\xEF" * cap for b in bufs), "output written on error"
        return rc

    assert save(prng=0) == -1 and save(prng=3) == -1
    assert save(capacity=cap - 1) == -1
    assert save(null_second=True) == -1
    assert save(level=ctx.k + 1) == -1
    assert save(seeds=None) == -6


SHIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref", "bin", "shim_serial_test")


@pytest.mark.skipif(not os.path.exists(SHIM), reason="oracle/_ref/bin/shim_serial_test not built (oracle/serial.mk, needs the reference sources)")
def test_cpp_serializable_against_reference():
    """seal_b200::KeyGenerator / Encryptor Serializable overloads against seal::'s: save (none and zlib) and save_size, loads"""
    r = subprocess.run([SHIM], capture_output=True, text=True, timeout=900)
    print(r.stdout, r.stderr)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "PASS" in r.stdout
