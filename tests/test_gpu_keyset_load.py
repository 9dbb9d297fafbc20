"""Key sets loaded in one pass on an H100 (-m gpu): sb200_kswitch_keys_load against the per-slot sb200_kswitch_key_load and against
sb200_kswitch_key_create on the reference's loaded words (oracle/ref_keyset.cpp), for RelinKeys and GaloisKeys streams saved with
compr_mode none and zlib and as seeded objects (blake2xb from the reference, shake256 from the device), with both stored forms of
the key (SB200_LIMIT_KS_ALGORITHM 0 and 2); sb200_kswitch_key_device_bytes at n = 65536, k = 32; the argument errors with the output
and the device memory left as they were; and the C++ key sets and batch streams (tests/cpp/shim_keyset_test.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle as O
import refprng as P
import refseal as R

pytestmark = pytest.mark.gpu
_HERE = os.path.dirname(os.path.abspath(__file__))
_REF = os.path.join(_HERE, "..", "oracle", "_ref", "libsealref_keyset.so")
needs_ref = pytest.mark.skipif(not os.path.exists(_REF), reason="oracle/_ref/libsealref_keyset.so not present (oracle/keyset.mk)")
_u64p = C.POINTER(C.c_uint64)
_lib = None
NONE, ZLIB, SEEDED = 0, 1, 2


def ref():
    global _lib
    if _lib is None:
        L = C.CDLL(_REF)
        vp, sz = C.c_void_p, C.c_size_t
        L.refks_last_error.restype = C.c_char_p
        L.refks_create.restype = vp
        L.refks_create.argtypes = [C.c_int, sz, _u64p, sz, C.c_uint64, C.c_uint64, C.c_int]
        L.refks_destroy.argtypes = [vp]
        L.refks_secret_key.argtypes = [vp, _u64p]
        L.refks_relin_keys.restype = C.c_long
        L.refks_relin_keys.argtypes = [vp, C.c_int, vp, sz]
        L.refks_galois_keys.restype = C.c_long
        L.refks_galois_keys.argtypes = [vp, C.POINTER(C.c_uint32), sz, C.c_int, C.c_int, vp, sz]
        L.refks_galois_elts_all.restype = C.c_long
        L.refks_galois_elts_all.argtypes = [vp, C.POINTER(C.c_uint32), sz]
        L.refks_load_kswitch.restype = C.c_long
        L.refks_load_kswitch.argtypes = [vp, C.c_char_p, sz, C.c_uint32, _u64p]
        _lib = L
    return _lib


def _p(a):
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(_u64p)


class Ref:
    """the reference's KeyGenerator under a fixed-seed Blake2xb factory: every key of an element is the same on every call"""

    def __init__(self, scheme, n, mods, t, seed=0x5E75):
        self.n, self.k = n, len(mods)
        self.h = ref().refks_create(scheme, n, _p(np.array(mods, dtype=np.uint64)), self.k, t, seed, P.BLAKE2XB)
        assert self.h, ref().refks_last_error().decode()

    def __del__(self):
        if getattr(self, "h", None):
            ref().refks_destroy(self.h)

    def _bytes(self, fn, *args):
        size = fn(self.h, *args, None, 0)
        assert size >= 0, ref().refks_last_error().decode()
        buf = C.create_string_buffer(size)
        assert fn(self.h, *args, C.addressof(buf), size) == size, ref().refks_last_error().decode()
        return buf.raw

    def secret_key(self):
        out = np.zeros((self.k, self.n), dtype=np.uint64)
        assert ref().refks_secret_key(self.h, _p(out)) == 0
        return out

    def relin_keys(self, mode):
        return self._bytes(ref().refks_relin_keys, mode)

    def galois_keys(self, elts, mode):
        e = (C.c_uint32 * max(len(elts or []), 1))(*(elts or []))
        return self._bytes(ref().refks_galois_keys, e, len(elts or []), int(elts is None), mode)

    def elts_all(self):
        out = (C.c_uint32 * 256)()
        got = ref().refks_galois_elts_all(self.h, out, 256)
        assert got > 0, ref().refks_last_error().decode()
        return [int(out[i]) for i in range(got)]

    def words(self, stream, elt):
        out = np.zeros((self.k - 1, 2, self.k, self.n), dtype=np.uint64)
        assert ref().refks_load_kswitch(self.h, stream, len(stream), elt, _p(out)) == self.k - 1, ref().refks_last_error().decode()
        return out


def sb():
    import seal_b200

    return seal_b200


def _rand(rng, mods, B, size, L, n):
    return np.stack([np.stack([np.stack([rng.integers(0, q, n, dtype=np.uint64) for q in mods[:L]]) for _ in range(size)])
                     for _ in range(B)])


def _switch(ctx, key, elt, c2, c3):
    """the key's output on a random batch: relinearize for elt 0, apply_galois otherwise"""
    return ctx.relinearize(c3, key) if elt == 0 else ctx.apply_galois(c2, elt, key)


def _check_set(ctx, r, stream, elts, keys, words, c2, c3):
    """every handle of the one-pass load equals the per-slot load and the handle made from the reference's words"""
    assert [k.slot for k in keys] == [0 if e == 0 else (e - 1) // 2 for e in elts]
    for key, elt in zip(keys, elts):
        want = _switch(ctx, ctx.load_key(words[elt]), elt, c2, c3)
        assert (_switch(ctx, key, elt, c2, c3) == want).all(), f"one-pass load, element {elt}"
        assert (_switch(ctx, ctx.load_key_stream(stream, key.slot), elt, c2, c3) == want).all(), f"per-slot load, element {elt}"


@needs_ref
@pytest.mark.parametrize("algo", [0, 2])
@pytest.mark.parametrize("n", [4096, 8192])
@pytest.mark.parametrize("scheme", [O.CKKS, O.BFV, O.BGV])
def test_one_pass_load_equals_per_slot_and_reference(scheme, n, algo):
    mods = R.coeff_modulus_create(n, [36, 36, 36, 37])
    t = R.plain_modulus_batching(n, 20) if scheme != O.CKKS else 0
    r = Ref(scheme, n, mods, t)
    S = sb()
    ctx = S.Context(scheme, n, mods, t)
    ctx.set_limit(ctx.LIMIT_KS_ALGORITHM, algo)
    k, L = ctx.k, ctx.k - 1
    rng = np.random.default_rng(n + scheme + algo)
    c2, c3 = _rand(rng, mods, 4, 2, L, n), _rand(rng, mods, 4, 3, L, n)
    all_elts = r.elts_all()
    # the reference's words of every key, from its own load of its none stream (the factory makes the same keys on every call)
    gk_none = r.galois_keys(None, NONE)
    words = {e: r.words(gk_none, e) for e in all_elts}
    words[0] = r.words(r.relin_keys(NONE), 0)
    for mode in (NONE, ZLIB, SEEDED):
        rk = r.relin_keys(mode)
        _check_set(ctx, r, rk, [0], ctx.load_kswitch_keys(rk), words, c2, c3)
        _check_set(ctx, r, rk, [0], ctx.load_kswitch_keys(rk, [0]), words, c2, c3)
    # the default set: every non-empty slot; an unordered subset of it
    subset = [all_elts[5], all_elts[1], 2 * n - 1, all_elts[3]]  # all_elts[0] is 2 n - 1
    for mode in (NONE, ZLIB, SEEDED):
        gk = gk_none if mode == NONE else r.galois_keys(None, mode)
        # (get_elts_all lists the element of order 2, n + 1, twice: as a power of the generator and as its inverse)
        _check_set(ctx, r, gk, sorted(set(all_elts)), ctx.load_kswitch_keys(gk), words, c2, c3)
        _check_set(ctx, r, gk, subset, ctx.load_kswitch_keys(gk, [(e - 1) // 2 for e in subset]), words, c2, c3)
    # seeded streams whose c_1 expands with shake256, written by the device's generator
    skd = ctx.load_secret_key(r.secret_key())
    seeds = np.arange(8 * 3 * (k - 1), dtype=np.uint64).reshape(3, k - 1, 8) * np.uint64(0x9E3779B97F4A7C15)
    elts = [all_elts[2], all_elts[1]]
    stream = ctx.generate_kswitch_keys_seeded(skd, elts, seeds[:2], ciphertext_prng=P.SHAKE256)
    shake = {e: ctx.generate_kswitch_key(skd, e, seeds[i], ciphertext_prng=P.SHAKE256, device=False)[0] for i, e in enumerate(elts)}
    _check_set(ctx, r, stream, sorted(elts), ctx.load_kswitch_keys(stream), shake, c2, c3)
    _check_set(ctx, r, stream, elts, ctx.load_kswitch_keys(stream, [(e - 1) // 2 for e in elts]), shake, c2, c3)
    rk_stream = ctx.generate_kswitch_keys_seeded(skd, [0], seeds[2], ciphertext_prng=P.SHAKE256)
    rk_words = {0: ctx.generate_kswitch_key(skd, 0, seeds[2], ciphertext_prng=P.SHAKE256, device=False)[0]}
    _check_set(ctx, r, rk_stream, [0], ctx.load_kswitch_keys(rk_stream), rk_words, c2, c3)


def test_headline_shape_device_bytes():
    """the relinearization key and two Galois keys at n = 65536, k = 32 from seeded streams: the handles hold the 64-bit key plus the
    integer path's copy, and switch keys like the generator's own handles"""
    S = sb()
    n, k = 65536, 32
    mods = O.coeff_modulus_create(n, [30] * k)
    ctx = S.Context(S.CKKS, n, mods)
    rng = np.random.default_rng(65536)
    skd = ctx.load_secret_key(np.stack([rng.integers(0, q, n, dtype=np.uint64) for q in mods]))
    seeds = rng.integers(0, 2 ** 63, (3, k - 1, 8), dtype=np.uint64)
    elts = [ctx.galois_elt_from_step(1), 2 * n - 1]
    rk = ctx.generate_kswitch_keys_seeded(skd, [0], seeds[0])
    gk = ctx.generate_kswitch_keys_seeded(skd, elts, seeds[1:])
    S_aux = len(ctx.ksint_primes())
    assert S_aux > 0
    words = (k - 1) * 2 * k * n
    expect = 8 * words + 4 * (S_aux * words + 8 * n)
    keys = ctx.load_kswitch_keys(rk) + ctx.load_kswitch_keys(gk, [(elts[1] - 1) // 2, (elts[0] - 1) // 2])
    assert [key.device_bytes for key in keys] == [expect] * 3
    assert S.lib().sb200_kswitch_key_device_bytes(None) == 0
    L, B = k - 1, 2
    c2, c3 = _rand(rng, mods, B, 2, L, n), _rand(rng, mods, B, 3, L, n)
    _, h = ctx.generate_kswitch_key(skd, 0, seeds[0], host=False)
    assert (ctx.relinearize(c3, keys[0]) == ctx.relinearize(c3, h)).all()
    del h
    _, h = ctx.generate_kswitch_key(skd, elts[0], seeds[1], host=False)
    assert (ctx.apply_galois(c2, elts[0], keys[2]) == ctx.apply_galois(c2, elts[0], h)).all()


def test_errors_leave_output_and_device_memory_untouched():
    import torch

    S = sb()
    L = S.lib()
    n = 8192
    mods = O.coeff_modulus_create(n, [30] * 8)
    ctx = S.Context(S.BGV, n, mods, R.plain_modulus_batching(n, 20))
    rng = np.random.default_rng(8)
    skd = ctx.load_secret_key(np.stack([rng.integers(0, q, n, dtype=np.uint64) for q in mods]))
    e1, e2 = 3, 2 * n - 1
    stream = ctx.generate_kswitch_keys_seeded(skd, [e1, e2])
    slot1, slot2 = (e1 - 1) // 2, (e2 - 1) // 2
    # a word >= its modulus in c_0 of the second key: found by the range check after the first handle exists.  The object is the
    # frame (header, parms_id, dim1: 56 bytes), one dim2 word per slot, and k - 1 seeded members per key: prefix, k n words, seed info
    digits, prefix = ctx.k - 1, 16 + 73 + 16 + 8
    member = prefix + 8 * ctx.k * n + 16 + 1 + 64
    assert len(stream) == 56 + 8 * n + 2 * digits * member
    first = 56 + 8 * (slot2 + 1) + digits * member
    assert S.ciphertext_inspect(stream[first:first + member]).data_offset == prefix
    bad = bytearray(stream)
    bad[first + prefix:first + prefix + 8] = (2 ** 64 - 1).to_bytes(8, "little")
    bad = bytes(bad)
    other = S.Context(S.BGV, n, O.coeff_modulus_create(n, [30] * 7), R.plain_modulus_batching(n, 20))
    ctx.load_kswitch_keys(stream)  # the context's scratch is now at its size for this shape
    torch.cuda.synchronize()
    key_bytes = 8 * (ctx.k - 1) * 2 * ctx.k * n

    def call(c=ctx, s=stream, idx=None, count=None, out=True, out_count=True):
        cap = 4
        arr = (C.c_void_p * cap)(*([0xDEAD] * cap))
        slots = (C.c_size_t * cap)(*([777] * cap))
        got = C.c_size_t(999)
        ip = None if idx is None else (C.c_size_t * max(len(idx), 1))(*idx)
        free0 = torch.cuda.mem_get_info()[0]
        rc = L.sb200_kswitch_keys_load(c.h if c is not None else None, s, 0 if s is None else len(s), ip,
                                       (len(idx) if idx is not None else cap) if count is None else count,
                                       arr if out else None, slots, C.byref(got) if out_count else None)
        torch.cuda.synchronize()
        free1 = torch.cuda.mem_get_info()[0]
        assert list(arr) == [0xDEAD] * cap and list(slots) == [777] * cap and got.value == 999, "output written on error"
        assert abs(free1 - free0) < key_bytes // 2, f"device memory moved by {free0 - free1} bytes"
        return rc, L.sb200_last_error().decode()

    assert call(idx=[n])[0] == -3                                   # an index at or past the slot count
    assert call(idx=[slot1, 5]) == (-1, "key not present")         # an empty slot
    assert call(idx=[slot1, slot1])[0] == -1                        # a duplicated index
    assert call(count=1)[0] == -1                                   # capacity below the two keys of the NULL form
    assert call(c=None)[0] == -6 and call(s=None)[0] == -6
    assert call(out=False)[0] == -6 and call(out_count=False)[0] == -6
    assert call(c=other) == (-2, "KSwitchKeys data is invalid")     # keys of another context
    assert call(s=bad, idx=[slot1, slot2]) == (-2, "KSwitchKeys data is invalid")
    assert call(s=bad)[0] == -2
    assert L.sb200_kswitch_key_load(ctx.h, bad, len(bad), slot2, C.byref(C.c_void_p())) == -2
    # the first key of the corrupted stream is intact and still loads
    assert len(ctx.load_kswitch_keys(bad, [slot1])) == 1


SHIM = os.path.join(_HERE, "..", "oracle", "_ref", "bin", "shim_keyset_test")


@pytest.mark.skipif(not os.path.exists(SHIM), reason="oracle/_ref/bin/shim_keyset_test not built (oracle/keyset.mk, needs the reference sources)")
def test_cpp_key_sets_and_batch_streams_against_reference():
    """DeviceRelinKeys / DeviceGaloisKeys overloads, KeyGenerator device keys, CiphertextBatch load / save against seal::"""
    r = subprocess.run([SHIM], capture_output=True, text=True, timeout=900)
    print(r.stdout, r.stderr)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "PASS" in r.stdout
