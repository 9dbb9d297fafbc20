"""Test infrastructure for the device's PRNG paths (TEST INFRASTRUCTURE ONLY; the product never loads any of it):
  * ctypes drivers for oracle/libshake256.so (SHAKE256 from FIPS 202) and oracle/_ref/libsealref_prng.so (the unmodified
    reference behind oracle/ref_prng.cpp: contexts with a Blake2xb or Shake256 random generator factory, PRNG streams, seeded
    ciphertext and key objects and the reference's loaders), both built by oracle/prng.mk;
  * a restatement, on a PRNG of either type, of what the reference samples from a PRNG stream (sample_poly_uniform,
    encrypt_zero_symmetric, encrypt_zero_asymmetric), composed from numpy and the transforms / divide-and-round steps of
    oracle/liboracle.so (tests/oracle.py) -- the same steps oracle/seal_oracle.c takes for the blake2xb stream only;
  * byte-level edits of serialized objects: retype a seeded stream's PRNG, wrap an object in the zlib form.
Types are SEAL's prng_type: 1 = blake2xb, 2 = shake256."""
import ctypes as C
import os

import numpy as np

import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_SHAKE = os.path.join(_HERE, "..", "oracle", "libshake256.so")
_REF = os.path.join(_HERE, "..", "oracle", "_ref", "libsealref_prng.so")
BLAKE2XB, SHAKE256 = 1, 2
BFV, CKKS, BGV = 1, 2, 3
_u64p = C.POINTER(C.c_uint64)
_shake = None
_ref = None


def _p(a):
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(_u64p)


def shake_lib():
    global _shake
    if _shake is None:
        L = C.CDLL(_SHAKE)
        L.orc_shake256.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]
        L.orc_shake256_stream.argtypes = [_u64p, C.c_size_t, _u64p]
        _shake = L
    return _shake


def ref_available():
    return os.path.exists(_REF)


def ref_lib():
    global _ref
    if _ref is None:
        L = C.CDLL(_REF)
        L.sealprng_last_error.restype = C.c_char_p
        L.sealprng_create.restype = C.c_void_p
        L.sealprng_create.argtypes = [C.c_int, C.c_size_t, _u64p, C.c_size_t, C.c_uint64, C.c_uint64, C.c_int]
        L.sealprng_destroy.argtypes = [C.c_void_p]
        L.sealprng_stream.argtypes = [C.c_int, _u64p, C.c_size_t, C.c_char_p]
        L.sealprng_secret_key.argtypes = [C.c_void_p, _u64p]
        L.sealprng_public_key.argtypes = [C.c_void_p, _u64p]
        L.sealprng_encrypt_zero_symmetric.argtypes = [C.c_void_p, C.c_size_t, _u64p]
        L.sealprng_encrypt_zero_asymmetric.argtypes = [C.c_void_p, C.c_size_t, _u64p]
        for f in ("sealprng_seeded_ct_stream", "sealprng_ct_load", "sealprng_seeded_kswitch_keys_stream", "sealprng_kswitch_keys_load"):
            getattr(L, f).restype = C.c_long
        L.sealprng_seeded_ct_stream.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t]
        L.sealprng_ct_load.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, _u64p, C.c_size_t]
        L.sealprng_seeded_kswitch_keys_stream.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_char_p, C.c_size_t]
        L.sealprng_kswitch_keys_load.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_size_t, _u64p, C.c_size_t]
        _ref = L
    return _ref


def _chk(rc):
    if rc < 0:
        raise RuntimeError(ref_lib().sealprng_last_error().decode())
    return rc


# ---- streams ----
def shake256(data, nbytes):
    """SHAKE256 (FIPS 202) of a byte string -> nbytes bytes (oracle/shake256.c)"""
    out = C.create_string_buffer(max(nbytes, 1))
    shake_lib().orc_shake256(bytes(data), len(data), out, nbytes)
    return out.raw[:nbytes]


def stream(prng, seed, words):
    """the first `words` 64-bit words of Blake2xbPRNG(seed) (oracle/seal_oracle.c) / Shake256PRNG(seed) (oracle/shake256.c)"""
    seed = np.ascontiguousarray(seed, dtype=np.uint64)
    out = np.zeros(words, dtype=np.uint64)
    if prng == BLAKE2XB:
        O.lib().orc_blake2xb_stream(_p(seed), words, _p(out))
    elif prng == SHAKE256:
        shake_lib().orc_shake256_stream(_p(seed), words, _p(out))
    else:
        raise ValueError("prng_type")
    return out


def ref_stream(prng, seed, nbytes):
    """UniformRandomGenerator::generate(nbytes) of the reference's Blake2xbPRNG(seed) / Shake256PRNG(seed)"""
    seed = np.ascontiguousarray(seed, dtype=np.uint64)
    buf = C.create_string_buffer(nbytes)
    _chk(ref_lib().sealprng_stream(prng, _p(seed), nbytes, buf))
    return buf.raw[:nbytes]


# ---- the restatement: what the reference samples from a stream ----
def _mulmod(a, b, q):
    return np.array([(int(x) * int(y)) % q for x, y in zip(a, b)], dtype=np.uint64)


class PrngOracle:
    """sample_poly_uniform / encrypt_zero_symmetric / encrypt_zero_asymmetric on PRNGs of either type, for the context of
    `oc` (a tests/oracle.py Oracle: its transforms, rescale and mod-switch steps are used as they are)"""

    def __init__(self, oc):
        self.oc, self.n, self.q = oc, oc.n, oc.moduli

    def expand_seed(self, L, seed, prng):
        """Ciphertext::expand_seed (util/rlwe.cpp:104-132): the first L n words fill the polynomial; every word >= max_multiple of
        its prime is replaced, in coefficient order, by the next words of the stream; the survivors are reduced -> [L][n]"""
        n, need = self.n, L * self.n
        words = stream(prng, seed, need + 4096)
        out = words[:need].copy()
        head = need
        for j in range(L):
            q = self.q[j]
            mm = np.uint64((2 ** 64 - 1) - (2 ** 64 - 1) % q - 1)
            seg = out[j * n:(j + 1) * n]
            for i in np.nonzero(seg >= mm)[0]:
                r = seg[i]
                while r >= mm:
                    if head == len(words):
                        words = stream(prng, seed, 2 * len(words))
                    r = words[head]
                    head += 1
                seg[i] = r
            out[j * n:(j + 1) * n] = seg % np.uint64(q)
        return out.reshape(L, n)

    def _noise(self, raw, count):
        """sample_poly_cbd (util/rlwe.cpp:73-102): 6 bytes per coefficient, hw(x0, x1, x2 & 31) - hw(x3, x4, x5 & 31)"""
        b = np.frombuffer(raw, dtype=np.uint8, count=6 * count).reshape(count, 6).copy()
        b[:, 2] &= 0x1F
        b[:, 5] &= 0x1F
        hw = np.unpackbits(b, axis=1).reshape(count, 6, 8).sum(axis=2).astype(np.int64)
        return hw[:, :3].sum(axis=1) - hw[:, 3:].sum(axis=1)

    def _residues(self, v, q):
        return np.where(v >= 0, v, v + q).astype(np.uint64)

    def encrypt_zero_symmetric(self, sk, seed, save_seed, boot_prng, ct_prng, L=None):
        """util/rlwe.cpp:264-408: the bootstrap PRNG (boot_prng) yields the public seed and the noise, c_1 is the public seed's
        expansion on a PRNG of type ct_prng; c_0 = -(c_1 s + e) (BGV: t e); BFV in coefficient form -> [2][L][n]"""
        oc, n = self.oc, self.n
        L = L or (oc.k - 1 if oc.k > 1 else 1)
        scheme = oc.scheme
        boot = stream(boot_prng, seed, (64 + 6 * n + 7) // 8)
        c1 = self.expand_seed(L, boot[:8], ct_prng)
        c1n = c1.copy()
        if scheme == O.BFV:
            for j in range(L):
                if save_seed:
                    c1n[j] = oc.ntt_row(j, c1[j])  # the sample is c_1 itself
                else:
                    c1[j] = oc.intt_row(j, c1[j])  # the sample is NTT(c_1)
        noise = self._noise(boot.tobytes()[64:], n)
        c0 = np.zeros((L, n), dtype=np.uint64)
        for j in range(L):
            q = self.q[j]
            e = self._residues(noise, q)
            p = _mulmod(np.ascontiguousarray(sk[j]), c1n[j], q)
            if scheme == O.BFV:
                p = oc.intt_row(j, p)
            else:
                e = oc.ntt_row(j, e)
            if scheme == O.BGV:
                e = _mulmod(e, np.full(n, oc.t % q, dtype=np.uint64), q)
            v = (p.astype(object) + e.astype(object)) % q
            c0[j] = np.array([(q - x) % q for x in v], dtype=np.uint64)
        return np.stack([c0, c1])

    def encrypt_zero_asymmetric(self, pk, seed, prng, L=None):
        """util/rlwe.cpp:184-276: one PRNG yields the ternary u (one 32-bit word per coefficient, (r * 3) >> 32, redraw for r == 0:
        libstdc++'s uniform_int_distribution) then e_0, e_1; c_p = pk_p u + e_p (BGV: t e_p) one level above, divided down"""
        oc, n, k = self.oc, self.n, self.oc.k
        L = L or (k - 1 if k > 1 else 1)
        Lp = L + 1 if L < k else L
        words = stream(prng, seed, (16 * n + 7) // 8 + 64)
        w32 = words.view(np.uint32)
        pos, r = 0, np.zeros(n, dtype=np.int64)
        for i in range(n):
            while w32[pos] == 0:
                pos += 1
            r[i] = (int(w32[pos]) * 3) >> 32
            pos += 1
        noise = self._noise(words.tobytes()[4 * pos:], 2 * n)
        t2 = np.zeros((2, Lp, n), dtype=np.uint64)
        for j in range(Lp):
            q = self.q[j]
            u = oc.ntt_row(j, self._residues(r - 1, q))
            for p in range(2):
                d = _mulmod(u, np.ascontiguousarray(pk[p, j]), q)
                e = self._residues(noise[p * n:(p + 1) * n], q)
                if oc.scheme == O.BFV:
                    d = oc.intt_row(j, d)
                else:
                    e = oc.ntt_row(j, e)
                if oc.scheme == O.BGV:
                    e = _mulmod(e, np.full(n, oc.t % q, dtype=np.uint64), q)
                t2[p, j] = ((d.astype(object) + e.astype(object)) % q).astype(np.uint64)
        if Lp == L:
            return t2
        if oc.scheme == O.CKKS:
            return oc.rescale(Lp, t2)
        return oc.bfv_mod_switch(Lp, t2) if oc.scheme == O.BFV else oc.bgv_mod_switch(Lp, t2)


# ---- the reference under a factory of either type ----
class RefPrngContext:
    """one reference SEALContext (sec_level none) whose parameters carry a Blake2xbPRNGFactory / Shake256PRNGFactory({seed, 0..})"""

    def __init__(self, scheme, n, moduli, plain_modulus=0, seed=0x5EA1, prng=SHAKE256):
        self.scheme, self.n, self.moduli, self.k = scheme, n, list(moduli), len(moduli)
        m = np.array(self.moduli, dtype=np.uint64)
        self.h = ref_lib().sealprng_create(scheme, n, _p(m), self.k, plain_modulus, seed, prng)
        if not self.h:
            raise RuntimeError(ref_lib().sealprng_last_error().decode())

    def __del__(self):
        if getattr(self, "h", None):
            ref_lib().sealprng_destroy(self.h)
            self.h = None

    def _L(self, L):
        return L or (self.k - 1 if self.k > 1 else 1)

    def secret_key(self):
        out = np.zeros((self.k, self.n), dtype=np.uint64)
        _chk(ref_lib().sealprng_secret_key(self.h, _p(out)))
        return out

    def public_key(self):
        out = np.zeros((2, self.k, self.n), dtype=np.uint64)
        _chk(ref_lib().sealprng_public_key(self.h, _p(out)))
        return out

    def encrypt_zero_symmetric(self, L=None):
        L = self._L(L)
        out = np.zeros((2, L, self.n), dtype=np.uint64)
        _chk(ref_lib().sealprng_encrypt_zero_symmetric(self.h, L, _p(out)))
        return out

    def encrypt_zero_asymmetric(self, L=None):
        L = self._L(L)
        out = np.zeros((2, L, self.n), dtype=np.uint64)
        _chk(ref_lib().sealprng_encrypt_zero_asymmetric(self.h, L, _p(out)))
        return out

    def seeded_ct_stream(self, compr=0):
        buf = C.create_string_buffer(2 * self.k * self.n * 8 + 4096)
        ln = _chk(ref_lib().sealprng_seeded_ct_stream(self.h, compr, buf, len(buf)))
        return buf.raw[:ln]

    def ct_load(self, data):
        """Ciphertext::load -> [size][L][n]"""
        out = np.zeros(16 * self.k * self.n, dtype=np.uint64)
        rows = _chk(ref_lib().sealprng_ct_load(self.h, data, len(data), _p(out), out.size))
        import seal_b200 as S

        info = S.ciphertext_inspect(data)
        return out[:rows * self.n].reshape(info.size, rows // info.size, self.n).copy()

    def seeded_kswitch_keys_stream(self, galois_elt=0, compr=0):
        raw = (self.k - 1) * 2 * self.k * self.n * 8
        buf = C.create_string_buffer(raw + raw // 8 + 8 * self.n + (1 << 16))
        ln = _chk(ref_lib().sealprng_seeded_kswitch_keys_stream(self.h, galois_elt, compr, buf, len(buf)))
        return buf.raw[:ln]

    def kswitch_keys_load(self, data, index):
        out = np.zeros((self.k - 1, 2, self.k, self.n), dtype=np.uint64)
        d = _chk(ref_lib().sealprng_kswitch_keys_load(self.h, data, len(data), index, _p(out), out.size))
        return out[:d]


# ---- byte-level edits of serialized objects ----
def with_prng_type(data, prng):
    """a copy of a seed-compressed Ciphertext stream (compr_mode none) whose prng_type byte (in front of the seed) names `prng`:
    the reference's own load then expands it with that PRNG"""
    import seal_b200 as S

    info = S.ciphertext_inspect(data)
    assert info.seeded and info.compr_mode == 0
    b = bytearray(data)
    b[info.seed_offset - 1] = prng
    return bytes(b)


def kswitch_with_prng_type(data, prng):
    """the same for every seeded member of a KSwitchKeys stream (compr_mode none): SEALHeader, parms_id, dim1, then per slot
    dim2 and dim2 Ciphertext streams (kswitchkeys.cpp:42-86)"""
    import seal_b200 as S

    b = bytearray(data)
    off = 16 + 32
    dim1 = int.from_bytes(b[off:off + 8], "little")
    off += 8
    for _ in range(dim1):
        dim2 = int.from_bytes(b[off:off + 8], "little")
        off += 8
        for _ in range(dim2):
            info = S.ciphertext_inspect(bytes(b[off:]))
            if info.seeded:
                b[off + info.seed_offset - 1] = prng
            off += info.stream_bytes
    return bytes(b)


def kswitch_members(data, index):
    """[(byte offset of the member, its sb200_ct_info)] of slot `index` of a KSwitchKeys stream (compr_mode none)"""
    import seal_b200 as S

    off, found = 16 + 32 + 8, []
    for slot in range(index + 1):
        dim2 = int.from_bytes(data[off:off + 8], "little")
        off += 8
        for _ in range(dim2):
            info = S.ciphertext_inspect(data[off:])
            if slot == index:
                found.append((off, info))
            off += info.stream_bytes
    return found


def zlib_stream(data):
    """compr_mode_type::zlib form of an uncompressed SEAL object: SEALHeader{compr_mode 1, size} + one zlib stream of the body
    (serialization.cpp:236-300)"""
    import zlib

    body = zlib.compress(data[16:])
    hdr = bytearray(data[:16])
    hdr[5] = 1
    hdr[8:16] = (16 + len(body)).to_bytes(8, "little")
    return bytes(hdr) + body
