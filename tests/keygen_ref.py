"""Test infrastructure for the device's key generation (TEST INFRASTRUCTURE ONLY; the product never loads any of it):
  * a ctypes driver for oracle/_ref/libsealref_keygen.so (oracle/ref_keygen.cpp, built by oracle/keygen.mk): the unmodified
    reference's KeyGenerator under a seeded Blake2xb / Shake256 factory;
  * a restatement of KeyGenerator::generate_pk and generate_one_kswitch_key (keygenerator.cpp:96-120, 327-360) on top of
    tests/refprng.py's symmetric encryption: key level, NTT form for every scheme, plus the factor term
    (q_{k-1} mod q_j) s'_j on row j of digit j's c_0.
Under a fixed-seed factory every create() returns the same seed, so every bootstrap seed is {seed, 0, ..., 0}."""
import ctypes as C
import os

import numpy as np

import oracle as O
import refprng as P

_HERE = os.path.dirname(os.path.abspath(__file__))
_REF = os.path.join(_HERE, "..", "oracle", "_ref", "libsealref_keygen.so")
_u64p = C.POINTER(C.c_uint64)
_ref = None


def _p(a):
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(_u64p)


def ref_available():
    return os.path.exists(_REF)


def ref_lib():
    global _ref
    if _ref is None:
        L = C.CDLL(_REF)
        L.refkg_last_error.restype = C.c_char_p
        L.refkg_create.restype = C.c_void_p
        L.refkg_create.argtypes = [C.c_int, C.c_size_t, _u64p, C.c_size_t, C.c_uint64, C.c_uint64, C.c_int]
        L.refkg_destroy.argtypes = [C.c_void_p]
        L.refkg_secret_key.argtypes = [C.c_void_p, _u64p]
        L.refkg_public_key.argtypes = [C.c_void_p, _u64p]
        L.refkg_kswitch_key.restype = C.c_long
        L.refkg_kswitch_key.argtypes = [C.c_void_p, C.c_uint32, _u64p]
        L.refkg_galois_elts_all.restype = C.c_long
        L.refkg_galois_elts_all.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.c_size_t]
        _ref = L
    return _ref


def _chk(rc):
    if rc < 0:
        raise RuntimeError(ref_lib().refkg_last_error().decode())
    return rc


class RefKeygen:
    """the reference's SEALContext (sec_level none) with a Blake2xbPRNGFactory / Shake256PRNGFactory({seed, 0, ...}) and its
    KeyGenerator; the secret key is the one that KeyGenerator sampled"""

    def __init__(self, scheme, n, moduli, plain_modulus=0, seed=0x6B67, prng=P.BLAKE2XB):
        self.scheme, self.n, self.moduli, self.k, self.t, self.seed = scheme, n, list(moduli), len(moduli), plain_modulus, seed
        m = np.array(self.moduli, dtype=np.uint64)
        self.h = ref_lib().refkg_create(scheme, n, _p(m), self.k, plain_modulus, seed, prng)
        if not self.h:
            raise RuntimeError(ref_lib().refkg_last_error().decode())

    def __del__(self):
        if getattr(self, "h", None):
            ref_lib().refkg_destroy(self.h)
            self.h = None

    def boot_seeds(self, count):
        """the bootstrap seeds the fixed-seed factory hands out: count x {seed, 0, ..., 0}"""
        s = np.zeros((count, 8), dtype=np.uint64)
        s[:, 0] = self.seed
        return s

    def secret_key(self):
        out = np.zeros((self.k, self.n), dtype=np.uint64)
        _chk(ref_lib().refkg_secret_key(self.h, _p(out)))
        return out

    def public_key(self, keep=True):
        out = np.zeros((2, self.k, self.n), dtype=np.uint64) if keep else None
        _chk(ref_lib().refkg_public_key(self.h, None if out is None else _p(out)))
        return out

    def kswitch_key(self, galois_elt=0, keep=True):
        """create_relin_keys (galois_elt 0) / create_galois_keys({galois_elt}) -> [k-1][2][k][n] (keep=False: made and dropped)"""
        out = np.zeros((self.k - 1, 2, self.k, self.n), dtype=np.uint64) if keep else None
        _chk(ref_lib().refkg_kswitch_key(self.h, galois_elt, None if out is None else _p(out)))
        return out

    def galois_elts_all(self):
        buf = (C.c_uint32 * 256)()
        cnt = _chk(ref_lib().refkg_galois_elts_all(self.h, buf, 256))
        return [int(buf[i]) for i in range(cnt)]


# ---- the restatement ----
def galois_table_ntt(n, elt):
    """GaloisTool::generate_table_ntt (galois.cpp:18-51): apply_galois_ntt maps out[i] = in[table[i]]"""
    logn = n.bit_length() - 1

    def rev(x, bits):
        return int(format(x, f"0{bits}b")[::-1], 2) if bits else 0

    return np.array([rev(((elt * rev(i + n, logn + 1)) >> 1) & (n - 1), logn) for i in range(n)], dtype=np.int64)


class KeygenOracle:
    """KeyGenerator's public and key-switching keys for the context (scheme, n, moduli, t) from a secret key sk [k][n] (NTT form)"""

    def __init__(self, scheme, n, moduli, plain_modulus=0):
        self.scheme, self.n, self.q, self.k = scheme, n, list(moduli), len(moduli)
        # is_ntt_form = true for every scheme: BFV's key-level encryption is the NTT-form computation refprng restates for CKKS
        oc = O.Oracle(O.CKKS if scheme == O.BFV else scheme, n, moduli, 0 if scheme == O.CKKS or scheme == O.BFV else plain_modulus)
        self.po = P.PrngOracle(oc)

    def _zero(self, sk, seed, boot_prng, ct_prng):
        return self.po.encrypt_zero_symmetric(sk, np.asarray(seed, dtype=np.uint64), False, boot_prng, ct_prng, L=self.k)

    def public_key(self, sk, seed, boot_prng=P.BLAKE2XB, ct_prng=P.BLAKE2XB):
        return self._zero(sk, seed, boot_prng, ct_prng)

    def new_key(self, sk, galois_elt):
        """s' = s^2 (relinearization) or apply_galois_ntt(s, galois_elt)"""
        if galois_elt == 0:
            return np.stack([np.array([(int(a) * int(a)) % q for a in sk[j]], dtype=np.uint64) for j, q in enumerate(self.q)])
        return np.ascontiguousarray(sk[:, galois_table_ntt(self.n, galois_elt)])

    def kswitch_key(self, sk, galois_elt, seeds, boot_prng=P.BLAKE2XB, ct_prng=P.BLAKE2XB):
        """generate_one_kswitch_key: digit j = encryption of zero at the key level, row j of c_0 += (q_{k-1} mod q_j) s'_j"""
        s_new = self.new_key(sk, galois_elt)
        out = []
        for j in range(self.k - 1):
            ct = self._zero(sk, seeds[j], boot_prng, ct_prng)
            q, factor = self.q[j], self.q[-1] % self.q[j]
            ct[0, j] = np.array([(int(c) + factor * int(s)) % q for c, s in zip(ct[0, j], s_new[j])], dtype=np.uint64)
            out.append(ct)
        return np.stack(out)
