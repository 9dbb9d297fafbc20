"""CKKSEncoder::encode of one scalar (ckks.h:272-377), twice: restated with Python integers, and driven in the UNMODIFIED reference
through oracle/_ref/libsealref_scalar.so (oracle/ref_scalar.cpp).  TEST INFRASTRUCTURE ONLY.

The restatement covers the real and int64 kinds, whose plaintexts are constant polynomials (the same residue in every NTT-form word
of a prime's row); the complex kind is the vector encode of n/2 copies and is checked against that instead."""
import ctypes as C
import math
import os
from fractions import Fraction

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "..", "oracle", "_ref", "libsealref_scalar.so")

REAL, COMPLEX, INT64 = 0, 1, 2
_u64p = C.POINTER(C.c_uint64)
_lib = None


def available():
    return os.path.exists(_LIB_PATH)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(_LIB_PATH)
        L.refsc_last_error.restype = C.c_char_p
        L.refsc_create.restype = C.c_void_p
        L.refsc_create.argtypes = [C.c_size_t, _u64p, C.c_size_t]
        L.refsc_destroy.argtypes = [C.c_void_p]
        L.refsc_ckks_encode_scalar.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_double, _u64p, C.POINTER(C.c_double)]
        _lib = L
    return _lib


def scalar_bytes(kind, value):
    """the value's bytes as the C ABI takes them: one double, one (re, im) pair or one int64_t"""
    if kind == REAL:
        return np.array([value], dtype=np.float64)
    if kind == COMPLEX:
        return np.array([complex(value).real, complex(value).imag], dtype=np.float64)
    return np.array([value], dtype=np.int64)


class RefScalar:
    """a reference CKKS context of the given primes and its CKKSEncoder"""

    def __init__(self, n, moduli):
        self.n, self.moduli = n, list(moduli)
        m = np.array(self.moduli, dtype=np.uint64)
        self.h = lib().refsc_create(n, m.ctypes.data_as(_u64p), len(self.moduli))
        if not self.h:
            raise RuntimeError(lib().refsc_last_error().decode())

    def __del__(self):
        if getattr(self, "h", None):
            lib().refsc_destroy(self.h)
            self.h = None

    def encode(self, L, kind, value, scale=1.0):
        """-> (words [L][n], plaintext scale) or (None, the invalid_argument message); L outside 1..k encodes at parms_id_zero"""
        v = scalar_bytes(kind, value)
        out = np.zeros((max(L, 1), self.n), dtype=np.uint64)
        s = C.c_double(0)
        rc = lib().refsc_ckks_encode_scalar(self.h, L, kind, v.ctypes.data, float(scale), out.ctypes.data_as(_u64p), C.byref(s))
        if rc == 1:
            return None, lib().refsc_last_error().decode()
        if rc != 0:
            raise RuntimeError(lib().refsc_last_error().decode())
        return out, s.value


def total_bits(moduli):
    return math.prod(moduli).bit_length()


def _round_half_away(x):
    """std::round of a finite double, exactly"""
    a = Fraction(abs(x))
    r = math.floor(a)
    if a - r >= Fraction(1, 2):
        r += 1
    return -r if x < 0 else r


def restate(moduli, n, kind, value, scale=1.0):
    """-> (words [L][n], None) or (None, the reference's message) for the real and int64 kinds"""
    tb = total_bits(moduli)
    if kind == REAL:
        # ckks.cpp:96-124
        if not math.isfinite(scale) or scale <= 0 or int(math.log2(scale)) >= tb:
            return None, "scale out of bounds"
        if not math.isfinite(value):
            return None, "value must be finite"
        p = float(value) * float(scale)
        if not math.isfinite(p):
            return None, "encoded value is too large"
        bits = 2 if abs(p) < 1.0 else int(math.log2(abs(p))) + 2
        if bits >= tb:
            return None, "encoded value is too large"
        r = _round_half_away(p)
        negative = math.copysign(1.0, p) < 0  # signbit(round(p)): round keeps the sign, and -0 residues stay 0
        words = [(-abs(r)) % q if negative else abs(r) % q for q in moduli]
    elif kind == INT64:
        # ckks.cpp:253-284: |INT64_MIN| = 2^63; a negative v is reduced as the 64-bit word (uint64)v + q, which does not wrap for |v| > q
        v = int(value)
        mag = -v if v < 0 else v
        if mag.bit_length() + 2 >= tb:
            return None, "encoded value is too large"
        words = [(((v + (1 << 64)) + q) % (1 << 64)) % q if v < 0 else v % q for q in moduli]
    else:
        raise ValueError("the complex kind is the vector encode of n/2 copies; it has no restatement here")
    return np.repeat(np.array(words, dtype=np.uint64)[:, None], n, axis=1), None


def real_cases(tb):
    """(value, scale) pairs for a level of tb total bits: rounding, the three decomposition branches, the bit-count bound on both
    sides, the scale bounds of encode(double) and every error"""
    cases = [(0.49, 1.0), (-0.49, 1.0), (0.0, 1.0), (-0.0, 1.0), (0.5, 1.0), (-0.5, 1.0), (2.5, 1.0), (-2.5, 1.0), (1.5, 1.0),
             (3.14159, 2.0 ** 40), (-0.4, 2.0 ** 40), (1.0, 2.0 ** 40)]
    # products around 2^64 and 2^128: the reference's one-word, two-word and multi-precision branches
    for e in (63, 64, 127, 128, 129):
        for f in (1.0 - 2.0 ** -53, 1.0, 1.0 + 2.0 ** -52, 1.5):
            if int(math.log2(2.0 ** e * f)) + 2 < tb:
                cases += [(2.0 ** e * f, 1.0), (-(2.0 ** e) * f, 1.0)]
    if tb <= 1000:  # above that every finite double fits, and 2^tb is no double
        big = 2.0 ** (tb - 2)
        # the largest accepted bit count (tb - 1) and the one above, and the double below 2^(tb - 2), whose log2 rounds up to tb - 2
        cases += [(1.5 * big / 2, 1.0), (-1.5 * big / 2, 1.0), (big, 1.0), (-big, 1.0), (math.nextafter(big, 0.0), 1.0)]
        cases += [(2.0 ** -tb, 2.0 ** (tb - 1)), (0.0, 2.0 ** (tb - 1)), (1.0, 2.0 ** tb)]  # (int)log2(scale) = tb - 1 accepted, tb not
    cases += [(1.0, 5e-324), (1e300, 1e10), (1e-300, 1e300)]  # a subnormal scale; large products
    cases += [(1.0, 0.0), (1.0, -1.0), (1.0, math.inf), (1.0, math.nan), (math.inf, 1.0), (-math.inf, 1.0), (math.nan, 1.0),
              (1e300, 2.0 ** 40), (-1e300, 2.0 ** 40)]
    return cases


def int64_cases(moduli):
    """int64 values: 0, +-1, +-(q_j - 1), +-q_j, +-(q_j + 1) of every prime, INT64_MAX and INT64_MIN + 1 (INT64_MIN is kept apart:
    the reference takes llabs of it, which C leaves undefined)"""
    vals = [0, 1, -1, (1 << 63) - 1, -(1 << 63) + 1, -(1 << 40), 1 << 40]
    for q in moduli:
        vals += [q - 1, -(q - 1), q, -q, q + 1, -(q + 1)]
    return [v for v in dict.fromkeys(vals) if -(1 << 63) < v < (1 << 63)]
