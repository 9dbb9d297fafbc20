"""Decryptor::invariant_noise_budget (decryptor.cpp:409-486) restated in Python integers, the reference's own value through
oracle/ref_noise.cpp (oracle/_ref/libsealref_noise.so, built by oracle/noise.mk), and ciphertexts with a chosen phase.  Shared by
test_noise_oracle.py (CPU) and test_gpu_noise.py (GPU)."""
import ctypes as C
import os

import numpy as np

import oracle as O
import refseal as R

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref", "libsealref_noise.so")
_u64p = C.POINTER(C.c_uint64)
_lib = None


def available():
    """the reference library and its noise-budget wrapper are both built"""
    return R.available() and os.path.exists(_LIB_PATH)


def _noise_lib():
    global _lib
    if _lib is None:
        L = C.CDLL(_LIB_PATH)
        L.sealnoise_last_error.restype = C.c_char_p
        L.sealnoise_create.restype = C.c_void_p
        L.sealnoise_create.argtypes = [C.c_int, C.c_size_t, _u64p, C.c_size_t, C.c_uint64, _u64p]
        L.sealnoise_destroy.argtypes = [C.c_void_p]
        L.sealnoise_budget.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, _u64p, C.POINTER(C.c_int)]
        _lib = L
    return _lib


class _NoiseRef:
    """the reference's Decryptor under the secret key of a RefContext"""

    def __init__(self, rc):
        m = np.array(rc.moduli, dtype=np.uint64)
        sk = np.ascontiguousarray(rc.secret_key(), dtype=np.uint64)
        self.h = _noise_lib().sealnoise_create(rc.scheme, rc.n, m.ctypes.data_as(_u64p), len(rc.moduli), rc.plain_modulus,
                                               sk.ctypes.data_as(_u64p))
        if not self.h:
            raise RuntimeError(_noise_lib().sealnoise_last_error().decode())

    def __del__(self):
        if getattr(self, "h", None):
            _noise_lib().sealnoise_destroy(self.h)


def _obj(a):
    return np.asarray(a, dtype=np.uint64).astype(object)


def restated_budget(scheme, n, mods, t, sk_ntt, ct):
    """steps 2-6 of the reference on one ciphertext [size][L][n] (BFV coefficient form, BGV NTT form); sk_ntt = [k][n] secret key
    in NTT form at the key level"""
    ct = np.ascontiguousarray(ct, dtype=np.uint64)
    size, L = ct.shape[0], ct.shape[1]
    q = [int(x) for x in mods[:L]]
    orc = O.Oracle(O.CKKS, n, mods)  # the transforms depend on the primes only
    polys = ct[1:] if scheme == R.BGV else orc.ntt_forward(L, ct[1:])
    phase = []
    for i in range(L):
        s, sp, acc = _obj(sk_ntt[i]), None, np.zeros(n, dtype=object)
        for p in range(size - 1):  # dot_product_ct_sk_array: sum_{p>=1} c_p s^p in NTT form
            sp = s if sp is None else (sp * s) % q[i]
            acc = (acc + _obj(polys[p, i]) * sp) % q[i]
        phase.append(acc)
    phase = np.array([[int(x) for x in row] for row in phase], dtype=object)
    if scheme == R.BGV:
        phase = (phase + _obj(ct[0])) % np.array(q, dtype=object)[:, None]
    inv = orc.ntt_inverse(L, np.array(phase.astype(np.uint64))[None])[0]
    phase = _obj(inv)
    if scheme == R.BFV:
        phase = (phase + _obj(ct[0])) % np.array(q, dtype=object)[:, None]
        phase = (phase * int(t)) % np.array(q, dtype=object)[:, None]
    Q = 1
    for x in q:
        Q *= x
    v = np.zeros(n, dtype=object)
    for i in range(L):  # compose_array: Python big-int CRT
        m = Q // q[i]
        v = (v + phase[i] * (m * pow(m % q[i], -1, q[i]))) % Q
    thr = (Q + 1) // 2
    norm = max(int(Q - x) if x >= thr else int(x) for x in v)
    return max(0, Q.bit_length() - norm.bit_length() - 1)


def ref_budget(rc, L, ct, is_ntt_form):
    """(status, budget or message) of the reference's Decryptor::invariant_noise_budget under rc's parameters and secret key"""
    ref = getattr(rc, "_noise_ref", None)
    if ref is None:  # created once per RefContext and released with it
        ref = rc._noise_ref = _NoiseRef(rc)
    lib = _noise_lib()
    ct = np.ascontiguousarray(ct, dtype=np.uint64)
    out = C.c_int(-7)
    status = lib.sealnoise_budget(ref.h, L, ct.shape[0], int(is_ntt_form), ct.ctypes.data_as(_u64p), C.byref(out))
    return (0, out.value) if status == 0 else (status, lib.sealnoise_last_error().decode())


def structured_ct(scheme, n, mods, t, L, size, values):
    """a ciphertext [size][L][n] with c_1 = ... = 0 whose composed noise is exactly `values` (n Python ints, signed): BGV c_0 =
    NTT(v), BFV c_0 = v t^-1 mod Q"""
    q = [int(x) for x in mods[:L]]
    ct = np.zeros((size, L, n), dtype=np.uint64)
    for i in range(L):
        inv_t = pow(int(t) % q[i], -1, q[i]) if scheme == R.BFV else 1
        ct[0, i] = np.array([(int(v) * inv_t) % q[i] for v in values], dtype=np.uint64)
    if scheme == R.BGV:
        ct[0] = O.Oracle(O.CKKS, n, mods).ntt_forward(L, ct[:1])[0]
    return ct


def total_bits(mods, L):
    Q = 1
    for x in mods[:L]:
        Q *= int(x)
    return Q, Q.bit_length()


def edge_values(Q, bits):
    """the noise magnitudes at the edges: 0, +-1, +-2^j at the word edges and at total_bits - 2, the centring edge, Q - 1"""
    out = [0, 1, -1]
    for j in (63, 64, 65, 127, 128, bits - 2):
        if 0 < j < bits - 1:
            out += [1 << j, -(1 << j)]
    out += [(Q - 1) // 2, (Q + 1) // 2, Q - 1]
    return out
