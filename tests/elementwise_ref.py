"""The reference's release-build word semantics of the element-wise operations, stated on numpy uint64 arrays for ANY 64-bit input
words (the reference's own debug checks are compiled out there, so these are the words a caller gets back):

- add (add_poly_coeffmod, polyarithsmallmod.cpp:93-96): s = x + y mod 2^64, then s - q if s >= q;
- sub (sub_poly_coeffmod, :126-128; sub_uint_mod, uintarithsmallmod.h:156-158): the borrow form x - y mod 2^64, plus q when x < y,
  not reduced further;
- negate (negate_poly_coeffmod, polyarithsmallmod.h:95-105): q - x mod 2^64 for x != 0, else 0;
- the dyadic products and the tensor (dyadic_product_coeffmod, barrett_reduce_128 on any 128-bit value): every product exactly
  x y mod q, which equals (x mod q)(y mod q) mod q, and the sums of products added as canonical residues;
- multiply_plain: the same dyadic product against the plaintext;
- add_plain / sub_plain: add / sub on c_0 of the transformed plaintext (CKKS, BGV) or of round(Q m / t) mod q_i (BFV,
  scalingvariant.cpp:70-160, where the scaled word is canonical and c_0 is any word).

Words are [..., L, n] with the prime of row i = moduli[i] (axis -2).  Products are exact: a 128-bit product from 32-bit limbs,
reduced three bits at a time.  Test infrastructure only."""
import numpy as np

U64 = np.uint64
M32 = U64(0xFFFFFFFF)


def qcol(moduli, L):
    """the primes of rows 0..L-1 broadcast against [..., L, n]"""
    return np.array(moduli[:L], dtype=U64)[:, None]


def add(x, y, q):
    with np.errstate(over="ignore"):
        s = x + y
    return np.where(s >= q, s - q, s)


def sub(x, y, q):
    with np.errstate(over="ignore"):
        d = x - y
        return np.where(x < y, d + q, d)


def negate(x, q):
    with np.errstate(over="ignore"):
        return np.where(x != 0, q - x, U64(0))


def mul128(x, y):
    """(hi, lo) of the exact 128-bit product of two uint64 arrays"""
    x0, x1, y0, y1 = x & M32, x >> U64(32), y & M32, y >> U64(32)
    with np.errstate(over="ignore"):
        ll, lh, hl, hh = x0 * y0, x0 * y1, x1 * y0, x1 * y1
        mid = (ll >> U64(32)) + (lh & M32) + (hl & M32)
        lo = (ll & M32) | (mid << U64(32))
        hi = hh + (lh >> U64(32)) + (hl >> U64(32)) + (mid >> U64(32))
    return hi, lo


def reduce128(hi, lo, q):
    """(hi 2^64 + lo) mod q for q < 2^61: r < q keeps r 2^3 + 7 below 2^64"""
    r = hi % q
    r = ((r << U64(1)) | (lo >> U64(63))) % q
    for s in range(60, -1, -3):
        r = ((r << U64(3)) | ((lo >> U64(s)) & U64(7))) % q
    return r


def mulmod(x, y, q):
    """x y mod q for any 64-bit words (the reference's Barrett step on the 128-bit product)"""
    x, y = np.asarray(x, dtype=U64), np.asarray(y, dtype=U64)
    q = np.broadcast_to(np.asarray(q, dtype=U64), np.broadcast(x, y).shape)
    hi, lo = mul128(*np.broadcast_arrays(x, y))
    return reduce128(hi, lo, q)


def linear(mode, a, b, moduli):
    """add (0) / sub (1) / negate (2) of [..., L, n] words"""
    q = qcol(moduli, a.shape[-2])
    return add(a, b, q) if mode == 0 else sub(a, b, q) if mode == 1 else negate(a, q)


def tensor(a, b, moduli):
    """a [..., s1, L, n] times b [..., s2, L, n]: out[k] = sum_{i+j=k} a_i b_j mod q (operands of any 64-bit words)"""
    s1, s2, L = a.shape[-3], b.shape[-3], a.shape[-2]
    q = qcol(moduli, L)
    ar, br = a % q, b % q
    out = []
    for k in range(s1 + s2 - 1):
        acc = np.zeros(np.broadcast_shapes(a.shape[:-3], b.shape[:-3]) + a.shape[-2:], dtype=U64)
        for i in range(max(0, k - s2 + 1), min(k, s1 - 1) + 1):
            acc = add(acc, mulmod(ar[..., i, :, :], br[..., k - i, :, :], q), q)
        out.append(acc)
    return np.stack(out, axis=-3)


def multiply_plain(a, plain, moduli):
    """a [..., size, L, n] times the plaintext [..., L, n] (one per ciphertext, or one for every ciphertext)"""
    q = qcol(moduli, a.shape[-2])
    return mulmod(a, np.expand_dims(plain, -3), q)


def add_plain_c0(a, t, moduli, subtract):
    """c_0 +/- T for T [..., L, n] already in c_0's form (CKKS: the plaintext; BGV: its transform); the other polynomials untouched"""
    q = qcol(moduli, a.shape[-2])
    out = a.copy()
    out[..., 0, :, :] = sub(a[..., 0, :, :], t, q) if subtract else add(a[..., 0, :, :], t, q)
    return out


def bfv_scaled_plain(plain, moduli, L, t):
    """round(Q m / t) = floor((Q m + (t + 1) / 2) / t) mod q_i for plaintexts [..., n] of words below t -> [..., L, n]"""
    Q = 1
    for q in moduli[:L]:
        Q *= q
    h = (t + 1) // 2
    flat = plain.reshape(-1)
    vals = [(Q * int(m) + h) // t for m in flat]
    out = np.array([[v % q for v in vals] for q in moduli[:L]], dtype=U64)  # [L][count]
    return np.moveaxis(out.reshape((L,) + plain.shape), 0, -2)
