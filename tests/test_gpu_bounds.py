"""Parity at the arithmetic bounds (-m gpu).  Every other parity test draws its words uniformly from [0, q), which sits far from
the range arguments the kernels rest on: the integer key-switching path's CRT bound P > 4 L n max q^2 and its unreduced 64-bit
product sums (seal_b200/csrc/sb_ksint.cu), the lazy 128-bit sums of the 64-bit key-switching path, the 128-bit tensor sums, the
quotient of BFV plaintext scaling and the rounding of rescale / mod-switch.  Each test builds structured inputs (tests/common.py)
whose effect on its bound can be computed, asserts in Python integers that the inputs reach that bound, and compares every output
word with the oracle, the reference (tests/refseal.py) or a closed form checked against the oracle elsewhere."""
import numpy as np
import pytest

import oracle as O
import refseal as R
from common import alternating_ct, assert_words, const_ntt_row, is_prime, max_ct, negacyclic_ones_square, ntt_primes_below, rand_ct, unreduce, zero_ct

pytestmark = pytest.mark.gpu

KS_64, KS_AUTO, KS_INT = 0, 1, 2  # SB200_LIMIT_KS_ALGORITHM


def sb():
    import seal_b200

    return seal_b200


def mod_down(acc, acc_sp, q, qsp):
    """the mod-down by the special prime of switch_key_inplace (evaluator.cpp:2809-2864) on residues of the digit sum: acc = the
    sum mod q_i, acc_sp = the sum mod q_sp (Python ints or object arrays); the formula of
    test_host_logic.py::test_integer_key_switching_identity_vs_oracle"""
    half = qsp >> 1
    return ((acc - ((acc_sp + half) % qsp % q - half % q)) * pow(qsp, -1, q)) % q


def auxiliary_product(aux):
    P = 1
    for p in aux:
        P *= p
    return P


# ------------------------------------------------------------------------------------------------------------------------------
# Accumulator width of the integer path: ks32_mac / ks32_mac_tile sum L products of canonical 29-bit words in 64 bits without a
# reduction.  Batch entry b carries the constant polynomial (p_{b mod S} - 1) delta_0 in every digit; key row (J, c, I) carries
# (p_{I mod S} - 1) delta_0.  Their transforms modulo p_t are those constants at every point, so for b = I = t (mod S) the sum
# reaches L (p_t - 1)^2, the largest value the accumulators can see at this level; one call covers every auxiliary prime.  At
# n = 4096 the largest auxiliary prime is 536813569 and L (p - 1)^2 < 2^64 holds up to L = 64 digits: deeper levels must leave the
# integer path (Context::ksint_on).  The result of a constant input is a constant row per (b, c, i), in closed form below.  Up to
# 32 digits (k = 9, 33) the chunks of 16 ciphertexts take the INT8 tensor-core kernel, whose class sums the same rows drive to their largest
# values; at k = 33 a level below the key level (strided key rows) is checked against the closed form too.
@pytest.mark.parametrize("k", [9, 33, 41, 42, 64, 65, 66, 67, 256])
def test_integer_path_accumulator_width(k):
    S = sb()
    n, L = 4096, k - 1
    mods = O.coeff_modulus_create(n, [30] * k) if k <= 64 else ntt_primes_below(30, n, k)
    ctx = S.Context(S.CKKS, n, mods)
    aux = [int(p) for p in ctx.ksint_primes()]
    St = len(aux)
    assert aux and max(aux) < min(mods), "every constant below must be a canonical residue of every coefficient prime"
    max_digits = (2 ** 64 - 1) // (max(aux) - 1) ** 2
    assert max_digits == 64
    # 32: the host entry points cut a batch of 4 or more into at least two pipeline chunks, here two key-switching chunks of 16, where
    # the tensor-core product kernel runs up to 32 digits, the key-tile one up to 40; above, the register-tile one
    batch = 32 if k <= 67 else St
    cb = [aux[b % St] - 1 for b in range(batch)]
    kI = [aux[I % St] - 1 for I in range(k)]
    c3 = np.empty((batch, 3, L, n), dtype=np.uint64)
    c3[:, :2] = max_ct(mods, n, 2, L)
    for b in range(batch):
        c3[b, 2] = const_ntt_row(cb[b], n)
    key = np.ascontiguousarray(np.broadcast_to(np.array(kI, dtype=np.uint64)[None, None, :, None], (L, 2, k, n)))
    # the bound: the largest digit sum of products of transformed words, from the arrays themselves
    reach = max(sum((int(c3[b, 2, J, 0]) % p) * (int(key[J, 0, I, 0]) % p) for J in range(L))
                for t, p in enumerate(aux) for b in range(min(batch, St)) for I in range(min(k, St)))
    assert reach == L * (max(aux) - 1) ** 2
    if L > max_digits:
        assert reach >= 2 ** 64, "an unreduced 64-bit sum would wrap at this level"
    else:
        assert reach >= 0.98 * L / 64 * 2 ** 64
    # closed form: digit sum at prime I = L c_b K_I (a constant polynomial), mod-down, added to the NTT-form constant rows
    qsp = int(mods[k - 1])

    def closed_form(Lv):
        want = np.empty((batch, 2, Lv, n), dtype=np.uint64)
        for b in range(batch):
            acc_sp = Lv * cb[b] * kI[k - 1] % qsp
            for i in range(Lv):
                q = int(mods[i])
                r = mod_down(Lv * cb[b] * kI[i] % q, acc_sp, q, qsp)
                want[b, :, i, :] = (q - 1 + r) % q
        return want

    def relinearize_int(x, Lv):
        """the integer path, and from the profile which product kernel ran: no 32-bit multiply-accumulates = the tensor cores"""
        ctx.profile(True)
        out = ctx.relinearize(x, rk)
        macs = [r[7] for r in ctx.profile_read_work32() if r[0] == "ks32_mac"]
        ctx.profile(False)
        if Lv <= max_digits:
            assert macs and (sum(macs) == 0) == (Lv <= 32), f"L = {Lv}: the tensor-core kernel runs for L <= 32 digits and chunks of 16"
        else:
            assert not macs, f"L = {Lv}: levels past {max_digits} digits leave the integer path"
        return out

    want = closed_form(L)
    rk = ctx.load_key(key)
    got = {}
    for mode in (KS_INT, KS_AUTO, KS_64):
        ctx.set_limit(S.Context.LIMIT_KS_ALGORITHM, mode)
        got[mode] = relinearize_int(c3, L) if mode == KS_INT else ctx.relinearize(c3, rk)
        assert_words(got[mode], want, f"relinearize, k = {k}, key-switching mode {mode}, vs the closed form")
    if k == 33:
        Ll = k - 3
        ctx.set_limit(S.Context.LIMIT_KS_ALGORITHM, KS_INT)
        assert_words(relinearize_int(np.ascontiguousarray(c3[:, :, :Ll]), Ll), closed_form(Ll),
                     f"relinearize at L = {Ll} (key rows strided by k = {k}) vs the closed form")
    if k <= 64:
        oc = O.Oracle(O.CKKS, n, mods)
        for b in (0, St - 1):
            assert_words(got[KS_INT][b], oc.relinearize(L, c3[b], key), f"integer path vs oracle, batch entry {b}")
    del rk
    ctx.close()


# ------------------------------------------------------------------------------------------------------------------------------
# CRT margin of the integer path: digits and keys whose coefficients are all q - 1.  The negacyclic product of two such constant-
# coefficient polynomials is (q_J - 1)(q_I - 1)(2x + 2 - n), so the digit sum reaches +sum_J (q_J - 1)(q_I - 1) n at x = n - 1,
# right at the bound P > 4 L n max q^2 the auxiliary primes are chosen for.  Shapes: 2.0 bits of margin (n = 65536, 32 primes),
# the tightest five-prime case (n = 131072, 61 primes of 60 bits) and six auxiliary primes (62 primes), never run before.
def _all_max_key(ctx, mods, n, L):
    k = len(mods)
    K = ctx.transform_to_ntt(max_ct(mods, n, 1, k))[0]  # NTT form of the all-(q - 1) polynomial at every key prime
    return np.ascontiguousarray(np.broadcast_to(K[None, None], (L, 2, k, n)))


def _check_crt_reach(ctx, mods, n, L):
    aux = [int(p) for p in ctx.ksint_primes()]
    P, qmax = auxiliary_product(aux), max(int(q) for q in mods)
    assert P > 4 * L * n * qmax ** 2
    qsp = int(mods[-1])
    reach = sum((int(q) - 1) for q in mods[:L]) * (qsp - 1) * n  # |c_sp| at x = n - 1
    assert reach >= 0.99 * L * n * (qmax - 1) ** 2
    return aux


@pytest.mark.parametrize("n,k", [(65536, 32), (131072, 61), (131072, 62)])
def test_crt_margin_bfv_closed_form(n, k):
    """BFV relinearize (coefficient-form target): the integer path equals the 64-bit path and, at every coefficient, the
    Python-integer mod-down of the exact digit sum"""
    S = sb()
    mods = O.coeff_modulus_create(n, [60] * k)
    L = k - 1
    ctx = S.Context(S.BFV, n, mods, 65537)
    aux = _check_crt_reach(ctx, mods, n, L)
    assert len(aux) == {65536: 5, 131072: 5 if k == 61 else 6}[n]
    c3 = zero_ct(mods, n, 3, L, batch=1)
    c3[0, 2] = max_ct(mods, n, 1, L)[0]
    rk = ctx.load_key(_all_max_key(ctx, mods, n, L))
    ctx.set_limit(S.Context.LIMIT_KS_ALGORITHM, KS_INT)
    got_int = ctx.relinearize(c3, rk)
    ctx.set_limit(S.Context.LIMIT_KS_ALGORITHM, KS_64)
    got_64 = ctx.relinearize(c3, rk)
    assert_words(got_int, got_64, "integer path vs 64-bit path")
    qsp = int(mods[k - 1])
    f = np.array(negacyclic_ones_square(n), dtype=object)
    sJ = sum(int(q) - 1 for q in mods[:L])
    acc_sp = (sJ * (qsp - 1) * f) % qsp
    for i in range(L):
        q = int(mods[i])
        r = mod_down((sJ * (q - 1) * f) % q, acc_sp, q, qsp)
        for c in range(2):
            assert_words(got_int[0, c, i], r.astype(np.uint64), f"component {c}, prime {i}, vs the closed form")
    del rk
    ctx.close()


@pytest.mark.parametrize("scheme_name", ["CKKS", "BGV"])
def test_crt_margin_ntt_schemes_vs_oracle(scheme_name):
    """CKKS / BGV relinearize and one rotation at n = 65536 with 32 primes of 60 bits, digits and keys all-(q - 1) polynomials:
    integer path = 64-bit path = oracle, every word"""
    S = sb()
    n, k = 65536, 32
    mods = O.coeff_modulus_create(n, [60] * k)
    L = k - 1
    t = 65537 if scheme_name == "BGV" else 0
    ctx = S.Context(getattr(S, scheme_name), n, mods, t) if t else S.Context(S.CKKS, n, mods)
    oc = O.Oracle(getattr(O, scheme_name), n, mods, t) if t else O.Oracle(O.CKKS, n, mods)
    _check_crt_reach(ctx, mods, n, L)
    key = _all_max_key(ctx, mods, n, L)
    rk = ctx.load_key(key)
    top = ctx.transform_to_ntt(max_ct(mods, n, 1, L))[0]
    c3 = np.stack([alternating_ct(mods, n, 1, L)[0], max_ct(mods, n, 1, L)[0], top])[None]
    elt = O.galois_elt_from_step(n, 1)
    out = {}
    for mode in (KS_INT, KS_64):
        ctx.set_limit(S.Context.LIMIT_KS_ALGORITHM, mode)
        out[mode] = (ctx.relinearize(c3, rk), ctx.apply_galois(np.ascontiguousarray(c3[:, 1:]), elt, rk))
    assert_words(out[KS_INT][0][0], oc.relinearize(L, c3[0], key), "relinearize, integer path vs oracle")
    assert_words(out[KS_64][0], out[KS_INT][0], "relinearize, 64-bit path vs integer path")
    assert_words(out[KS_INT][1][0], oc.apply_galois(L, np.ascontiguousarray(c3[0, 1:]), elt, key), "apply_galois vs oracle")
    assert_words(out[KS_64][1], out[KS_INT][1], "apply_galois, 64-bit path vs integer path")
    del rk
    ctx.close()


def test_auxiliary_primes_equal_to_coefficient_primes():
    """29-bit coefficient primes at n = 4096 are exactly the auxiliary primes (both are the largest primes = 1 mod 2n below
    2^29); bit-exactness must not depend on the two sets being disjoint (DESIGN.md 3.2).  All-(q - 1) digits and keys."""
    S = sb()
    n, k = 4096, 9
    mods = O.coeff_modulus_create(n, [29] * k)
    L = k - 1
    ctx = S.Context(S.CKKS, n, mods)
    oc = O.Oracle(O.CKKS, n, mods)
    aux = [int(p) for p in ctx.ksint_primes()]
    assert set(aux) <= set(int(q) for q in mods)
    key = np.ascontiguousarray(np.broadcast_to(ntt_rows(oc, max_ct(mods, n, 1, k)[0])[None, None], (L, 2, k, n)))
    rk = ctx.load_key(key)
    rng = np.random.default_rng(29)
    c3 = rand_ct(rng, mods, n, 3, L, batch=2)
    c3[:, 2] = ntt_rows(oc, max_ct(mods, n, 1, L)[0])
    for mode in (KS_INT, KS_64):
        ctx.set_limit(S.Context.LIMIT_KS_ALGORITHM, mode)
        got = ctx.relinearize(c3, rk)
        for b in range(2):
            assert_words(got[b], oc.relinearize(L, c3[b], key), f"mode {mode}, batch entry {b}")


# ------------------------------------------------------------------------------------------------------------------------------
# The 64-bit key-switching path (ks_local_mac_kernel) at its lazy limits, all-(q - 1) digits and keys: the guard-free forward
# butterflies at the largest primes they allow (< 2^57), the guarded path (60 bits), and digit primes just above / below four
# times the smallest output prime (the digit re-reduction on / off).
def _reduction_pair(n, above):
    """[digit prime next to 4 q_min, a 50-bit digit prime, q_min = the special prime]"""
    p1, p2 = O.coeff_modulus_create(n, [50, 50])
    qmin = min(p1, p2)
    c = (4 * qmin) // (2 * n) * (2 * n) + 1
    step = 2 * n if above else -2 * n
    while not (is_prime(c) and (c >= 4 * qmin) == above):
        c += step
    return [c, max(p1, p2), qmin]


def ntt_rows(oc, a):
    """oracle NTT of a coefficient-form [rows][n] array, row i modulo prime i"""
    return np.stack([oc.ntt_row(i, r) for i, r in enumerate(a)])


@pytest.mark.parametrize("case", ["fast57", "guarded60", "reduce_on", "reduce_off"])
def test_64bit_path_lazy_limits_vs_oracle(case):
    S = sb()
    n = 4096
    mods = {"fast57": lambda: O.coeff_modulus_create(n, [56, 56, 57, 57]), "guarded60": lambda: O.coeff_modulus_create(n, [60] * 4),
            "reduce_on": lambda: _reduction_pair(n, True), "reduce_off": lambda: _reduction_pair(n, False)}[case]()
    k, L = len(mods), len(mods) - 1
    qmax = max(mods[:L])
    qmin = min(mods)
    if case == "fast57":
        assert max(mods).bit_length() == 57  # the largest primes of the guard-free forward butterflies
    elif case == "guarded60":
        assert min(mods).bit_length() == 60
    else:
        assert ((qmax >> 2) >= qmin) == (case == "reduce_on") and abs(qmax / (4 * qmin) - 1) < 1e-6
    ctx = S.Context(S.CKKS, n, mods)
    oc = O.Oracle(O.CKKS, n, mods)
    key = np.ascontiguousarray(np.broadcast_to(ntt_rows(oc, max_ct(mods, n, 1, k)[0])[None, None], (L, 2, k, n)))
    rk = ctx.load_key(key)
    c3 = max_ct(mods, n, 3, L, batch=2)
    c3[0, 2] = ntt_rows(oc, max_ct(mods, n, 1, L)[0])
    ctx.set_limit(S.Context.LIMIT_KS_ALGORITHM, KS_64)
    got = ctx.relinearize(c3, rk)
    for b in range(2):
        assert_words(got[b], oc.relinearize(L, c3[b], key), f"{case}, batch entry {b}")


# ------------------------------------------------------------------------------------------------------------------------------
# Tensors: 60-bit primes, canonical words at q - 1, and every word replaced by its LARGEST 64-bit representative (near 2^64).
# The reference's dyadic products accept any representative (dyadic_product_coeffmod + add_poly_coeffmod, evaluator.cpp:692); two
# products of raw words near 2^64 already overflow a 128-bit sum, so the kernels must canonicalise on the way in.
@pytest.mark.parametrize("s1,s2", [(2, 2), (3, 3), (2, 15), (8, 8)])
def test_tensor_sizes_at_word_limits(s1, s2):
    S = sb()
    n, batch = 4096, 2
    mods = O.coeff_modulus_create(n, [60, 60, 60])
    L = 2
    ctx = S.Context(S.CKKS, n, mods)
    oc = O.Oracle(O.CKKS, n, mods)
    rng = np.random.default_rng(100 * s1 + s2)
    cases = {"all q-1": (max_ct(mods, n, s1, L, batch), max_ct(mods, n, s2, L, batch)),
             "alternating x q-1": (alternating_ct(mods, n, s1, L, batch), max_ct(mods, n, s2, L, batch)),
             "random": (rand_ct(rng, mods, n, s1, L, batch), rand_ct(rng, mods, n, s2, L, batch))}
    m = min(s1, s2)
    qmax = max(mods)
    assert m * (qmax - 1) ** 2 < 2 ** 128 and m * (qmax - 1) ** 2 >= m * 0.99 * 2 ** 120  # canonical sums: inside, near 2^(120+log m)
    for name, (a, b) in cases.items():
        ua, ub = unreduce(a, mods), unreduce(b, mods)
        assert int(ua.min()) >= 2 ** 64 - qmax and 2 * int(ua.min()) ** 2 >= 2 ** 128, "two raw products would overflow 128 bits"
        want = [oc.multiply(L, a[i], b[i]) for i in range(batch)]
        for label, x, y in (("canonical", a, b), ("largest representatives", ua, ub)):
            got = ctx.multiply(x, y)
            for i in range(batch):
                assert_words(got[i], want[i], f"{s1}x{s2} multiply, {name}, {label}, batch entry {i}")
        if (s1, s2) == (2, 2):
            plain = a[:, 0]
            got_s, got_p = ctx.square(ua), ctx.multiply_plain(ua, unreduce(plain, mods))
            for i in range(batch):
                assert_words(got_s[i], oc.multiply(L, a[i], a[i]), f"square, {name}, batch entry {i}")
                assert_words(got_p[i], oc.multiply_plain(L, a[i], plain[i]), f"multiply_plain, {name}, batch entry {i}")
        if R.available():
            rc = R.RefContext(O.CKKS, n, mods)
            assert_words(rc.multiply(L, ua[0], ub[0]), want[0], "the reference is insensitive to the representative")


# ------------------------------------------------------------------------------------------------------------------------------
# BFV plaintext scaling with a 60-bit plain modulus: the 128-bit quotient floor((m (q mod t) + (t + 1) / 2) / t) of
# bfv_add_plain_kernel at m = t - 1, 0 and the two words around t / 2; one coefficient prime below t, two above.
def test_bfv_add_sub_plain_60bit_plain_modulus():
    S = sb()
    n, batch = 4096, 2
    mods = O.coeff_modulus_create(n, [40, 60, 60, 60])
    t = max(mods) - 2  # the largest prime below the largest coefficient prime: 60 bits, above the 40-bit prime
    while not is_prime(t) or t in mods:
        t -= 2
    assert t.bit_length() == 60 and min(mods) < t < max(mods)
    L = len(mods) - 1
    ctx = S.Context(S.BFV, n, mods, t)
    oc = O.Oracle(O.BFV, n, mods, t)
    words = np.array([t - 1, 0, (t - 1) // 2, (t + 1) // 2], dtype=np.uint64)
    plain = np.stack([np.resize(np.roll(words, b), n) for b in range(batch)])
    Q = 1
    for q in mods[:L]:
        Q *= int(q)
    assert (t - 1) * (Q % t) + (t + 1) // 2 >= 2 ** 100, "the scaling quotient needs the 128-bit path"
    rng = np.random.default_rng(60)
    for a in (rand_ct(rng, mods, n, 2, L, batch), max_ct(mods, n, 2, L, batch)):
        for sub in (False, True):
            got = ctx.add_plain_coeff(a, plain, subtract=sub)
            for b in range(batch):
                assert_words(got[b], oc.add_plain_coeff(L, a[b], plain[b], subtract=sub), f"subtract={sub}, batch entry {b}")


# ------------------------------------------------------------------------------------------------------------------------------
# Rescale (CKKS) and mod-switch (BFV, BGV): the last prime's coefficient-form words at 0, q - 1 and floor(q_top / 2) +- 1, where
# the rounding of the division by q_top turns; a 60-bit top prime above 40- and 50-bit ones, and a 50-bit top prime.
@pytest.mark.parametrize("scheme_name", ["CKKS", "BFV", "BGV"])
def test_rescale_mod_switch_at_rounding_edges(scheme_name):
    S = sb()
    n = 4096
    mods = O.coeff_modulus_create(n, [40, 50, 60, 60])
    t = 65537 if scheme_name != "CKKS" else 0
    ctx = S.Context(getattr(S, scheme_name), n, mods, t) if t else S.Context(S.CKKS, n, mods)
    oc = O.Oracle(getattr(O, scheme_name), n, mods, t) if t else O.Oracle(O.CKKS, n, mods)
    rng = np.random.default_rng(7)
    for L in (3, 2):
        qt = int(mods[L - 1])
        h = qt // 2
        edge = np.resize(np.array([0, qt - 1, h - 1, h, h + 1], dtype=np.uint64), n)
        assert {0, qt - 1, h - 1, h + 1} <= set(int(v) for v in edge[:5])
        a = rand_ct(rng, mods, n, 2, L)
        a[0, L - 1] = edge
        a[1, L - 1] = np.roll(edge, 2)
        if scheme_name != "BFV":  # NTT-form ciphertexts: the edges are the top prime's coefficient-form words
            a[:, L - 1] = np.stack([oc.ntt_row(L - 1, r) for r in a[:, L - 1]])
        if scheme_name == "CKKS":
            got, want = ctx.rescale_to_next(a), oc.rescale(L, a)
        else:
            got = ctx.mod_switch_to_next(a)
            want = oc.bfv_mod_switch(L, a) if scheme_name == "BFV" else oc.bgv_mod_switch(L, a)
        assert_words(got, want, f"{scheme_name}, level {L}")
