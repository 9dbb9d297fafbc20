"""Parity matrix of the 64-bit key-switching path (-m gpu; key_switch_chunk in seal_b200/csrc/sb_engine.cu, DESIGN 3.2b).  It
serves every ring below n = 4096, every level with fewer than 16 digits, and every level deeper than the integer path's
max_digits, in every mode.  The axes crossed on purpose, every group with LIMIT_KS_ALGORITHM = 0 and again in the automatic mode
(which takes this path at all these levels; the profile shows no ks32_* kernel):

- transform size: n = 2, 8, 64, 128, 256, 512, 2048 (ntt_fwd_small with clamp(n / 2, 32, 256) threads, then ks_mac_kernel) and
  4096 .. 131072 (ks_digit_col_kernel at every LOGNA 4 .. 9, then ks_local_mac_kernel);
- butterfly class: every prime below 2^57 (FAST), or a set with 60- and 61-bit primes (guarded);
- digit-row class, the decision of key_switch_chunk restated in row_class(): plain rows (ks_digit_col_kernel<.., PLAIN = true>),
  digits re-reduced (a data prime at least 4x the smallest output prime; also sets right at that edge), or a Galois view (BFV
  rotations read the target through a signed automorphism);
- target: a plain slab (relinearize, multiply_relinearize: ks_local_mac_kernel<FAST, true>) or a Galois view (apply_galois);
- scheme: CKKS (OpModDownFwd), BGV (OpTopIntt with K + OpModDownFwdBgv) with t below the data primes and above them, BFV
  (OpProdIntt + moddown_coeff_kernel on a coefficient-form target);
- epilogue base: BaseSrc (relinearize, apply_galois) and BaseAddSrc (apply_galois_add, with a fresh output and out = addend);
- operation: relinearize at sizes 3, 4 and 16 (op_relinearize_sized), multiply_relinearize (the tensor written into scratch),
  apply_galois with steps +1, -1, n/4 - 1 and the element 2n - 1;
- level: the key level L = k - 1 (re-reduced digits) and L = k - 3 (plain digit rows; key rows at a stride of k);
- chunks: LIMIT_KS_CHUNK = 2 on 5 ciphertexts, so that a batch ends in a ragged chunk;
- words: member j draws pattern j mod 3 -- uniform, every word q - 1, and the target (q_min - 1) delta_0 (a constant digit, the
  extreme of the digit sums when keys are q_I - 1).

Every member of every batch is compared word for word with the oracle (tests/oracle.py), and the automatic mode with the forced
one.  The last test asserts that the module reached exactly the (size class, FAST, digit-row class, target, scheme, base) tuples of
expected_coverage().

test_digit_sum_bound is the 128-bit bound of the digit sums at 61-bit primes: L (q - 1)^2 reaches 2^128 past 64 digits, where
ks_mac_kernel / ks_local_mac_kernel reduce once every kKsSumWindow digits (tests/test_ks64_bounds.py)."""
import itertools
import os
from collections import namedtuple
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import oracle as O
from common import assert_words, is_prime, ntt_primes_below
from test_gpu_bounds import _reduction_pair, mod_down

pytestmark = pytest.mark.gpu

KS_64, KS_AUTO = 0, 1  # SB200_LIMIT_KS_ALGORITHM
SIZES = (2, 8, 64, 128, 256, 512, 2048, 4096, 8192, 16384, 32768, 65536, 131072)
# k = 5: the key level (L = 4) holds a 50-bit prime under 4x smaller than the others (digits re-reduced); L = 2 holds the two
# largest primes of one size with the special prime (plain digit rows).  BFV's guarded set stays at 60 bits: its BEHZ base takes
# the largest 61-bit primes = 1 mod 2n, the very prime the 61-bit set would share with it
BITS = {True: [57, 56, 50, 55, 57], False: [61, 60, 50, 58, 60]}
BITS_BFV_GUARDED = [60, 59, 50, 58, 60]
BATCH, CHUNK = 5, 2  # chunks 2, 2, 1
GALOIS = ("galois(+1)", "galois(-1)", "galois(n/4-1)", "galois(2n-1)")
REL, MULREL, GAL, GAL_ADD, GAL_ADD_INPLACE = "relinearize", "multiply_relinearize", "apply_galois", "apply_galois_add", "apply_galois_add(out=addend)"
SCHEMES = ("CKKS", "BGV-t-below", "BGV-t-above", "BFV")
PATTERNS = ("uniform", "max", "const")

Group = namedtuple("Group", "n scheme fast mods t levels size galois")


def sb():
    import seal_b200

    return seal_b200


def prime_below(bound):
    c = bound - 1
    while not is_prime(c):
        c -= 1
    return c


def size_class(n):
    """ntt_fwd_small with clamp(n / 2, 32, 256) threads + ks_mac_kernel below n = 4096, else ks_digit_col_kernel<LOGNA = log2(n) - 8>
    + ks_local_mac_kernel"""
    logn = n.bit_length() - 1
    return f"small{min(max(n // 2, 32), 256)}" if logn < 12 else f"LOGNA{logn - 8}"


def row_class(scheme, mods, L, galois):
    """key_switch_chunk's digit rows: re-reduced when a digit prime reaches 4x an output prime ((qmax >> 2) >= qmin over the L data
    primes and the special prime); else a Galois view for BFV rotations (CKKS / BGV apply the permutation in the target's inverse
    transform, so their digit rows stay plain); else plain"""
    qmax, qmin = max(mods[:L]), min(list(mods[:L]) + [mods[-1]])
    if (qmax >> 2) >= qmin:
        return "reduce"
    return "view" if scheme == "BFV" and galois else "plain"


def plain_modulus(scheme, mods):
    if scheme == "BGV-t-below":
        return 65537
    if scheme == "BGV-t-above":
        return prime_below(2 ** 60)  # above every prime of the FAST sets
    return 65537 if scheme == "BFV" else 0


def _groups():
    """every transform size x scheme x butterfly class (BGV with t above the data primes only for the FAST sets, whose primes sit
    below 2^57), the relinearize size and the Galois step rotating; then sets right at the re-reduction edge"""
    out, i = [], 0
    for n in SIZES:
        for scheme, fast in itertools.product(SCHEMES, (True, False)):
            if scheme == "BGV-t-above" and not fast:
                continue
            mods = O.coeff_modulus_create(n, BITS_BFV_GUARDED if scheme == "BFV" and not fast else BITS[fast])
            out.append(Group(n, scheme, fast, tuple(mods), plain_modulus(scheme, mods), (4, 2), (3, 4, 16)[i % 3], GALOIS[i % 4]))
            i += 1
    # [digit prime next to 4 q_min, a 50-bit digit prime, q_min]: re-reduction on just above the edge, off just below it
    for n, scheme, above in ((64, "CKKS", True), (64, "BFV", False), (8192, "CKKS", False), (8192, "BFV", True), (2048, "BGV-t-below", True)):
        mods = _reduction_pair(n, above)
        out.append(Group(n, scheme, True, tuple(mods), plain_modulus(scheme, mods), (2,), 3, GALOIS[i % 4]))
        i += 1
    return out


def _group_id(g):
    edge = "" if len(g.mods) == 5 else "-edge"
    return f"n{g.n}-{g.scheme}-{'fast' if g.fast else 'guarded'}{edge}-size{g.size}-{g.galois}"


GROUPS = _groups()
GROUP_IDS = [_group_id(g) for g in GROUPS]
COVERAGE, DONE = set(), set()


def expected_coverage():
    """every size class x scheme x butterfly class (BGV with t above the data primes: FAST only), each with plain and re-reduced
    digit rows, a plain target and a Galois view, BaseSrc and (under the view) BaseAddSrc; BFV rotations with the view as their row
    class where no re-reduction is needed"""
    out = set()
    for cls, scheme, fast in itertools.product({size_class(n) for n in SIZES}, SCHEMES, (True, False)):
        if scheme == "BGV-t-above" and not fast:
            continue
        for rows in ("plain", "reduce"):
            out.add((cls, fast, rows, "plain", scheme, "src"))
            g_rows = "view" if scheme == "BFV" and rows == "plain" else rows
            out |= {(cls, fast, g_rows, "galois", scheme, base) for base in ("src", "add")}
    return out


def galois_elt(op, n):
    if n == 2:  # one slot: the only element besides the identity is 2n - 1 = 3
        return 2 * n - 1
    return {"galois(+1)": lambda: O.galois_elt_from_step(n, 1), "galois(-1)": lambda: O.galois_elt_from_step(n, -1),
            "galois(n/4-1)": lambda: O.galois_elt_from_step(n, n // 4 - 1), "galois(2n-1)": lambda: 2 * n - 1}[op]()


def const_target(mods, n, L, ntt):
    """(q_min - 1) delta_0 at every prime: its NTT form is the word q_min - 1 at every point"""
    c = min(int(q) for q in mods) - 1
    row = np.full(n, c, dtype=np.uint64) if ntt else np.concatenate([[c], np.zeros(n - 1)]).astype(np.uint64)
    return np.broadcast_to(row, (L, n)).copy()


def draw(rng, mods, n, size, L, pattern, ntt):
    """one member's [size][L][n] words: the pattern's target in the last polynomial, every other polynomial uniform or q - 1"""
    if pattern == "uniform":
        return np.stack([np.stack([rng.integers(0, mods[i], n, dtype=np.uint64) for i in range(L)]) for _ in range(size)])
    x = np.stack([np.stack([np.full(n, mods[i] - 1, dtype=np.uint64) for i in range(L)]) for _ in range(size)])
    if pattern == "const":
        x[-1] = const_target(mods, n, L, ntt)
    return x


def to_dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def to_np(t):
    return t.cpu().numpy().view(np.uint64)


def run_op(ctx, rk, op, elt, args, L, B):
    """the device entry points (relinearize of size > 3 through the host one, op_relinearize_sized); [B][out size][L][n]"""
    import torch

    if op == REL and args[0].shape[1] > 3:
        return ctx.relinearize_step(args[0], rk)
    d = [to_dev(a) for a in args]
    out = torch.empty((B, 2, L, ctx.n), dtype=torch.int64, device="cuda")
    if op == REL:
        ctx.d_relinearize(d[0], rk, out, L, B)
    elif op == MULREL:
        ctx.d_multiply_relinearize(d[0], d[1], rk, out, L, B)
    elif op == GAL:
        ctx.d_apply_galois(d[0], elt, rk, out, L, B)
    elif op == GAL_ADD:
        ctx.d_apply_galois_add(d[0], elt, rk, d[1], out, L, B)
    else:
        ctx.d_apply_galois_add(d[0], elt, rk, d[1], d[1], L, B)
        out = d[1]
    torch.cuda.synchronize()
    return to_np(out)


def oracle_op(oc, op, elt, args, L, key, mods):
    if op == REL:
        c = args[0]
        out = c.copy()
        out[:2] = oc.relinearize(L, np.ascontiguousarray(np.stack([c[0], c[1], c[-1]])), key)
        return out if len(c) > 3 else out[:2]  # op_relinearize_sized keeps the size; size 3 returns two polynomials
    if op == MULREL:
        return oc.multiply_relin(L, args[0], args[1], key)
    g = oc.apply_galois(L, args[0], elt, key)
    if op == GAL:
        return g
    q = np.array([int(x) for x in mods[:L]], dtype=object)[None, :, None]
    return ((g.astype(object) + args[1].astype(object)) % q).astype(np.uint64)


def check_profile(prof, n, bfv, chunks, what):
    names = [r[0].split(":")[0] for r in prof]
    assert not [x for x in names if x.startswith("ks32")], f"{what}: the integer path ran: {sorted(set(names))}"
    assert "ks_digit_ntt" in names, (what, sorted(set(names)))
    mac = "ks_local_mac" if n >= 4096 else "ks_mac"
    launches = sum(r[2] for r in prof if r[0].split(":")[0] == mac)
    assert launches > 0 and (not chunks or launches == chunks), f"{what}: {mac} launched {launches} times, want {chunks}"
    assert ("moddown_coeff" in names) == bfv and ("ks_moddown_ntt" in names) == (not bfv), (what, sorted(set(names)))


@pytest.mark.parametrize("g", [pytest.param(g, id=i) for g, i in zip(GROUPS, GROUP_IDS)])
def test_ks64_matrix(g):
    S = sb()
    n, mods, k = g.n, list(g.mods), len(g.mods)
    scheme = "BGV" if g.scheme.startswith("BGV") else g.scheme
    ntt = scheme != "BFV"
    assert all(q < 2 ** 57 for q in mods) == g.fast
    if not g.fast and scheme != "BFV":
        assert {q.bit_length() for q in mods} >= {60, 61}
    if g.scheme == "BGV-t-above":
        assert g.t > max(mods)
    elif g.t:
        assert g.t < min(mods)
    oc = O.Oracle(getattr(O, scheme), n, mods, g.t)
    rng = np.random.default_rng(GROUP_IDS.index(_group_id(g)))
    key = np.stack([np.stack([np.stack([rng.integers(0, q, n, dtype=np.uint64) for q in mods]) for _ in range(2)]) for _ in range(k - 1)])
    elt = galois_elt(g.galois, n)
    ops = (REL, MULREL, GAL, GAL_ADD, GAL_ADD_INPLACE)
    inputs = {}
    for L, op in itertools.product(g.levels, ops):
        pats = [PATTERNS[j % len(PATTERNS)] for j in range(BATCH)]
        if op == REL:
            args = (np.stack([draw(rng, mods, n, g.size, L, p, ntt) for p in pats]),)
        elif op == MULREL:
            args = tuple(np.stack([draw(rng, mods, n, 2, L, p, ntt) for p in pats]) for _ in range(2))
        else:
            args = (np.stack([draw(rng, mods, n, 2, L, p, ntt) for p in pats]), np.stack([draw(rng, mods, n, 2, L, "uniform", ntt) for _ in pats]))
        inputs[(L, op)] = args

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as pool:
        want = {(L, op, b): pool.submit(oracle_op, oc, op, elt, tuple(a[b] for a in args), L, key, mods)
                for (L, op), args in inputs.items() for b in range(BATCH)}
        ctx = S.Context(getattr(S, scheme), n, mods, g.t) if g.t else S.Context(S.CKKS, n, mods)
        rk = ctx.load_key(key)
        ctx.set_limit(ctx.LIMIT_KS_CHUNK, CHUNK)
        got = {}
        for mode in (KS_64, KS_AUTO):
            ctx.set_limit(ctx.LIMIT_KS_ALGORITHM, mode)
            for (L, op), args in inputs.items():
                what = f"{op} at L = {L}, key-switching mode {mode}"
                if op != REL or g.size == 3:
                    assert ctx.keyswitch_chunk(L, BATCH, fused=(op == MULREL)) == CHUNK
                ctx.profile(True)
                out = run_op(ctx, rk, op, elt, args, L, BATCH)
                prof = ctx.profile_read()
                ctx.profile(False)
                check_profile(prof, n, scheme == "BFV", 3 if (op != REL or g.size == 3) else 0, what)
                if mode == KS_64:
                    got[(L, op)] = out
                else:
                    assert_words(out, got[(L, op)], f"{what}: the automatic mode vs the forced 64-bit path")
        del rk
        ctx.close()
        for (L, op, b), fut in want.items():
            assert_words(got[(L, op)][b], fut.result(), f"{op} at L = {L}, member {b} ({PATTERNS[b % 3]}) vs the oracle")
    for L, op in inputs:
        galois = op.startswith("apply_galois")
        base = "add" if op.startswith(GAL_ADD) else "src"
        if op in (REL, GAL, GAL_ADD):  # multiply_relinearize and out = addend repeat a tuple of the same group
            COVERAGE.add((size_class(n), g.fast, row_class(scheme, mods, L, galois), "galois" if galois else "plain", g.scheme, base))
    DONE.add(_group_id(g))


def test_matrix_coverage():
    """the dispatch tuples the matrix reached are exactly the listed ones"""
    if DONE != set(GROUP_IDS):
        pytest.skip("asserted when every group of the matrix has run and passed")
    assert COVERAGE == expected_coverage(), (sorted(expected_coverage() - COVERAGE), sorted(COVERAGE - expected_coverage()))


# ------------------------------------------------------------------------------------------------------------------------------
# The digit-count bound.  Target rows (q_min - 1) delta_0 (in NTT form for CKKS, coefficient form for BFV) make every transformed
# digit the word q_min - 1 at every point; every key word of prime I is q_I - 1.  The digit sum at prime I is then the constant
# L (q_min - 1)(q_I - 1) at every point, past 2^128 from 65 digits of the largest 61-bit primes on.  The result is the mod-down of
# that constant added to the base rows (every word q - 1; apply_galois has no base in component 1): a closed form per (component,
# prime).  The oracle takes at most 64 primes, so it checks the closed form itself at L = 63, the deepest level it accepts, the
# same formula as deeper down.  The 60-bit level of 255 digits stays just below 2^128 (0.996); the FAST primes at L = 200 and 201
# (the guard-free transform outputs are reduced to below 4q from 201 digits on, sb_engine.cu) stay far below.
Bound = namedtuple("Bound", "scheme n bits L op")
ORACLE_MAX_PRIMES = 64
BOUNDS = [Bound("CKKS", 1024, 61, 63, REL), Bound("BFV", 1024, 61, 63, REL), Bound("CKKS", 4096, 61, 63, GAL),
          Bound("CKKS", 1024, 61, 64, REL), Bound("CKKS", 1024, 61, 65, REL), Bound("CKKS", 1024, 61, 255, REL),
          Bound("BFV", 1024, 61, 65, REL), Bound("BFV", 1024, 61, 255, REL),
          Bound("CKKS", 4096, 61, 64, REL), Bound("CKKS", 4096, 61, 65, REL), Bound("CKKS", 4096, 61, 66, REL),
          Bound("BFV", 4096, 61, 65, REL),
          Bound("CKKS", 1024, 61, 65, GAL), Bound("CKKS", 4096, 61, 65, GAL),
          Bound("CKKS", 1024, 60, 255, REL), Bound("BFV", 1024, 60, 255, REL),
          Bound("CKKS", 4096, 57, 200, REL), Bound("CKKS", 4096, 57, 201, REL)]


@pytest.mark.parametrize("case", BOUNDS, ids=[f"{b.scheme}-n{b.n}-q{b.bits}-L{b.L}-{b.op}" for b in BOUNDS])
def test_digit_sum_bound(case):
    S = sb()
    n, L = case.n, case.L
    k = L + 1
    mods = ntt_primes_below(case.bits, n, k)  # the largest primes = 1 mod 2n of that size; the special prime is the smallest
    ntt = case.scheme != "BFV"
    t = 65537 if case.scheme == "BFV" else 0
    qmin, qsp = min(mods), mods[-1]
    reach = max(L * (qmin - 1) * (q - 1) for q in mods)
    assert (reach >= 2 ** 128) == (case.bits == 61 and L > 64), reach / 2 ** 128
    if case.bits == 60:
        assert reach >= 0.99 * 2 ** 128
    ctx = S.Context(getattr(S, case.scheme), n, mods, t) if t else S.Context(S.CKKS, n, mods)
    key = np.ascontiguousarray(np.broadcast_to(np.array([q - 1 for q in mods], dtype=np.uint64)[None, None, :, None], (L, 2, k, n)))
    rk = ctx.load_key(key)
    size = 3 if case.op == REL else 2
    c = np.stack([np.full((L, n), 0, dtype=np.uint64) for _ in range(size)])
    for i in range(L):
        c[:-1, i] = mods[i] - 1
    c[-1] = const_target(mods, n, L, ntt)
    c = c[None]
    # closed form: digit sum L (q_min - 1)(q_I - 1) at every point of prime I, mod-down, plus the base word q - 1
    acc_sp = L * (qmin - 1) * (qsp - 1) % qsp
    want = np.empty((1, 2, L, n), dtype=np.uint64)
    for i in range(L):
        q = mods[i]
        r = mod_down(L * (qmin - 1) * (q - 1) % q, acc_sp, q, qsp)
        want[0, :, i, :] = (q - 1 + r) % q
        if not ntt:  # coefficient form: the sum sits at coefficient 0; elsewhere the base word is unchanged
            want[0, :, i, 1:] = q - 1
        if case.op == GAL:
            want[0, 1, i, :] = r
    aux = ctx.ksint_primes()
    auto_64 = not aux or L < 16 or L > (2 ** 64 - 1) // (max(aux) - 1) ** 2  # Context::ksint_on at the default switches
    for mode in (KS_64, KS_AUTO) if auto_64 else (KS_64,):
        ctx.set_limit(ctx.LIMIT_KS_ALGORITHM, mode)
        ctx.profile(True)
        got = ctx.relinearize(c, rk) if case.op == REL else ctx.apply_galois(c, O.galois_elt_from_step(n, 1), rk)
        names = {r[0].split(":")[0] for r in ctx.profile_read()}
        ctx.profile(False)
        assert ("ks_local_mac" if n >= 4096 else "ks_mac") in names and not any(x.startswith("ks32") for x in names), sorted(names)
        assert_words(got, want, f"{case}: key-switching mode {mode} vs the closed form")
    del rk
    ctx.close()
    if k <= ORACLE_MAX_PRIMES:
        oc = O.Oracle(getattr(O, case.scheme), n, mods, t)
        w = oc.relinearize(L, c[0], key) if case.op == REL else oc.apply_galois(L, c[0], O.galois_elt_from_step(n, 1), key)
        assert_words(want[0], w, f"{case}: the closed form vs the oracle")
