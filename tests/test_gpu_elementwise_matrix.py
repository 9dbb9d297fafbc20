"""Parity matrix of the element-wise operations (-m gpu; seal_b200/csrc/sb_engine.cu): add / sub / negate (linear_kernel), add_many
(fold_kernel), multiply 2 x 2 (ckks_tensor_kernel), square (ckks_square_kernel), general sizes (tensor_general_kernel),
multiply_plain (plain_mul_kernel, shared_plain_kernel mode 0), CKKS add_plain / sub_plain (add_c0_kernel, shared_plain_kernel
modes 1 and 2), BFV / BGV add_plain / sub_plain with coefficient-form plaintexts (bfv_add_plain_kernel, add_c0_kernel) and
transform_to_ntt / transform_from_ntt of ciphertexts (op_ntt).  Every output word is checked against the statement of the
reference's release-build word semantics (tests/elementwise_ref.py; the transforms against the oracle's); the first and last
ciphertext of every case also against the reference where its SEALContext takes the parameters and level, else the oracle.
The axes crossed on purpose:

- ring size n = 2, 4, ..., 131072 (logn = 1 is where plain_mul_kernel's in-row mask is 0; the transforms change shape at 4096);
- prime class: the smallest NTT-friendly primes for the ring, primes just below and just above 2^57 (the guard-free and the
  guarded butterflies), 60-bit primes, and primes just below 2^61, where ckks_tensor_kernel's middle term 2 (q - 1)^2 meets
  barrett_wide's bound 2^(b + 62): in every class a batch whose every word is q - 1 goes through multiply, square, general
  sizes and multiply_plain (per ciphertext and shared);
- level: L = 1, a middle level and the key level (the reference keeps no ciphertexts there: oracle only), a 64-prime level (the
  oracle's and the reference's limit, so a key level too) in groups of its own, and for the shared-plaintext kernels the deepest
  level the context accepts (256 primes);
- words: member j of a batch draws its word class j mod P (test_elementwise_words.KINDS: canonical, 0 / 1 / q - 1, unreduced up to
  2^64 - 1, x + y >= 2^64, x - y > 2^64 - q, y - x > q, unreduced against canonical and the reverse); the transforms take
  canonical words and 0 / 1 / q - 1 only, as their lazy butterflies presume in the reference too;
- entry points: the stream entry points on a non-default torch stream, in place where the layout allows it; the host entry
  points with LIMIT_HOST_STAGE_BYTES cut for three or more staging chunks with a ragged tail (test_host_staging); 19 ciphertexts
  against one plaintext, so that shared_plain_kernel's groups of 8 end ragged; op_ntt's row seam (2^20 - 2^20 mod L rows per
  launch: inside a ciphertext with L = 3, between two ciphertexts with L = 7 and 3 polynomials); shared_plain_kernel at 256 primes and n = 131072, where L n / 512 exceeds the 65535
  blocks grid.y takes.

Each case checks the profile for the kernels that ran.  The last test asserts that the module reached exactly the (operation, prime
class, level kind) tuples of expected_coverage() and the ring sizes of every operation."""
from collections import namedtuple

import numpy as np
import pytest

import elementwise_ref as E
import oracle as O
import refseal as R
from common import assert_words, is_prime
from test_elementwise_words import KINDS, pair_words

pytestmark = pytest.mark.gpu

SIZES = tuple(2 ** k for k in range(1, 18))
CLASSES = ("smallest", "below-2^57", "above-2^57", "60-bit", "below-2^61")
K = 5  # primes of a group: levels 1, 3 (middle) and 5 (key level)
LEVELS = ((1, "L1"), (3, "mid"), (5, "key"))
GENERAL = ((2, 3), (3, 2), (3, 3), (2, 15), (15, 2), (8, 8))
OPS = ("add", "sub", "negate", "add_many", "multiply", "square", "multiply_sized", "multiply_plain", "multiply_plain_shared",
       "add_plain_ntt", "sub_plain_ntt", "add_plain_ntt_shared", "sub_plain_ntt_shared", "ntt")
# the products on a batch whose every word is q - 1
QOPS = ("multiply@q-1", "square@q-1", "multiply_sized@q-1", "multiply_plain@q-1", "multiply_plain_shared@q-1")
COEFF_OPS = ("bfv_add_plain", "bfv_sub_plain", "bgv_add_plain", "bgv_sub_plain")
STAGE_MIN = 1 << 16

COVERAGE, SIZES_SEEN, DONE, COMPARED = set(), {}, set(), {}


def sb():
    import seal_b200

    return seal_b200


def primes_for(n, cls, k):
    m = 2 * n
    if cls == "smallest":
        out, p = [], m + 1
        while len(out) < k:
            if is_prime(p):
                out.append(p)
            p += m
        return out
    if cls == "above-2^57":
        out, p = [], (2 ** 57 // m + 1) * m + 1
        while len(out) < k:
            if is_prime(p):
                out.append(p)
            p += m
        return out
    return O.get_primes(m, {"below-2^57": 57, "60-bit": 60, "below-2^61": 61}[cls], k)


Group = namedtuple("Group", "n cls")
GROUPS = [Group(n, c) for n in SIZES for c in CLASSES]
GROUP_IDS = [f"n{g.n}-{g.cls}" for g in GROUPS]


def expected_coverage():
    out = {(op, cls, lk) for op in OPS + QOPS for cls in CLASSES for _, lk in LEVELS}
    out |= {(op, cls, "64") for op in OPS + QOPS for cls in ("60-bit", "below-2^61")}
    out |= {(op, cls, lk) for op in COEFF_OPS for cls in ("below-2^57", "60-bit") for _, lk in LEVELS}
    out |= {(op, "60-bit", "256") for op in ("multiply_plain_shared", "add_plain_ntt_shared", "sub_plain_ntt_shared")}
    return out


def to_dev(a):
    import torch

    return torch.from_numpy(np.array(a, dtype=np.uint64, order="C").view(np.int64)).cuda()  # a writable copy (broadcasts are not)


def to_np(t):
    return t.cpu().numpy().view(np.uint64)


def draw_pair(rng, mods, B, size, L, n, kinds, offset=0):
    """[B][size][L][n] words x, y; member j by kinds[(j + offset) % len(kinds)]; member B - 1 of a canonical draw is all q - 1"""
    x = np.empty((B, size, L, n), dtype=np.uint64)
    y = np.empty_like(x)
    for j in range(B):
        kind = kinds[(j + offset) % len(kinds)]
        for i in range(L):
            x[j, :, i], y[j, :, i] = pair_words(kind, rng, mods[i], (size, n))
    if B > 1 and kinds == ("canonical",):
        for i in range(L):
            x[B - 1, :, i] = y[B - 1, :, i] = mods[i] - 1
    return x, y


class Runner:
    """runs one device entry point on a non-default stream with the profile on; returns the profile's kernel names"""

    def __init__(self, ctx):
        self.ctx = ctx

    def __call__(self, fn):
        import torch

        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        self.ctx.profile(True)
        with torch.cuda.stream(s):
            fn()
        s.synchronize()
        names = {r[0] for r in self.ctx.profile_read()}
        self.ctx.profile(False)
        return names


def lin(S, ctx, name, L, size, B, a, b, out):
    fn = getattr(S.lib(), f"sb200_{name}")
    if name == "negate":
        S._check(fn(ctx.h, L, size, B, S._dp(a), S._dp(out), ctx._stream()))
    else:
        S._check(fn(ctx.h, L, size, B, S._dp(a), S._dp(b), S._dp(out), ctx._stream()))


def record(gid, op, cls, lk, n, how):
    COVERAGE.add((op, cls, lk))
    SIZES_SEEN.setdefault(op, set()).add(n)
    COMPARED.setdefault((gid, op, lk), set()).update(how)


def ref_context(scheme, n, mods, t=0):
    """the reference's context when it takes the parameters (primes of at most 60 bits, at most 64 of them), else None"""
    if not R.available() or max(mods) >= 2 ** 60 or len(mods) > 64:
        return None
    try:
        return R.RefContext(scheme, n, mods, t)
    except RuntimeError:
        return None


def check_members(rc, oc, L, k, got, members, fn_ref, fn_oracle, what):
    """the first and last members against the reference (below the key level) or the oracle; returns the comparisons made"""
    how = {"statement"}
    for j in members:
        if rc is not None and L < k:
            try:
                assert_words(got[j], fn_ref(rc, j), f"{what}, ciphertext {j}: vs the reference")
                how.add("reference")
                continue
            except RuntimeError as e:  # the reference throws on a result whose c_1 is zero, as edge words give at small n
                if "transparent" not in str(e):
                    raise
        assert_words(got[j], fn_oracle(oc, j), f"{what}, ciphertext {j}: vs the oracle")
        how.add("oracle")
    return how


def run_level(S, g, gid, ctx, oc, rc, mods, L, lk, rng, big):
    import torch

    n, k = g.n, len(mods)
    B = 1 if big else 3
    run = Runner(ctx)
    # one ciphertext per case at n >= 32768: its word class turns with the level and the group, so that every class is met there
    offset = (GROUPS.index(g) if g in GROUPS else 0) * 3 + L
    kinds = KINDS[offset % len(KINDS):] + KINDS[:offset % len(KINDS)]
    ends = sorted({0, B - 1})

    # ---- add / sub / negate, sizes 2, 3 and 16 (16 only at small n) ----
    for size in ((2, 3, 16) if n <= 1024 else (2, 3)):
        x, y = draw_pair(rng, mods, B, size, L, n, kinds)
        dx, dy = to_dev(x), to_dev(y)
        for mode, name in enumerate(("add", "sub", "negate")):
            out = torch.empty_like(dx)
            ran = run(lambda: lin(S, ctx, name, L, size, B, dx, dy, out))
            assert ran == {name}, (name, ran)
            want = E.linear(mode, x, y, mods)
            got = to_np(out)
            assert_words(got, want, f"{gid} {name} L={L} size={size}: vs the statement")
            how = check_members(rc, oc, L, k, got, ends, lambda r, j: r.linear(mode, L, x[j], y[j]),
                                lambda o, j: o.linear(mode, L, x[j], y[j]), f"{gid} {name} L={L} size={size}")
            record(gid, name, g.cls, lk, n, how)
        # in place: out = a
        da = dx.clone()
        run(lambda: lin(S, ctx, "sub", L, size, B, da, dy, da))
        assert_words(to_np(da), E.linear(1, x, y, mods), f"{gid} sub in place L={L} size={size}")

    # ---- add_many: sub steps, mixed sizes, a longer subtrahend's negated tail, more than 16 operands at small n ----
    count = 17 if n <= 1024 else 4
    sizes = [2 if j % 3 else 3 for j in range(count)]
    sizes[-1] = 4 if n <= 1024 else 3
    modes = [int(j % 2 == 0) for j in range(count - 1)]
    ops = [draw_pair(rng, mods, B, s, L, n, kinds)[0] for s in sizes]
    acc = [ops[0][:, p] for p in range(sizes[0])]
    for j in range(1, count):
        for p in range(sizes[j]):
            v = ops[j][:, p]
            if p < len(acc):
                acc[p] = E.linear(modes[j - 1], acc[p], v, mods)
            else:
                acc.append(E.negate(v, E.qcol(mods, L)) if modes[j - 1] else v)
    want = np.stack(acc, axis=1)
    out = torch.empty((B, max(sizes), L, n), dtype=torch.int64, device="cuda")
    dops = [to_dev(o) for o in ops]
    ran = run(lambda: ctx.d_add_many(dops, out, L, B, sizes, modes))
    assert ran == {"add_many"}, ran
    got = to_np(out)
    assert_words(got, want, f"{gid} add_many L={L} count={count}: vs the statement")

    def fold_oracle(o, j):
        r = ops[0][j]
        for jj in range(1, count):
            y = ops[jj][j]
            if y.shape[0] > r.shape[0]:
                pad = np.zeros((y.shape[0] - r.shape[0], L, n), dtype=np.uint64)
                r = np.concatenate([r, pad])
            if y.shape[0] < r.shape[0]:
                y = np.concatenate([y, np.zeros((r.shape[0] - y.shape[0], L, n), dtype=np.uint64)])
            r = o.linear(modes[jj - 1], L, r, y)
        return r

    # the oracle and the reference take equal sizes only: the padded chain is the fold's words wherever no tail is involved, so the
    # members are compared on the polynomials every operand has (the statement covers the tails)
    how = {"statement"}
    for j in ends:
        r = fold_oracle(oc, j)
        assert_words(got[j, :min(sizes)], r[:min(sizes)], f"{gid} add_many L={L}, ciphertext {j}: vs the oracle")
        how.add("oracle")
    record(gid, "add_many", g.cls, lk, n, how)

    # ---- multiply 2 x 2, square, general sizes ----
    x, y = draw_pair(rng, mods, B, 2, L, n, kinds)
    dx, dy = to_dev(x), to_dev(y)
    out = torch.empty((B, 3, L, n), dtype=torch.int64, device="cuda")
    ran = run(lambda: ctx.d_multiply(dx, dy, out, L, B))
    assert ran == {"ckks_tensor"}, ran
    got = to_np(out)
    assert_words(got, E.tensor(x, y, mods), f"{gid} multiply L={L}: vs the statement")
    how = check_members(rc, oc, L, k, got, ends, lambda r, j: r.multiply(L, x[j], y[j]), lambda o, j: o.multiply(L, x[j], y[j]),
                        f"{gid} multiply L={L}")
    record(gid, "multiply", g.cls, lk, n, how)
    ran = run(lambda: S._check(S.lib().sb200_square(ctx.h, L, B, S._dp(dx), S._dp(out), ctx._stream())))
    assert ran == {"ckks_square"}, ran
    got = to_np(out)
    assert_words(got, E.tensor(x, x, mods), f"{gid} square L={L}: vs the statement")
    how = check_members(rc, oc, L, k, got, ends, lambda r, j: r.square(L, x[j]), lambda o, j: o.multiply(L, x[j], x[j]),
                        f"{gid} square L={L}")
    record(gid, "square", g.cls, lk, n, how)
    # every general size at n <= 256; three of them below 32768; one at L = 1 above (the statement's exact products cost the time)
    for sa, sb_ in (GENERAL if n <= 256 else GENERAL[:3] if n < 32768 else GENERAL[:1] if L == 1 else ()):
        xa = draw_pair(rng, mods, B, sa, L, n, kinds)[0]
        xb = draw_pair(rng, mods, B, sb_, L, n, kinds)[1]
        out = torch.empty((B, sa + sb_ - 1, L, n), dtype=torch.int64, device="cuda")
        da, db = to_dev(xa), to_dev(xb)
        ran = run(lambda: ctx.d_multiply_sized(da, db, out, L, sa, sb_, B))
        assert ran == {"tensor_general"}, ran
        got = to_np(out)
        assert_words(got, E.tensor(xa, xb, mods), f"{gid} multiply {sa}x{sb_} L={L}: vs the statement")
        how = check_members(rc, oc, L, k, got, ends, lambda r, j: r.multiply(L, xa[j], xb[j]), lambda o, j: o.multiply(L, xa[j], xb[j]),
                            f"{gid} multiply {sa}x{sb_} L={L}")
        record(gid, "multiply_sized", g.cls, lk, n, how)

    # ---- multiply_plain and CKKS add_plain / sub_plain, per ciphertext and shared ----
    size = 3 if n <= 1024 else 2
    x, p = draw_pair(rng, mods, B, size, L, n, kinds)
    plains = np.ascontiguousarray(p[:, 0])
    dx, dp = to_dev(x), to_dev(plains)
    for shared in (False, True):
        pw = plains[:1] if shared else plains
        dpw = to_dev(pw[0]) if shared else dp
        cnt = 1 if shared else B
        out = torch.empty_like(dx)
        ran = run(lambda: ctx.d_multiply_plain_n(dx, dpw, out, L, size, B, cnt))
        assert ran == {"multiply_plain"}, ran
        got = to_np(out)
        want = E.multiply_plain(x, pw if not shared else pw[0], mods)
        op = "multiply_plain_shared" if shared else "multiply_plain"
        assert_words(got, want, f"{gid} {op} L={L}: vs the statement")
        pj = (lambda j: pw[0]) if shared else (lambda j: pw[j])
        how = check_members(rc, oc, L, k, got, ends, lambda r, j: r.multiply_plain(L, x[j], pj(j)),
                            lambda o, j: o.multiply_plain(L, x[j], pj(j)), f"{gid} {op} L={L}")
        record(gid, op, g.cls, lk, n, how)
        for sub in (False, True):
            op = f"{'sub' if sub else 'add'}_plain_ntt{'_shared' if shared else ''}"
            da = dx.clone()
            ran = run(lambda: ctx.d_add_plain_ntt(da, dpw, da, L, size, B, cnt, sub))  # in place
            assert ran == {"ckks_sub_plain" if sub else "ckks_add_plain"}, ran
            got = to_np(da)
            want = E.add_plain_c0(x, pw if not shared else pw[0], mods, sub)
            assert_words(got, want, f"{gid} {op} L={L}: vs the statement")
            # the reference's add_plain on c_0 is add_poly_coeffmod / sub_poly_coeffmod: the same words as add / sub of c_0
            mode = 1 if sub else 0
            c0_plain = lambda j: np.stack([pj(j), np.zeros_like(pj(j))])  # the plaintext as a size-2 operand; c_0 compared only
            how = check_members(rc, oc, L, k, got[:, :1], ends, lambda r, j: r.linear(mode, L, x[j, :2], c0_plain(j))[:1],
                                lambda o, j: o.linear(mode, L, x[j, :2], c0_plain(j))[:1], f"{gid} {op} L={L}")
            assert_words(got[:, 1:], x[:, 1:], f"{gid} {op} L={L}: c_1 untouched")
            record(gid, op, g.cls, lk, n, how)

    # ---- every word at q - 1: the products at their largest canonical operands.  Below 2^61 the 2 x 2 tensor's middle term
    # 2 (q - 1)^2 lies in [2^(b + 61), 2^(b + 62)), the top half of the range barrett_wide takes (b = bit length of q) ----
    if g.cls == "below-2^61":
        assert all(2 ** (q.bit_length() + 61) <= 2 * (q - 1) ** 2 < 2 ** (q.bit_length() + 62) for q in mods[:L]), mods[:L]
    Bq = 1 if big else 2
    top = np.stack([np.full(n, mods[i] - 1, dtype=np.uint64) for i in range(L)])  # [L][n]
    xq = np.ascontiguousarray(np.broadcast_to(top, (Bq, 2, L, n)))
    dq = to_dev(xq)
    out = torch.empty((Bq, 3, L, n), dtype=torch.int64, device="cuda")
    dq2 = dq.clone()  # a second slab of the same words: multiply, not square
    ran = run(lambda: ctx.d_multiply(dq, dq2, out, L, Bq))
    assert ran == {"ckks_tensor"}, ran
    got = to_np(out)
    assert_words(got, E.tensor(xq, xq, mods), f"{gid} multiply, every word q - 1, L={L}: vs the statement")
    how = check_members(rc, oc, L, k, got, [0], lambda r, j: r.multiply(L, xq[j], xq[j]), lambda o, j: o.multiply(L, xq[j], xq[j]),
                        f"{gid} multiply, every word q - 1, L={L}")
    record(gid, "multiply@q-1", g.cls, lk, n, how)
    ran = run(lambda: S._check(S.lib().sb200_square(ctx.h, L, Bq, S._dp(dq), S._dp(out), ctx._stream())))
    assert ran == {"ckks_square"}, ran
    got = to_np(out)
    assert_words(got, E.tensor(xq, xq, mods), f"{gid} square, every word q - 1, L={L}: vs the statement")
    how = check_members(rc, oc, L, k, got, [0], lambda r, j: r.square(L, xq[j]), lambda o, j: o.multiply(L, xq[j], xq[j]),
                        f"{gid} square, every word q - 1, L={L}")
    record(gid, "square@q-1", g.cls, lk, n, how)
    for sa, sb_ in (GENERAL if n <= 256 else ((3, 3),) if n < 32768 or L == 1 else ()):
        xa = np.ascontiguousarray(np.broadcast_to(top, (Bq, sa, L, n)))
        xb = np.ascontiguousarray(np.broadcast_to(top, (Bq, sb_, L, n)))
        out = torch.empty((Bq, sa + sb_ - 1, L, n), dtype=torch.int64, device="cuda")
        da, db = to_dev(xa), to_dev(xb)
        ran = run(lambda: ctx.d_multiply_sized(da, db, out, L, sa, sb_, Bq))
        assert ran == {"tensor_general"}, ran
        got = to_np(out)
        assert_words(got, E.tensor(xa, xb, mods), f"{gid} multiply {sa}x{sb_}, every word q - 1, L={L}: vs the statement")
        how = check_members(rc, oc, L, k, got, [0], lambda r, j: r.multiply(L, xa[j], xb[j]), lambda o, j: o.multiply(L, xa[j], xb[j]),
                            f"{gid} multiply {sa}x{sb_}, every word q - 1, L={L}")
        record(gid, "multiply_sized@q-1", g.cls, lk, n, how)
    dtop = to_dev(top)
    for shared in (False, True):
        op = "multiply_plain_shared@q-1" if shared else "multiply_plain@q-1"
        out = torch.empty_like(dq)
        dpl = dtop if shared else to_dev(np.ascontiguousarray(np.broadcast_to(top, (Bq, L, n))))
        ran = run(lambda: ctx.d_multiply_plain_n(dq, dpl, out, L, 2, Bq, 1 if shared else Bq))
        assert ran == {"multiply_plain"}, ran
        got = to_np(out)
        assert_words(got, E.multiply_plain(xq, top, mods), f"{gid} {op}, L={L}: vs the statement")
        how = check_members(rc, oc, L, k, got, [0], lambda r, j: r.multiply_plain(L, xq[j], top),
                            lambda o, j: o.multiply_plain(L, xq[j], top), f"{gid} {op}, L={L}")
        record(gid, op, g.cls, lk, n, how)

    # ---- transform_to_ntt / transform_from_ntt of ciphertexts of sizes 2, 3 and 16 (canonical words, 0 / 1 / q - 1) ----
    for size in ((2, 3, 16) if n <= 1024 else (2,)):
        x = draw_pair(rng, mods, B, size, L, n, ("canonical", "edges"))[0]
        d = to_dev(x)
        ran = run(lambda: ctx.d_ntt_forward(d, L, size, B))
        assert ran and all(r.startswith("ntt_fwd") for r in ran), ran
        fwd = to_np(d)
        ran = run(lambda: ctx.d_ntt_inverse(d, L, size, B))
        assert ran and all(r.startswith("ntt_inv") for r in ran), ran
        back = to_np(d)
        for j in range(B):
            assert_words(fwd[j], oc.ntt_forward(L, x[j]), f"{gid} transform_to_ntt L={L} size={size}, ciphertext {j}: vs the oracle")
            assert_words(back[j], oc.ntt_inverse(L, fwd[j]), f"{gid} transform_from_ntt L={L} size={size}, ciphertext {j}")
        assert_words(back, x, f"{gid} transforms L={L} size={size}: round trip")
        how = {"oracle"}
        if rc is not None and L < k:
            for j in ends:
                assert_words(fwd[j], rc.ntt_forward(L, x[j]), f"{gid} transform_to_ntt L={L}, ciphertext {j}: vs the reference")
            how.add("reference")
        record(gid, "ntt", g.cls, lk, n, how)


def run_coeff_plain(S, g, gid, mods, L, lk, rng, big):
    """BFV and BGV add_plain / sub_plain with coefficient-form plaintexts (words below t) on c_0 words of every class"""
    import torch

    n, k = g.n, len(mods)
    t = 65537 if 65537 not in mods else 114689
    B = 1 if big else 3
    for scheme in ("bfv", "bgv"):
        ctx = S.Context(S.BFV if scheme == "bfv" else S.BGV, n, mods, t)
        oc = O.Oracle(O.BFV if scheme == "bfv" else O.BGV, n, mods, t)
        run = Runner(ctx)
        x = draw_pair(rng, mods, B, 2, L, n, KINDS)[0]
        plain = rng.integers(0, t, (B, n), dtype=np.uint64)
        plain[:, 0], plain[:, -1] = t - 1, (t + 1) // 2
        cf = [1] * B if scheme == "bfv" else [int(v) for v in rng.integers(1, t, B)]
        dx, dplain = to_dev(x), to_dev(plain)
        for sub in (False, True):
            op = f"{scheme}_{'sub' if sub else 'add'}_plain"
            out = torch.empty_like(dx)
            ran = run(lambda: ctx.d_add_plain_coeff_n(dx, dplain, out, L, 2, B, B, sub, None if scheme == "bfv" else cf))
            assert ran >= {"bfv_add_plain" if scheme == "bfv" else "bgv_add_plain"}, ran
            got = to_np(out)
            for j in range(B):
                if scheme == "bfv":
                    T = E.bfv_scaled_plain(plain[j], mods, L, t)
                else:
                    T = oc.plain_to_ntt(L, (plain[j].astype(object) * cf[j] % t).astype(np.uint64))
                assert_words(got[j], E.add_plain_c0(x[j], T, mods, sub), f"{gid} {op} L={L}, ciphertext {j}: vs the statement")
                assert_words(got[j], oc.add_plain_coeff(L, x[j], plain[j], sub, cf[j]), f"{gid} {op} L={L}, ciphertext {j}: vs the oracle")
            record(gid, op, g.cls, lk, n, {"statement", "oracle"})
        ctx.close()


@pytest.mark.parametrize("g", [pytest.param(g, id=i) for g, i in zip(GROUPS, GROUP_IDS)])
def test_elementwise_matrix(g):
    S = sb()
    gid = GROUP_IDS[GROUPS.index(g)]
    mods = primes_for(g.n, g.cls, K)
    ctx = S.Context(S.CKKS, g.n, mods)
    oc = O.Oracle(O.CKKS, g.n, mods)
    rc = ref_context(R.BGV, g.n, mods, 65537 if 65537 not in mods else 114689) if g.cls != "smallest" else None
    rng = np.random.default_rng(GROUPS.index(g))
    big = g.n >= 32768
    for L, lk in LEVELS:
        run_level(S, g, gid, ctx, oc, rc, mods, L, lk, rng, big)
        if g.cls in ("below-2^57", "60-bit"):
            run_coeff_plain(S, g, gid, mods, L, lk, rng, big)
    ctx.close()
    if rc is not None:
        rc.close()
    DONE.add(gid)


@pytest.mark.parametrize("cls", ["60-bit", "below-2^61"])
@pytest.mark.parametrize("n", [2, 4096])
def test_64_primes(cls, n):
    """a level of 64 primes (the reference's and the oracle's limit, so the key level here: samples against the oracle), every
    operation"""
    S = sb()
    mods = primes_for(n, cls, 64)
    ctx = S.Context(S.CKKS, n, mods)
    oc = O.Oracle(O.CKKS, n, mods)
    rc = ref_context(R.BGV, n, mods, 65537)
    g = Group(n, cls)
    gid = f"n{n}-{cls}-k64"
    run_level(S, g, gid, ctx, oc, rc, mods, 64, "64", np.random.default_rng(64 + n), False)
    ctx.close()
    DONE.add(gid)


def test_shared_plain_19_ciphertexts():
    """19 ciphertexts against one plaintext: shared_plain_kernel's groups of 8 end with 3"""
    import torch

    S = sb()
    n, L, B, size = 1024, 3, 19, 2
    mods = primes_for(n, "60-bit", 4)
    ctx = S.Context(S.CKKS, n, mods)
    rng = np.random.default_rng(19)
    x, p = draw_pair(rng, mods, B, size, L, n, KINDS)
    plain = np.ascontiguousarray(p[0, 0])
    dx, dp = to_dev(x), to_dev(plain)
    out = torch.empty_like(dx)
    ctx.d_multiply_plain_n(dx, dp, out, L, size, B, 1)
    assert_words(to_np(out), E.multiply_plain(x, plain, mods), "multiply_plain, 19 ciphertexts, one plaintext")
    for sub in (False, True):
        out = torch.empty_like(dx)
        ctx.d_add_plain_ntt(dx, dp, out, L, size, B, 1, sub)
        assert_words(to_np(out), E.add_plain_c0(x, plain, mods, sub), f"{'sub' if sub else 'add'}_plain, 19 ciphertexts, one plaintext")


def test_host_staging():
    """the host entry points with LIMIT_HOST_STAGE_BYTES cut for three or more staging chunks and a ragged tail"""
    S = sb()
    n, L = 4096, 3
    mods = primes_for(n, "below-2^57", 4)
    ctx = S.Context(S.CKKS, n, mods)
    rng = np.random.default_rng(4096)
    size, B = 2, 7
    per_ct = 3 * size * L * n * 8
    ctx.set_limit(ctx.LIMIT_HOST_STAGE_BYTES, max(2 * per_ct, STAGE_MIN))  # 2 ciphertexts per chunk: 2, 2, 2, 1
    x, y = draw_pair(rng, mods, B, size, L, n, KINDS)

    def launches(fn, name):
        """fn's result and the launches of kernel `name` it made: one per staging chunk"""
        ctx.profile(True)
        r = fn()
        prof = {p[0]: p[2] for p in ctx.profile_read()}
        ctx.profile(False)
        return r, prof.get(name, 0)

    got, cnt = launches(lambda: ctx.add(x, y), "add")
    assert cnt == 4, cnt  # chunks of 2, 2, 2 and 1 ciphertexts
    assert_words(got, E.linear(0, x, y, mods), "host add")
    got, cnt = launches(lambda: ctx.sub(x, y), "sub")
    assert cnt == 4, cnt
    assert_words(got, E.linear(1, x, y, mods), "host sub")
    assert_words(ctx.negate(x), E.linear(2, x, y, mods), "host negate")
    got, cnt = launches(lambda: ctx.multiply(x, y), "ckks_tensor")
    assert cnt == B, cnt  # 7 words per coefficient of a ciphertext where add moves 6: one ciphertext per chunk
    assert_words(got, E.tensor(x, y, mods), "host multiply")
    assert_words(ctx.square(x), E.tensor(x, x, mods), "host square")
    assert_words(ctx.multiply(x, np.concatenate([y, x[:, :1]], axis=1)), E.tensor(x, np.concatenate([y, x[:, :1]], axis=1), mods),
                 "host multiply 2x3")
    plains = np.ascontiguousarray(y[:, 0])
    assert_words(ctx.multiply_plain_n(x, plains), E.multiply_plain(x, plains, mods), "host multiply_plain")
    assert_words(ctx.multiply_plain_n(x, plains[0]), E.multiply_plain(x, plains[0], mods), "host multiply_plain, shared")
    for sub in (False, True):
        assert_words(ctx.add_plain_ntt(x, plains, sub), E.add_plain_c0(x, plains, mods, sub), f"host add_plain sub={sub}")
        assert_words(ctx.add_plain_ntt(x, plains[0], sub), E.add_plain_c0(x, plains[0], mods, sub), f"host add_plain shared sub={sub}")
    ops = [x, y, x]
    got, cnt = launches(lambda: ctx.add_many(ops, [1, 0]), "add_many")
    assert cnt >= 3, cnt
    assert_words(got, E.linear(0, E.linear(1, x, y, mods), x, mods), "host add_many")
    c = draw_pair(rng, mods, B, size, L, n, ("canonical",))[0]
    oc = O.Oracle(O.CKKS, n, mods)
    f = ctx.transform_to_ntt(c)
    for j in range(B):
        assert_words(f[j], oc.ntt_forward(L, c[j]), f"host transform_to_ntt, ciphertext {j}")
    assert_words(ctx.transform_from_ntt(f), c, "host transform round trip")


@pytest.mark.parametrize("L,size,inside", [(3, 2, True), (3, 3, True), (7, 3, False)])
def test_ntt_row_seam(L, size, inside):
    """op_ntt launches 2^20 - (2^20 mod L) rows at a time, so a launch never splits the L rows of one polynomial.  With L = 3 that
    is 2^20 - 1 rows, which splits a ciphertext of 2 or 3 polynomials (6 and 9 do not divide it); with L = 7 it is 2^20 - 4 =
    21 * 49932 rows, so the seam falls between two ciphertexts of 3 polynomials"""
    import torch

    S = sb()
    n = 4
    mods = primes_for(n, "60-bit", L)
    ctx = S.Context(S.CKKS, n, mods)
    oc = O.Oracle(O.CKKS, n, mods)
    per_launch = 2 ** 20 - 2 ** 20 % L
    assert (per_launch % (size * L) != 0) == inside, (per_launch, size, L)
    B = per_launch // (size * L) + 2
    rng = np.random.default_rng(L)
    x = np.stack([rng.integers(0, q, (B, size, n), dtype=np.uint64) for q in mods], axis=2)
    d = to_dev(x)
    ctx.profile(True)
    ctx.d_ntt_forward(d, L, size, B)
    import torch as _t

    _t.cuda.synchronize()
    prof = {r[0]: r[2] for r in ctx.profile_read()}
    ctx.profile(False)
    assert sum(prof.values()) == 2, prof  # two launches: the seam is crossed
    got = to_np(d)
    seam = per_launch // (size * L)  # the ciphertext holding row per_launch
    for j in sorted({0, seam - 1, seam, seam + 1, B - 1}):
        assert_words(got[j], oc.ntt_forward(L, x[j]), f"L={L} size={size}: ciphertext {j} around the row seam (row {per_launch})")
    ctx.d_ntt_inverse(d, L, size, B)
    assert_words(to_np(d), x, "round trip across the seam")


def test_shared_plain_256_primes():
    """n = 131072 with 256 primes: L n / 512 = 65536 exceeds the 65535 blocks of grid.y; shared_plain_kernel strides over y, so
    the last prime's pairs are reached on the second pass of the stride loop.  One ciphertext of 0.5 GiB on the device; every
    word of the first and last primes' rows checked against the statement"""
    import torch

    S = sb()
    n, L = 131072, 256
    free, _ = torch.cuda.mem_get_info()
    if free < (6 << 30):
        pytest.skip(f"needs 6 GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
    mods = primes_for(n, "60-bit", L)
    ctx = S.Context(S.CKKS, n, mods)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(256)
    a = torch.empty((1, 2, L, n), dtype=torch.int64, device="cuda")
    p = torch.empty((L, n), dtype=torch.int64, device="cuda")
    a.random_(generator=gen)  # unreduced words
    for i in range(L):
        p[i].random_(0, mods[i], generator=gen)
    rows = [0, L - 1]
    ai = np.stack([to_np(a[0, :, i]) for i in rows], axis=1)  # [2][2 rows][n]
    pi = np.stack([to_np(p[i]) for i in rows])
    sub_mods = [mods[i] for i in rows]
    for op in ("multiply_plain_shared", "add_plain_ntt_shared", "sub_plain_ntt_shared"):
        out = torch.empty_like(a)
        ctx.profile(True)
        if op == "multiply_plain_shared":
            ctx.d_multiply_plain_n(a, p, out, L, 2, 1, 1)
            want = E.multiply_plain(ai, pi, sub_mods)
        else:
            sub = op.startswith("sub")
            ctx.d_add_plain_ntt(a, p, out, L, 2, 1, 1, sub)
            want = E.add_plain_c0(ai, pi, sub_mods, sub)
        torch.cuda.synchronize()
        names = {r[0] for r in ctx.profile_read()}
        ctx.profile(False)
        assert names, op
        got = np.stack([to_np(out[0, :, i]) for i in rows], axis=1)
        assert_words(got, want, f"{op}, n = {n}, {L} primes: rows {rows}")
        record(f"n{n}-60-bit-k256", op, "60-bit", "256", n, {"statement"})
        del out
    del a, p
    ctx.close()
    torch.cuda.empty_cache()
    DONE.add(f"n{n}-60-bit-k256")


@pytest.mark.parametrize("op", ["add", "multiply", "rescale_to_next", "apply_galois", "add_many"])
def test_overlapping_slabs_refused(op):
    """a stream entry point refuses an output slab that overlaps an input slab other than exactly in place
    (SB200_E_INVALID_ARG), before any launch: the output words stay as they were.  Every slab lies inside one allocation large
    enough for every range, so that no access could leave it"""
    import torch

    S = sb()
    n, B = 1024, 3
    mods = primes_for(n, "60-bit", 4)
    L, k = 3, 4
    ctx = S.Context(S.CKKS, n, mods)
    rng = np.random.default_rng(7)
    poly = L * n
    base = torch.from_numpy(rng.integers(0, mods[0], 16 * B * poly, dtype=np.uint64).view(np.int64)).cuda()
    ptr = base.data_ptr()
    at = lambda words: ptr + 8 * words  # a device pointer `words` words into the allocation
    if op == "add":  # out starts one polynomial into a: ciphertext 0's output is ciphertext 0's second input polynomial
        call = lambda: S._check(S.lib().sb200_add(ctx.h, L, 2, B, C_p(at(0)), C_p(at(8 * B * poly)), C_p(at(poly)), ctx._stream()))
        out_words = (poly, poly + 2 * B * poly)
    elif op == "multiply":  # the three-polynomial output starts inside the two-polynomial input
        call = lambda: ctx.d_multiply(at(0), at(8 * B * poly), at(poly), L, B)
        out_words = (poly, poly + 3 * B * poly)
    elif op == "rescale_to_next":  # the output of L - 1 primes starts inside the input
        call = lambda: ctx.d_rescale_to_next_sized(at(0), at(B * poly), L, 2, B)
        out_words = (B * poly, B * poly + 2 * B * (L - 1) * n)
    elif op == "add_many":  # the output starts one polynomial inside operand 1, away from operand 0
        call = lambda: ctx.d_add_many([at(8 * B * poly), at(0)], at(poly), L, B, [2, 2])
        out_words = (poly, poly + 2 * B * poly)
    else:
        key = ctx.load_key(np.stack([np.stack([np.stack([rng.integers(0, mods[i], n, dtype=np.uint64) for i in range(k)])
                                               for _ in range(2)]) for _ in range(k - 1)]))
        call = lambda: ctx.d_apply_galois(at(0), ctx.galois_elt_from_step(1), key, at(2 * poly), L, B)
        out_words = (2 * poly, 2 * poly + 2 * B * poly)
    before = to_np(base[out_words[0]:out_words[1]]).copy()
    launches = ctx.launch_count
    message = r"add_many: the output slab must not overlap an operand \[1\]" if op == "add_many" else "must not overlap input"
    with pytest.raises(ValueError, match=message):  # SB200_E_INVALID_ARG from the overlap check
        call()
    torch.cuda.synchronize()
    assert ctx.launch_count == launches, op
    assert_words(to_np(base[out_words[0]:out_words[1]]), before, f"{op}: the output slab after the refusal")
    words = lambda w0, cts, polys: to_np(base[w0:w0 + cts * polys * poly]).reshape(cts, polys, L, n)
    if op == "add":  # exactly in place (out == a, the same layout) runs, and gives the words of add
        a, b = words(0, B, 2), words(8 * B * poly, B, 2)
        S._check(S.lib().sb200_add(ctx.h, L, 2, B, C_p(at(0)), C_p(at(8 * B * poly)), C_p(at(0)), ctx._stream()))
        torch.cuda.synchronize()
        assert_words(words(0, B, 2), E.linear(0, a, b, mods), "add exactly in place")
    if op == "multiply":  # out == a with three polynomials per ciphertext written over two: refused for a batch above 1
        with pytest.raises(ValueError, match="must not overlap input"):
            ctx.d_multiply(at(0), at(8 * B * poly), at(0), L, B)
        assert ctx.launch_count == launches
    torch.cuda.synchronize()
    ctx.close()


def C_p(v):
    import ctypes

    return ctypes.c_void_p(v)


def test_matrix_coverage():
    """the tuples the matrix reached are exactly the listed ones; every operation ran at every ring size"""
    ids = set(GROUP_IDS) | {f"n{n}-{c}-k64" for n in (2, 4096) for c in ("60-bit", "below-2^61")} | {"n131072-60-bit-k256"}
    if not ids <= DONE:
        pytest.skip("asserted when every group of the matrix has run and passed")
    assert COVERAGE == expected_coverage(), (sorted(expected_coverage() - COVERAGE), sorted(COVERAGE - expected_coverage()))
    for op in OPS + QOPS:
        assert set(SIZES) <= SIZES_SEEN[op], (op, sorted(set(SIZES) - SIZES_SEEN[op]))
    if R.available():
        assert any("reference" in v for v in COMPARED.values())
    print("\n".join(f"{k}: {sorted(v)}" for k, v in sorted(COMPARED.items())))
