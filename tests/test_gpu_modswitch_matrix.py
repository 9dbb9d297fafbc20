"""Parity matrix of rescale and modulus switching (-m gpu; seal_b200/csrc/sb_engine.cu, op_rescale / op_mod_switch).  Every output
word is checked against the big-integer statement of the division (tests/modswitch_ref.py); sampled ciphertexts also against the
oracle (tests/oracle.py) and, where its SEALContext takes the level, the reference.  The axes crossed on purpose:

- transform size n = 2, 8, 64, 128, 256, 512, 2048 (ntt_fwd_small / ntt_inv_small with 32, 64, 128 and 256 threads, fewer and more
  threads than butterflies) and 4096 .. 131072 (the column and local passes at every LOGNA, 4 .. 9);
- butterfly class: every prime below 2^57 with the largest 57-bit prime as data prime and as top prime (the guard-free forward
  butterflies, FAST), or a 60-bit prime in the set (guarded);
- the top prime against the data primes: one set of four primes gives, level by level, a top prime between the data primes (L = 4,
  "mixed"), below every one (L = 3, 25 bits) and far above (L = 2: 57 or 60 bits over 30, the Barrett branch of OpModDownFwd with a
  quotient of 2^27 and more);
- scheme: CKKS rescale_to_next (OpTopIntt + OpModDownFwd) and mod_switch_to_next (the drop, a strided copy), BFV mod_switch_to_next
  (moddown_coeff_kernel<true>), BGV mod_switch_to_next (OpTopIntt writing K = -U q_top^-1 mod t + OpModDownFwdBgv) with t = 65537
  below every prime, a 27-bit t between them and a 60-bit t above all;
- ciphertext size 2, 3 and 16 through the sized entry points;
- words: member j of a batch draws its words by pattern j mod P (modswitch_ref.words): uniform, every word q_i - 1, coefficients at
  the rounding turns X + h = 0, 1, q_l - 1 (mod q_l), coefficients 0, Q - 1 and floor(Q / 2), and for BGV the top residues where
  k = (-r q_l^-1) mod t is 0 and t - 1;
- entry points: the stream entry point on a non-default torch stream; the host entry point with LIMIT_HOST_STAGE_BYTES cut for three
  or more staging chunks and a ragged tail; the stream entry point with LIMIT_SCRATCH_BYTES an odd multiple of the bytes one
  polynomial needs, so that a device chunk (counted in polynomials) ends inside a ciphertext.

The profile asserts the kernels that ran and how many device chunks each entry point cut.  The last test asserts that the module
reached exactly the (transform-size class, operation, FAST, top prime against the data primes, BGV t against the data primes, chunk
split inside a ciphertext) tuples listed in expected_coverage()."""
import itertools
import os
from collections import namedtuple
from concurrent.futures import ProcessPoolExecutor, ThreadPoolExecutor

import numpy as np
import pytest

import modswitch_ref as M
import oracle as O
import refseal as R
from common import assert_words, is_prime, product

pytestmark = pytest.mark.gpu

SIZES = (2, 8, 64, 128, 256, 512, 2048, 4096, 8192, 16384, 32768, 65536, 131072)
# the top prime q_3 (L = 4) between the data primes, q_2 (L = 3) below both, q_1 (L = 2) 57 or 60 bits over a 30-bit q_0
BITS = {True: [30, 57, 25, 45], False: [30, 60, 25, 45]}
LEVELS = (4, 3, 2)
SCRATCH_DEFAULT = 8 << 30  # Context::scratch_budget
STAGE_MIN, SCRATCH_MIN = 1 << 16, 1 << 20  # the smallest LIMIT_HOST_STAGE_BYTES / LIMIT_SCRATCH_BYTES sb200_context_set_limit keeps


def prime_below(bound):
    c = bound - 1
    while not is_prime(c):
        c -= 1
    return c


T_BGV = (65537, prime_below(2 ** 27), prime_below(2 ** 60))
RESCALE, DROP, BFV, BGV = "CKKS-rescale", "CKKS-drop", "BFV", "BGV"

# kind: "CKKS" (rescale and drop), "BFV" or "BGV" (every t of T_BGV on the same words); samples: None = the first and last members
# and both members on each side of every chunk boundary, else these members only
Group = namedtuple("Group", "n kind fast bits size levels samples batch", defaults=(None,))


def sb():
    import seal_b200

    return seal_b200


def size_class(n):
    """which instantiation of the transforms runs: ntt_*_small with clamp(n / 2, 32, 256) threads below n = 4096, else the column
    pass of LOGNA = log2(n) - 8"""
    logn = n.bit_length() - 1
    return f"small{min(max(n // 2, 32), 256)}" if logn < 12 else f"LOGNA{logn - 8}"


def _groups():
    out, i = [], 0
    for n in SIZES:
        for kind, fast in (("CKKS", True), ("CKKS", False), ("BGV", True), ("BGV", False), ("BFV", i % 2 == 0)):
            sizes = (2, 3, 16) if n <= 4096 else (2, 3)
            out.append(Group(n, kind, fast, BITS[fast], sizes[i % len(sizes)], LEVELS, None))
            i += 1
    # the benchmark's shape: 32 primes of 55 bits, the key level L = 32 -> 31, 17 ciphertexts cut into chunks of one polynomial
    out.append(Group(65536, "CKKS", True, [55] * 32, 2, (32,), (0, 16), 17))
    return out


def _group_id(g):
    return f"n{g.n}-{g.kind}-{'q57' if g.fast else 'q60'}-k{len(g.bits)}-size{g.size}"


GROUPS = _groups()
GROUP_IDS = [_group_id(g) for g in GROUPS]
COVERAGE, DONE, REF_COMPARED = set(), set(), set()
ORACLE_ONLY = {}  # (group id, t, L[, ciphertext]): why only the oracle was compared there


def relation(x, others):
    return "above" if all(x > q for q in others) else "below" if all(x < q for q in others) else "mixed"


def expected_coverage():
    """every transform-size class for CKKS rescale and BGV in both butterfly classes, with the top prime between, below and above the
    data primes, a device chunk ending inside a ciphertext and not; BGV with t below, between and above the data primes; BFV (no
    transform, no scratch chunks: its 2^31-word limit is crossed by test_limit_chunks) at every relation of the top prime; the CKKS
    drop (a strided copy) at every size class"""
    out = set()
    classes = {size_class(n) for n in SIZES}
    rel_t = {65537: ("below",) * 3, T_BGV[1]: ("mixed", "below", "below"), T_BGV[2]: ("above",) * 3}  # by level 4, 3, 2
    for cls in classes:
        for fast, (L, rel), split in itertools.product((True, False), zip(LEVELS, ("mixed", "below", "above")), (False, True)):
            out.add((cls, RESCALE, fast, rel, None, split))
            for t in T_BGV:
                out.add((cls, BGV, fast, rel, rel_t[t][LEVELS.index(L)], split))
        for rel in ("mixed", "below", "above"):
            out.add((cls, BFV, None, rel, None, False))
        out.add((cls, DROP, None, None, None, False))
    return out


# ---- chunking, mirrored from op_rescale / op_mod_switch and HostPipe::run ----
def poly_bytes(op, n, L):
    """device scratch one polynomial needs: U and T rows (rescale), U, K and T rows (BGV)"""
    return ((2 if op == BGV else 1) + L - 1) * n * 8


def device_chunk(op, n, L, polys, scratch):
    if op == BFV:
        return max(1, 2 ** 31 // (L * n))
    c = min(polys, max(1, scratch // poly_bytes(op, n, L)))
    return min(c, max(1, 2 ** 30 // (L * n)))


def device_chunks(op, n, L, polys, scratch):
    c = device_chunk(op, n, L, polys, scratch)
    return [c] * (polys // c) + ([polys % c] if polys % c else [])


def host_chunks(B, per_ct, stage):
    chunk = max(1, min(B, stage // per_ct))
    if chunk >= B and B >= 4:
        chunk = (B + 1) // 2
    return [chunk] * (B // chunk) + ([B % chunk] if B % chunk else [])


def host_ct_bytes(n, L, size):
    return size * (2 * L - 1) * n * 8


def split_scratch(op, n, L, size):
    """(LIMIT_SCRATCH_BYTES, polynomials per chunk m): m odd, not a multiple of the ciphertext size, and the budget m polynomials'
    scratch no smaller than the least the library keeps"""
    per = poly_bytes(op, n, L)
    m = max(1, -(-SCRATCH_MIN // per))
    while m % 2 == 0 or m % size == 0:
        m += 1
    return m * per, m


def host_stage(n, L, size):
    """LIMIT_HOST_STAGE_BYTES and the ciphertexts per staging chunk: two at least (so that a tail can be ragged)"""
    per_ct = host_ct_bytes(n, L, size)
    stage = max(2 * per_ct, STAGE_MIN)
    return stage, stage // per_ct


def batch_for(g):
    """ciphertexts: two scratch chunks and a ragged tail at every level, and two staging chunks and a ragged tail"""
    ops = {"CKKS": (RESCALE,), "BGV": (BGV,), "BFV": (BFV,)}[g.kind]
    B = 1
    for L, op in itertools.product(g.levels, ops):
        if op != BFV:
            m = split_scratch(op, g.n, L, g.size)[1]
            B = max(B, -(-(2 * m + 1) // g.size))
        hc = host_stage(g.n, L, g.size)[1]
        B = max(B, 2 * hc + 1)
    while any(B % host_stage(g.n, L, g.size)[1] == 0 for L in g.levels):
        B += 1
    return B


def boundary_members(chunks, per_member):
    """the members on both sides of every boundary between chunks of `chunks` units (polynomials or ciphertexts)"""
    out, u = set(), 0
    for c in chunks[:-1]:
        u += c
        out |= {(u - 1) // per_member, u // per_member}
    return out


# ---- words and checks ----
def member_patterns(g, B):
    pats = [p for p in M.patterns(M.BGV_SWITCH if g.kind == "BGV" else M.CKKS_RESCALE) if p != "bgv_edges"]
    if g.kind == "BGV":
        pats += [("bgv_edges", t) for t in T_BGV]
    return [pats[j % len(pats)] for j in range(B)]


def draw(g, kind, oracles, rng, L, pats):
    """[B][size][L][n] words, member j by pats[j]"""
    B, n = len(pats), g.n
    a = np.empty((B, g.size, L, n), dtype=np.uint64)
    for pat in dict.fromkeys(pats):
        idx = [j for j, p in enumerate(pats) if p == pat]
        name, oc = (pat[0], oracles[pat[1]]) if isinstance(pat, tuple) else (pat, next(iter(oracles.values())))
        a[idx] = M.words(kind, name, rng, oc, L, len(idx) * g.size).reshape(len(idx), g.size, L, n)
    return a


def to_dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def to_np(t):
    return t.cpu().numpy().view(np.uint64)


def check_profile(prof, op, n, L, chunks, what):
    """the kernels of the operation and one launch of each pass per device chunk; a transform pass moves 16 n bytes per row"""
    names = {r[0]: r for r in prof}
    if op == DROP:
        assert not names, f"{what}: the drop launched kernels {sorted(names)}"
        return
    polys = sum(chunks)
    if op == BFV:
        assert set(names) == {"moddown_coeff"}, (what, sorted(names))
        assert names["moddown_coeff"][2] == len(chunks), (what, names["moddown_coeff"], chunks)
        return
    top, ntt = ("rescale_top_intt", "rescale_ntt") if op == RESCALE else ("modswitch_top_intt", "modswitch_ntt")
    passes = ("",) if n < 4096 else (":col", ":local")
    assert set(names) == {f + p for f in (top, ntt) for p in passes}, (what, sorted(names))
    for p in passes:
        assert names[top + p][2] == len(chunks) and names[ntt + p][2] == len(chunks), (what, p, names[top + p], names[ntt + p], chunks)
        assert names[top + p][3] == 16.0 * n * polys and names[ntt + p][3] == 16.0 * n * polys * (L - 1), (what, p)


def ref_switch(rc, op, L, polys):
    """the reference on [P][L][n], two polynomials at a time (an odd last one paired with the first)"""
    P = len(polys)
    pairs = [(p, p + 1 if p + 1 < P else 0) for p in range(0, P, 2)]
    fn = rc.rescale if op == RESCALE else rc.mod_switch
    return np.stack([fn(L, np.ascontiguousarray(polys[[i, j]]))[k] for i, j in pairs for k in ((0, 1) if j else (0,))][:P])


def oracle_switch(oc, op, L, polys):
    P = len(polys)
    fn = {RESCALE: oc.rescale, BFV: oc.bfv_mod_switch, BGV: oc.bgv_mod_switch}[op]
    pad = np.concatenate([polys, polys[:1]]) if P % 2 else polys
    return np.concatenate([fn(L, np.ascontiguousarray(pad[p:p + 2])) for p in range(0, len(pad), 2)])[:P]


def run_entry_points(S, ctx, op, g, L, a_np, a_dev, B):
    """(entry point, output [B][size][L-1][n], device chunks) of the three entry points on the same words"""
    import torch

    n, size = g.n, g.size
    host = ctx.rescale_to_next if op == RESCALE else ctx.mod_switch_to_next
    stream_fn = ctx.d_rescale_to_next_sized if op == RESCALE else ctx.d_mod_switch_to_next_sized
    res = []

    def on_stream(label, scratch):
        ctx.set_limit(ctx.LIMIT_SCRATCH_BYTES, scratch)
        out = torch.empty((B, size, L - 1, n), dtype=torch.int64, device="cuda")
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        ctx.profile(True)
        with torch.cuda.stream(s):
            stream_fn(a_dev, out, L, size, B)
        s.synchronize()
        prof = ctx.profile_read()
        ctx.profile(False)
        chunks = device_chunks(op, n, L, B * size, scratch)
        check_profile(prof, op, n, L, chunks if op != DROP else [], f"{label}, L = {L}")
        res.append((label, to_np(out), chunks))

    on_stream("stream entry point, non-default stream", SCRATCH_DEFAULT)
    stage, _ = host_stage(n, L, size)
    ctx.set_limit(ctx.LIMIT_HOST_STAGE_BYTES, stage)
    ctx.profile(True)
    got = host(a_np)
    prof = ctx.profile_read()
    ctx.profile(False)
    hchunks = host_chunks(B, host_ct_bytes(n, L, size), stage)
    assert len(hchunks) >= 3 and hchunks[-1] != hchunks[0], hchunks
    dchunks = [c for h in hchunks for c in device_chunks(op, n, L, h * size, SCRATCH_DEFAULT)]
    check_profile(prof, op, n, L, dchunks if op != DROP else [], f"host entry point, staging chunks {hchunks}, L = {L}")
    res.append((f"host entry point, staging chunks {hchunks}", got, hchunks))
    if op not in (BFV, DROP):
        on_stream("stream entry point, scratch cut inside a ciphertext", split_scratch(op, n, L, size)[0])
    ctx.set_limit(ctx.LIMIT_SCRATCH_BYTES, SCRATCH_DEFAULT)
    return res


@pytest.fixture(scope="module")
def statement_pool():
    """processes for the big-integer statement (spawned: they import numpy and tests/modswitch_ref.py only, never CUDA)"""
    import multiprocessing

    with ProcessPoolExecutor(max_workers=min(16, os.cpu_count() or 1), mp_context=multiprocessing.get_context("spawn")) as pool:
        yield pool


@pytest.mark.parametrize("g", [pytest.param(g, id=i) for g, i in zip(GROUPS, GROUP_IDS)])
def test_modswitch_matrix(g, statement_pool):
    S = sb()
    gid = GROUP_IDS[GROUPS.index(g)]
    n, cls = g.n, size_class(g.n)
    mods = O.coeff_modulus_create(n, g.bits)
    assert all(q < 2 ** 57 for q in mods) == g.fast and (57 not in g.bits or max(mods) >> 56 == 1)
    ts = {"CKKS": (0,), "BFV": (65537,), "BGV": T_BGV}[g.kind]
    oracles = {t: O.Oracle(getattr(O, g.kind), n, mods, t) for t in ts}
    kind = {"CKKS": M.CKKS_RESCALE, "BFV": M.BFV_SWITCH, "BGV": M.BGV_SWITCH}[g.kind]
    B = g.batch or batch_for(g)
    pats = member_patterns(g, B)
    rng = np.random.default_rng(GROUPS.index(g))
    refs = {}
    for t in ts:
        try:
            refs[t] = R.RefContext(getattr(R, g.kind), n, mods, t) if R.available() else None
        except RuntimeError as e:
            refs[t] = None
            ORACLE_ONLY[(gid, t, None)] = f"the reference's SEALContext refused the parameters: {e}"

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as pool:
        for L in g.levels:
            a = draw(g, kind, oracles, rng, L, pats)
            a_dev = to_dev(a)
            lout = L - 1
            data, q_top = mods[:lout], mods[L - 1]
            ops = [(RESCALE, 0), (DROP, 0)] if g.kind == "CKKS" else [(g.kind, t) for t in ts]
            for op, t in ops:
                what = f"{op}{f' t = {t}' if t else ''}, L = {L}"
                want = a[:, :, :lout] if op == DROP else M.expected(kind, oracles[t], a, statement_pool)
                ctx = S.Context(getattr(S, g.kind), n, mods, t) if t else S.Context(S.CKKS, n, mods)
                results = run_entry_points(S, ctx, op, g, L, a, a_dev, B)
                ctx.close()
                samples = set(g.samples or ()) or {0, B - 1}
                for label, got, chunks in results:
                    assert_words(got, want, f"{what}, {label}: vs the big-integer statement")
                    per_member = 1 if label.startswith("host") else g.size
                    if g.samples is None:
                        samples |= boundary_members(chunks, per_member)
                    split = any(u % g.size for u in itertools.accumulate(chunks[:-1])) if per_member == g.size else False
                    rel = relation(q_top, data) if op != DROP else None
                    COVERAGE.add((cls, op, g.fast if op in (RESCALE, BGV) else None, rel, relation(t, data) if op == BGV else None,
                                  split if op in (RESCALE, BGV) else False))
                if op == DROP:
                    continue
                # sampled members against the oracle (on the host threads) and the reference
                futs = {j: pool.submit(oracle_switch, oracles[t], op, L, a[j]) for j in sorted(samples) if j < B}
                rc = refs[t]
                for j, f in futs.items():
                    assert_words(results[0][1][j], f.result(), f"{what}, ciphertext {j}: vs the oracle")
                    if rc is None:
                        continue
                    if L == len(mods):
                        ORACLE_ONLY[(gid, t, L)] = "the reference keeps no ciphertexts at the key level"
                        continue
                    if t and product(mods[:lout]) <= t:
                        ORACLE_ONLY[(gid, t, L)] = "the reference's modulus chain ends above a level whose modulus is not above t"
                        continue
                    try:
                        rw = ref_switch(rc, op, L, a[j])
                    except RuntimeError as e:  # SEAL throws on a result whose c_1 is zero, as the words q_i - 1 give
                        if "transparent" not in str(e):
                            raise
                        ORACLE_ONLY[(gid, t, L, j)] = "the reference refused the transparent result"
                        continue
                    assert_words(results[0][1][j], rw, f"{what}, ciphertext {j}: vs the reference")
                    REF_COMPARED.add(op)
            del a_dev
    for rc in refs.values():
        if rc is not None:
            rc.close()
    DONE.add(gid)


@pytest.mark.parametrize("op", [RESCALE, BFV])
def test_limit_chunks(op):
    """the 2^30 / (L n)-polynomial chunks of op_rescale and the 2^31 / (L n)-polynomial chunks of BFV's op_mod_switch at L = 2,
    crossed by a batch of 8 GiB / 16 GiB on the device; the two polynomials on each side of the limit against the statement"""
    import torch

    S = sb()
    n, L = 131072, 2
    limit = (2 ** 30 if op == RESCALE else 2 ** 31) // (L * n)
    polys = limit + 2
    in_bytes, out_bytes = polys * L * n * 8, polys * (L - 1) * n * 8
    scratch = poly_bytes(op, n, L) * limit if op == RESCALE else 0
    free, _ = torch.cuda.mem_get_info()
    need = in_bytes + out_bytes + scratch + (2 << 30)
    if free < need:
        pytest.skip(f"needs {need / 2 ** 30:.1f} GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
    mods = O.coeff_modulus_create(n, [50, 45])
    t = 65537 if op == BFV else 0
    ctx = S.Context(S.BFV, n, mods, t) if t else S.Context(S.CKKS, n, mods)
    oc = O.Oracle(O.BFV if t else O.CKKS, n, mods, t)
    a = torch.empty((polys // 2, 2, L, n), dtype=torch.int64, device="cuda")
    g = torch.Generator(device="cuda")
    g.manual_seed(polys)
    for i in range(L):
        a[:, :, i].random_(0, mods[i], generator=g)
    out = torch.empty((polys // 2, 2, L - 1, n), dtype=torch.int64, device="cuda")
    ctx.set_limit(ctx.LIMIT_SCRATCH_BYTES, 4 * SCRATCH_DEFAULT)  # the polynomial limit, not the scratch budget, cuts the chunks
    ctx.profile(True)
    (ctx.d_rescale_to_next_sized if op == RESCALE else ctx.d_mod_switch_to_next_sized)(a, out, L, 2, polys // 2)
    torch.cuda.synchronize()
    prof = {r[0]: r for r in ctx.profile_read()}
    ctx.profile(False)
    name = "rescale_ntt:local" if op == RESCALE else "moddown_coeff"
    assert prof[name][2] == 2, (prof, limit)
    idx = [0, limit - 1, limit, polys - 1]  # polynomial indices; limit - 1 | limit straddle the chunk boundary
    flat_in, flat_out = a.view(polys, L, n), out.view(polys, L - 1, n)
    got = np.stack([to_np(flat_out[p]) for p in idx])
    src = np.stack([to_np(flat_in[p]) for p in idx])
    del a, out, flat_in, flat_out
    ctx.close()
    torch.cuda.empty_cache()
    kind = M.CKKS_RESCALE if op == RESCALE else M.BFV_SWITCH
    assert_words(got, M.expected(kind, oc, src), f"{op}: polynomials {idx} around the {limit}-polynomial chunk limit")


def test_matrix_coverage():
    """the tuples the matrix reached are exactly the listed ones; the reference was compared for every operation it has"""
    if DONE != set(GROUP_IDS):
        pytest.skip("asserted when every group of the matrix has run and passed")
    assert COVERAGE == expected_coverage(), (sorted(expected_coverage() - COVERAGE, key=str), sorted(COVERAGE - expected_coverage(), key=str))
    if R.available():
        assert REF_COMPARED == {RESCALE, BFV, BGV}, REF_COMPARED
    # where only the oracle was compared, and why
    print("\n".join(f"oracle only: {k}: {v}" for k, v in sorted(ORACLE_ONLY.items(), key=str)))
