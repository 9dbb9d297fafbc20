"""Parity matrix of the integer key-switching path (-m gpu; seal_b200/csrc/sb_ksint.cu).  The path picks among many kernel
instantiations on the transform size, the scheme, the prime sizes, the chunk size and four environment switches; this module
crosses those axes on purpose, so that every instantiation runs inside a whole key switch and is compared word for word:

- transform size n = 4096 .. 131072: every LOGN of launch_mac_logn / launch_crt / ksint_target_intt, every LOGNA of
  launch_crt_ntt (the outer stages ride in other kernels at n = 8192 .. 65536 only);
- scheme CKKS / BFV / BGV (reconstruction MODE 0 / 1 / 3);
- primes all below 2^57, or a set with 60-bit primes (FAST = false: the guarded 64-bit butterflies);
- level: the key level L = k - 1, and L = k - 3, where key row (J, c, I') of the product kernels sits at a stride of k, not L + 1;
- operation: relinearize, multiply_relinearize, and apply_galois with steps 1, -1, n/4 - 1 and the element 2n - 1 (Galois views
  of the target: a permutation of NTT-form words for CKKS / BGV, a signed automorphism of coefficients for BFV);
- batch 16, 17, 33 and 33 in chunks of 20 (a chunk of 20 and a ragged tail of 13), and prefixes of 15 and 1 ciphertexts;
- product kernel, selected per chunk by launch_mac: the INT8 tensor-core kernel ks32_mac_mma when L <= 32 digits and the chunk
  holds at least 16 ciphertexts (unless SB200_KS_MAC_MMA=0); else the key-tile kernel ks32_mac_tile when the chunk holds at least
  16 ciphertexts and the key tile L * 4096 bytes + the 64 KB ring fits 227 KB (unless SB200_KS_MAC_TILE=0); else the register-tile
  kernel ks32_mac.  The profile shows whether the tensor-core kernel ran (it does no 32-bit multiply-accumulates); key tile and
  register tile are told apart only by the switches, so each group runs under all three;
- reconstruction: entry and exit fused into the 64-bit transforms' column passes (ks32_intt_fwd_outer, ks32_inv_crt_ntt), the
  outer inverse stages fused into ks32_crt_kernel, or neither (SB200_KS_FUSE_NTT=0, SB200_KS_FUSE_CRT=0).

Each group draws one batch on the device and checks: sampled ciphertexts {0, 15, 16, B - 1} of the 64-bit path against the oracle
(tests/oracle.py), every word; every variant's whole batch against the 64-bit path (LIMIT_KS_ALGORITHM = 0, independent code),
word for word; and, from the profile, that the intended kernels ran.  The last test asserts that the module reached exactly the
(LOGN, scheme, FAST, product kernel, reconstruction, Galois view) tuples listed in expected_coverage()."""
import itertools
import os
from collections import namedtuple
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import oracle as O
from common import assert_words

pytestmark = pytest.mark.gpu

KS_64, KS_INT = 0, 2  # SB200_LIMIT_KS_ALGORITHM
MMA, TILE, REG = "mma", "tile", "reg"
KERNELS = (MMA, TILE, REG)
KERNEL_ENV = {MMA: {}, TILE: {"SB200_KS_MAC_MMA": "0"}, REG: {"SB200_KS_MAC_MMA": "0", "SB200_KS_MAC_TILE": "0"}}
FUSION_ENV = {"default": {}, "no_fuse_ntt": {"SB200_KS_FUSE_NTT": "0"}, "no_fuse_crt": {"SB200_KS_FUSE_CRT": "0"}}
SWITCHES = ("SB200_KS_MAC_MMA", "SB200_KS_MAC_TILE", "SB200_KS_FUSE_NTT", "SB200_KS_FUSE_CRT")
MMA_MAX_DIGITS, TILE_RING_BYTES, TILE_SMEM_MAX = 32, 8 * 4 * 512 * 4, 227 * 1024  # sb_ksint.cu: kMmaMaxDigits, kMacRingBytes
PLAIN_MODULUS = {"CKKS": 0, "BFV": 65537, "BGV": 65537}
# k = 6 primes; the first data prime and the special prime are the largest: 57 bits (the guard-free butterflies' limit) or 60
BITS = {True: [57, 50, 54, 52, 56, 57], False: [60, 50, 54, 52, 56, 60]}
SIZES = (4096, 8192, 16384, 32768, 65536, 131072)
BATCHES = ((16, 0), (17, 0), (33, 0), (33, 20))  # (ciphertexts, LIMIT_KS_CHUNK)
GALOIS = ("galois(+1)", "galois(-1)", "galois(n/4-1)", "galois(2n-1)")
REL, MULREL = "relinearize", "multiply_relinearize"

# runs: ((operation, level), ...) on the whole batch under every variant; prefixes: ((operation, level, ciphertexts), ...) under
# the default product-kernel switches only (below 16 ciphertexts the register-tile kernel runs whatever they say)
Group = namedtuple("Group", "n scheme fast bits batch chunk runs prefixes fusions samples")


def sb():
    import seal_b200

    return seal_b200


def _groups():
    """every (transform size, scheme, prime class) once -- BFV with one prime class per size, alternating -- with the batch
    shape, the Galois step, the other operation and the level of each rotating independently; then the headline shape"""
    out, i = [], 0
    for n in SIZES:
        logn = n.bit_length() - 1
        for scheme in ("CKKS", "BGV", "BFV"):
            for fast in ((True, False) if scheme != "BFV" else (logn % 2 == 0,)):
                batch, chunk = BATCHES[i % 4]
                gal, other = GALOIS[(i + i // 4) % 4], (REL, MULREL)[(i // 2) % 2]
                lg, lo = (5, 3) if i % 2 == 0 else (3, 5)
                out.append(Group(n, scheme, fast, BITS[fast], batch, chunk, ((gal, lg), (other, lo)), ((gal, lg, 15), (other, lo, 1)),
                                 tuple(FUSION_ENV), None))
                i += 1
    # the benchmark's shape: 31 digits (the tensor-core kernel's largest output tiling short of 32), 5 auxiliary primes; the oracle
    # takes seconds per ciphertext here, so two samples per operation
    out.append(Group(65536, "CKKS", True, [55] * 32, 17, 0, ((REL, 31), (GALOIS[0], 29)), (), ("default",), (0, 16)))
    return out


def _group_id(g):
    runs = "-".join(f"{op}@L{L}" for op, L in g.runs)
    return f"n{g.n}-{g.scheme}-{'q57' if g.fast else 'q60'}-k{len(g.bits)}-B{g.batch}" + (f"c{g.chunk}" if g.chunk else "") + "-" + runs


GROUPS = _groups()
GROUP_IDS = [_group_id(g) for g in GROUPS]
COVERAGE, KEY_ROWS, DONE = set(), set(), set()


def fusion_label(logn, scheme, env):
    """what ksint_core fuses under a SB200_KS_FUSE_* setting: "ntt" = entry and exit in the 64-bit column passes
    (ks32_intt_fwd_outer, ks32_inv_crt_ntt; CKKS / BGV), "crt" = the outer inverse stages in the reconstruction; n = 8192 .. 65536"""
    outer = 13 <= logn <= 16
    crt = outer and env != "no_fuse_crt"
    ntt = outer and scheme != "BFV" and env != "no_fuse_ntt"
    return {(True, True): "ntt+crt", (False, True): "crt", (True, False): "ntt", (False, False): "none"}[(ntt, crt)]


def product_kernel(switch, L, chunk):
    """launch_mac's choice for one chunk under the product-kernel switch (MMA: the defaults)"""
    if switch == MMA and L <= MMA_MAX_DIGITS and chunk >= 16:
        return MMA
    if switch != REG and L * 4096 + TILE_RING_BYTES <= TILE_SMEM_MAX and chunk >= 16:
        return TILE
    return REG


def expected_coverage():
    """(LOGN, scheme, FAST, product kernel, reconstruction, Galois view): every product kernel at every transform size
    (launch_mac_logn: LOGN 12 .. 17), under every reconstruction the size has (launch_crt: outer stages fused at LOGN 13 .. 16;
    launch_crt_ntt / ksint_target_intt: entry and exit fused at LOGN 13 .. 16 for MODE 0 and 3), plain and through a Galois view,
    for CKKS and BGV with both prime classes (ks32_inv_crt_ntt<MODE, LOGNA, FAST>) and BFV with one (FAST does not reach MODE 1)"""
    fusions = {"CKKS": ("ntt+crt", "crt", "ntt"), "BGV": ("ntt+crt", "crt", "ntt"), "BFV": ("crt", "none")}
    out = set()
    for logn in range(12, 18):
        for scheme in ("CKKS", "BGV", "BFV"):
            fasts = (True, False) if scheme != "BFV" else (logn % 2 == 0,)
            fus = fusions[scheme] if 13 <= logn <= 16 else ("none",)
            out |= set(itertools.product((logn,), (scheme,), fasts, KERNELS, fus, (False, True)))
    return out


def device_rand(mods, n, prefix, rows, seed):
    """uniform residues [*prefix][rows][n] on the device, row i modulo mods[i]"""
    import torch

    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    t = torch.empty((*prefix, rows, n), dtype=torch.int64, device="cuda")
    for i in range(rows):
        t[..., i, :] = torch.randint(0, mods[i], (*prefix, n), generator=g, dtype=torch.int64, device="cuda")
    return t


def to_np(t):
    return t.cpu().numpy().view(np.uint64)


def galois_elt(op, n):
    return {"galois(+1)": lambda: O.galois_elt_from_step(n, 1), "galois(-1)": lambda: O.galois_elt_from_step(n, -1),
            "galois(n/4-1)": lambda: O.galois_elt_from_step(n, n // 4 - 1), "galois(2n-1)": lambda: 2 * n - 1}[op]()


def keyswitch(ctx, rk, op, args, L, B):
    import torch

    out = torch.empty((B, 2, L, ctx.n), dtype=torch.int64, device="cuda")
    if op == REL:
        ctx.d_relinearize(args[0][:B], rk, out, L, B)
    elif op == MULREL:
        ctx.d_multiply_relinearize(args[0][:B], args[1][:B], rk, out, L, B)
    else:
        ctx.d_apply_galois(args[0][:B], galois_elt(op, ctx.n), rk, out, L, B)
    torch.cuda.synchronize()
    return out


def oracle_keyswitch(oc, op, L, host_args, key):
    if op == REL:
        return oc.relinearize(L, host_args[0], key)
    if op == MULREL:
        return oc.multiply_relin(L, host_args[0], host_args[1], key)
    return oc.apply_galois(L, host_args[0], galois_elt(op, oc.n), key)


def chunks_of(ctx, op, L, B):
    c = ctx.keyswitch_chunk(L, B, fused=(op == MULREL))
    return [c] * (B // c) + ([B % c] if B % c else [])


def check_profile(prof, ctx, logn, label, L, chunks, kernels, what):
    """the kernels of ksint_core that ran, from the profile: 32-bit multiply-accumulates only in the chunks that did not take the
    tensor cores, and the entry / reconstruction kernels of the fusion in effect"""
    names = {r[0].split(":")[0] for r in prof}  # the transform kernels' records carry their pass: "ks_target_intt_aux:col"
    assert "ks32_mac" in names, f"{what}: the integer path did not run"
    S, n = len(ctx.ksint_primes()), ctx.n
    want = sum(c * 2 * (L + 1) * L * S * n for c, kern in zip(chunks, kernels) if kern != MMA)
    got = sum(r[7] for r in prof if r[0] == "ks32_mac")
    assert got == want, f"{what}: 32-bit multiply-accumulates {got}, want {want} (chunks {chunks}, kernels {kernels})"
    ntt, crt = label in ("ntt+crt", "ntt"), label in ("ntt+crt", "crt")
    assert ("ks_target_intt_aux" in names) == ntt and ("ks32_fwd_outer" in names) == (not ntt), (what, sorted(names))
    assert ("ks32_inv_crt_ntt" in names) == (ntt and crt) and ("ks32_crt" in names) == (not (ntt and crt)), (what, sorted(names))
    assert ("ks32_inv_outer" in names) == (logn > 12 and not crt), (what, sorted(names))


@pytest.mark.parametrize("g", [pytest.param(g, id=i) for g, i in zip(GROUPS, GROUP_IDS)])
def test_keyswitch_matrix(g, monkeypatch):
    import torch

    S = sb()
    for v in SWITCHES:
        monkeypatch.delenv(v, raising=False)
    n, logn, scheme, B = g.n, g.n.bit_length() - 1, g.scheme, g.batch
    mods = O.coeff_modulus_create(n, g.bits)
    k, t = len(mods), PLAIN_MODULUS[scheme]
    assert all(q < 2 ** 57 for q in mods) == g.fast
    oc = O.Oracle(getattr(O, scheme), n, mods, t)
    seed = GROUPS.index(g)
    key_d = device_rand(mods, n, (k - 1, 2), k, 1000 + seed)
    key = to_np(key_d)
    del key_d
    parts = {REL: (3,), MULREL: (2, 2)}
    full = {}
    for j, (op, _) in enumerate(g.runs):
        full[op] = tuple(device_rand(mods, n, (B, p), k - 1, 2000 + 10 * seed + 3 * j + h) for h, p in enumerate(parts.get(op, (2,))))
    args = {(op, L): tuple(x[:, :, :L].contiguous() for x in full[op]) for op, L in g.runs}
    del full
    assert {L for _, L in g.runs} == {k - 1, k - 3}

    def samples(B_):
        return sorted({s for s in (g.samples or (0, 15, 16, B_ - 1)) if s < B_} | {B_ - 1})

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as pool:
        # the oracle runs on the host while the device works (its entry points only read the context)
        want = {}
        for op, L in g.runs:
            idx = set(samples(B)) | {s for o, l, b in g.prefixes if (o, l) == (op, L) for s in samples(b)}
            for i in sorted(idx):
                want[(op, L, i)] = pool.submit(oracle_keyswitch, oc, op, L, tuple(to_np(x[i]) for x in args[(op, L)]), key)

        def context(env):
            for v in SWITCHES:
                monkeypatch.delenv(v, raising=False)
            for v, val in env.items():
                monkeypatch.setenv(v, val)
            ctx = S.Context(getattr(S, scheme), n, mods, t) if t else S.Context(S.CKKS, n, mods)
            rk = ctx.load_key(key)
            if g.chunk:
                ctx.set_limit(ctx.LIMIT_KS_CHUNK, g.chunk)
            return ctx, rk

        # the 64-bit path: the whole batch every variant must reproduce
        ctx, rk = context({})
        ctx.set_limit(ctx.LIMIT_KS_ALGORITHM, KS_64)
        ref = {(op, L): keyswitch(ctx, rk, op, args[(op, L)], L, B) for op, L in g.runs}
        del rk
        ctx.close()

        labels = {}
        for env in g.fusions:
            labels.setdefault(fusion_label(logn, scheme, env), env)  # switches that change nothing here are not rerun
        for (label, fenv), ksw in itertools.product(labels.items(), KERNELS):
            variant = f"kernel switch {ksw}, reconstruction {label}"
            ctx, rk = context({**KERNEL_ENV[ksw], **FUSION_ENV[fenv]})
            ctx.set_limit(ctx.LIMIT_KS_ALGORITHM, KS_INT)
            runs = [(op, L, B) for op, L in g.runs] + [p for p in g.prefixes if ksw == MMA]
            for op, L, b in runs:
                chunks = chunks_of(ctx, op, L, b)
                kernels = [product_kernel(ksw, L, c) for c in chunks]
                what = f"{op} at L = {L}, {b} ciphertexts, {variant}"
                ctx.profile(True)
                got = keyswitch(ctx, rk, op, args[(op, L)], L, b)
                prof = ctx.profile_read_work32()
                ctx.profile(False)
                check_profile(prof, ctx, logn, label, L, chunks, kernels, what)
                if not torch.equal(got, ref[(op, L)][:b]):
                    assert_words(to_np(got), to_np(ref[(op, L)][:b]), f"{what} (chunks {chunks}, kernels {kernels}) vs the 64-bit path")
                for kern in kernels:
                    COVERAGE.add((logn, scheme, g.fast, kern, label, op.startswith("galois")))
                    KEY_ROWS.add((logn, kern, L < k - 1))
            del rk
            ctx.close()

        for (op, L, i), fut in want.items():
            assert_words(to_np(ref[(op, L)][i]), fut.result(), f"{op} at L = {L}, ciphertext {i}: the 64-bit and integer paths vs the oracle")
    DONE.add(GROUP_IDS[GROUPS.index(g)])


def test_matrix_coverage():
    """the dispatch tuples the matrix reached are exactly the listed ones: a dispatcher change that stops running a kernel
    instantiation (or starts running one the list does not name) fails here"""
    if DONE != set(GROUP_IDS):
        pytest.skip("asserted when every group of the matrix has run and passed")
    assert COVERAGE == expected_coverage(), (sorted(expected_coverage() - COVERAGE), sorted(COVERAGE - expected_coverage()))
    # every product kernel at every transform size with the key's own stride (L = k - 1) and with strided key rows (L < k - 1)
    assert KEY_ROWS == set(itertools.product(range(12, 18), KERNELS, (False, True))), sorted(KEY_ROWS)
