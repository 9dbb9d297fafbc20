"""Plaintext matrix times encrypted vector by diagonals: sb200_apply_galois_multiply_plain_add (out = addend + plain *
apply_galois(in)) and sb200_diagonal_sum (out = sum_i plain_i * apply_galois(in, elt_i), element 1 = no rotation), both entry points,
word for word against the chained device calls (sb200_apply_galois, then sb200_multiply_plain_n or _coeff_n, then a two-operand
sb200_add_many), against the plain-C oracle (tests/oracle.py) and against the reference's own rotate / multiply_plain / add chain
(oracle/_ref); and a CKKS and a BFV 8 x 8 matrix times a vector, decrypted and decoded by the reference."""
import os
import subprocess
import zlib

import numpy as np
import pytest

import oracle as O
import refseal as R
from common import assert_words, max_ct, rand_ct, unreduce

pytestmark = pytest.mark.gpu

KS_64, KS_INT = 0, 2  # SB200_LIMIT_KS_ALGORITHM
SCHEMES = ("CKKS", "BFV", "BGV")
FUSE_SWITCHES = ("SB200_KS_FUSE_NTT", "SB200_KS_FUSE_CRT")


def sb():
    import seal_b200

    return seal_b200


def dev(x):
    import torch

    return torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint64)


def sync():
    import torch

    torch.cuda.synchronize()


def seed_of(*parts):
    """a seed that depends only on the test's parameters (Python's str hash is randomised per process)"""
    return zlib.crc32(repr(parts).encode())


def scheme_id(name):
    return {"CKKS": sb().CKKS, "BFV": sb().BFV, "BGV": sb().BGV}[name]


def make(name, n, mods, algo=KS_64):
    t = 0 if name == "CKKS" else int(O.get_primes(2 * n, 20, 1)[0])
    ctx = sb().Context(scheme_id(name), n, mods, t)
    ctx.set_limit(ctx.LIMIT_KS_ALGORITHM, algo)
    return ctx, t


def rand_key(rng, mods, n):
    k = len(mods)
    return np.stack([np.stack([np.stack([rng.integers(0, mods[i], n, dtype=np.uint64) for i in range(k)])
                               for _ in range(2)]) for _ in range(k - 1)])


def elt_of(n, step):
    """step None: the element 2n - 1; step 0: the identity element 1"""
    if step is None:
        return 2 * n - 1
    return 1 if step == 0 else O.galois_elt_from_step(n, step)


def default_ntt(name):
    """the plaintext form each scheme's diagonals usually come in: NTT form for CKKS / BGV, coefficient form for BFV"""
    return name != "BFV"


def rand_plain(rng, mods, n, L, count, t, ntt):
    """count plaintexts: NTT form [count][L][n] (words below q_i) or coefficient form [count][n] (words below t)"""
    if ntt:
        return np.stack([np.stack([rng.integers(0, mods[i], n, dtype=np.uint64) for i in range(L)]) for _ in range(count)])
    return rng.integers(0, t, (count, n), dtype=np.uint64)


def chain_term(ctx, name, x, elt, key, plain, plain_ntt):
    """t = apply_galois(x) (x itself for element 1), then multiply_plain as the reference multiplies t: the NTT-form product, the
    coefficient-form plaintext's lift (_coeff_n), or (BFV with an NTT-form plaintext) t to NTT form, the product, back"""
    B, _, L, n = x.shape
    d_t = dev(x)
    if elt != 1:
        src, d_t = d_t, dev(np.zeros_like(x))
        ctx.d_apply_galois(src, elt, key, d_t, L, B)
    d_p, pc = dev(plain), plain.shape[0]
    if not plain_ntt:
        ctx.d_multiply_plain_coeff_n(d_t, d_p, d_t, L, 2, B, pc, int(name != "BFV"))
    elif name == "BFV":
        ctx.d_ntt_forward(d_t, L, 2, B)
        ctx.d_multiply_plain_n(d_t, d_p, d_t, L, 2, B, pc)
        ctx.d_ntt_inverse(d_t, L, 2, B)
    else:
        ctx.d_multiply_plain_n(d_t, d_p, d_t, L, 2, B, pc)
    return d_t


def chain_mpa(ctx, name, x, elt, key, plain, addend, plain_ntt=True):
    """the chained device calls of one term: chain_term, then a two-operand add_many onto the addend"""
    B, _, L, n = x.shape
    d_t = chain_term(ctx, name, x, elt, key, plain, plain_ntt)
    out = dev(np.zeros_like(x))
    ctx.d_add_many([dev(addend), d_t], out, L, B, [2, 2])
    sync()
    return host(out)


def chain_diag(ctx, name, x, elts, keys, plains, plain_ntt):
    """for each i: t = chain_term(x, elt_i, plain_i); i == 0 ? destination = t : destination = add_many(destination, t)"""
    B, _, L, n = x.shape
    dest = None
    for e, k, p in zip(elts, keys, plains):
        d_t = chain_term(ctx, name, x, e, k, p, plain_ntt)
        if dest is None:
            dest = d_t
        else:
            out = dev(np.zeros_like(x))
            ctx.d_add_many([dest, d_t], out, L, B, [2, 2])
            dest = out
    sync()
    return host(dest)


def fused_mpa(ctx, x, elt, key, plain, addend):
    """the stream entry point (a fresh output, then accumulated into the addend) and the host form: all equal, inputs unchanged"""
    B, _, L, n = x.shape
    d_x, d_p, d_a, out = dev(x), dev(plain), dev(addend), dev(np.zeros_like(x))
    ctx.d_apply_galois_multiply_plain_add(d_x, elt, key, d_p, plain.shape[0], d_a, out, L, B)
    ctx.d_apply_galois_multiply_plain_add(d_x, elt, key, d_p, plain.shape[0], d_a, d_a, L, B)  # out = addend: accumulate
    sync()
    got = host(out)
    assert_words(host(d_a), got, "accumulated into the addend vs a fresh output")
    assert_words(host(d_x), x, "input unchanged")
    assert_words(host(d_p), plain, "plaintext unchanged")
    assert_words(ctx.apply_galois_multiply_plain_add(x, elt, key, plain, addend), got, "host form vs stream form")
    return got


def fused_diag(ctx, x, elts, keys, plains, plain_ntt):
    """the stream entry point and the host form: equal, input unchanged"""
    B, _, L, n = x.shape
    d_x, out = dev(x), dev(np.zeros_like(x))
    ctx.d_diagonal_sum(d_x, elts, keys, [dev(p) for p in plains], [p.shape[0] for p in plains], out, L, B, plain_ntt)
    sync()
    got = host(out)
    assert_words(host(d_x), x, "input unchanged")
    assert_words(ctx.diagonal_sum(x, elts, keys, plains, plain_ntt), got, "host form vs stream form")
    return got


def oracle_term(oc, name, L, xb, elt, hkey, plain, plain_ntt):
    t = xb if elt == 1 else oc.apply_galois(L, xb, elt, hkey)
    if not plain_ntt:
        return oc.multiply_plain_coeff(L, t, plain, int(name != "BFV"))
    if name == "BFV":
        return oc.ntt_inverse(L, oc.multiply_plain(L, oc.ntt_forward(L, t), plain))
    return oc.multiply_plain(L, t, plain)


def oracle_diag(oc, name, L, x, elts, hkeys, plains, plain_ntt):
    out = []
    for b in range(x.shape[0]):
        acc = None
        for e, h, p in zip(elts, hkeys, plains):
            term = oracle_term(oc, name, L, x[b], e, h, p[0] if p.shape[0] == 1 else p[b], plain_ntt)
            acc = term if acc is None else oc.linear(0, L, acc, term)
        out.append(acc)
    return np.stack(out)


_CASES = {}


def case(name, algo):
    """one context per scheme and key-switching path: n = 4096, k = 6 (the integer path at every level with algo = KS_INT)"""
    key = (name, algo)
    if key not in _CASES:
        n = 4096
        mods = O.coeff_modulus_create(n, [50, 40, 40, 40, 40, 50])
        ctx, t = make(name, n, mods, algo)
        _CASES[key] = (n, mods, t, ctx, O.Oracle(scheme_id(name), n, mods, t))
    return _CASES[key]


def terms(rng, n, mods, t, L, B, steps, counts, plain_ntt, ctx):
    elts = [elt_of(n, s) for s in steps]
    hkeys = [None if e == 1 else rand_key(rng, mods, n) for e in elts]
    keys = [None if h is None else ctx.load_key(h) for h in hkeys]
    plains = [rand_plain(rng, mods, n, L, c, t, plain_ntt) for c in counts]
    return elts, hkeys, keys, plains


@pytest.mark.parametrize("name", SCHEMES)
@pytest.mark.parametrize("algo", [KS_64, KS_INT])
@pytest.mark.parametrize("step", [1, -1, "n/4-1", None])
@pytest.mark.parametrize("shared", [True, False])
def test_apply_galois_multiply_plain_add_matrix(name, algo, step, shared):
    """every scheme, both key-switching paths, steps 1, -1, n/4 - 1 and the element 2n - 1, shared and per-member NTT-form
    plaintexts, against the chain and the oracle"""
    n, mods, t, ctx, oc = case(name, algo)
    L, B = 4, 3
    s = n // 4 - 1 if step == "n/4-1" else step
    elt = elt_of(n, s)
    rng = np.random.default_rng(seed_of(name, algo, str(step), shared))
    hkey = rand_key(rng, mods, n)
    key = ctx.load_key(hkey)
    x, a = rand_ct(rng, mods, n, 2, L, B), rand_ct(rng, mods, n, 2, L, B)
    plain = rand_plain(rng, mods, n, L, 1 if shared else B, t, True)
    got = fused_mpa(ctx, x, elt, key, plain, a)
    assert_words(got, chain_mpa(ctx, name, x, elt, key, plain, a), f"{name} vs chain")
    want = np.stack([oc.linear(0, L, a[b], oracle_term(oc, name, L, x[b], elt, hkey, plain[0 if shared else b], True)) for b in range(B)])
    assert_words(got, want, f"{name} vs oracle")


@pytest.mark.parametrize("name", SCHEMES)
@pytest.mark.parametrize("algo", [KS_64, KS_INT])
@pytest.mark.parametrize("layout", ["identity first", "identity middle", "no identity", "repeated", "count 1", "count 1 identity",
                                    "count 8"])
def test_diagonal_sum_matrix(name, algo, layout):
    """identity element first, in the middle or absent, a repeated element, count 1, 2 and 8, shared and per-member plaintexts mixed,
    plaintexts in the scheme's usual form, against the chain and the oracle"""
    n, mods, t, ctx, oc = case(name, algo)
    L, B = 3, 3
    steps = {"identity first": [0, 1], "identity middle": [1, 0, -1], "no identity": [-1, n // 4 - 1], "repeated": [1, 0, 1],
             "count 1": [None], "count 1 identity": [0], "count 8": [0, 1, -1, 2, 3, n // 4 - 1, None, 0]}[layout]
    counts = [1 if i % 2 == 0 else B for i in range(len(steps))]
    rng = np.random.default_rng(seed_of(name, algo, layout))
    plain_ntt = default_ntt(name)
    elts, hkeys, keys, plains = terms(rng, n, mods, t, L, B, steps, counts, plain_ntt, ctx)
    x = rand_ct(rng, mods, n, 2, L, B)
    got = fused_diag(ctx, x, elts, keys, plains, plain_ntt)
    assert_words(got, chain_diag(ctx, name, x, elts, keys, plains, plain_ntt), f"{name} {layout} vs chain")
    if len(steps) <= 3:
        assert_words(got, oracle_diag(oc, name, L, x, elts, hkeys, plains, plain_ntt), f"{name} {layout} vs oracle")


@pytest.mark.parametrize("name", ["BFV", "BGV"])
@pytest.mark.parametrize("plain_ntt", [True, False])
def test_diagonal_sum_plaintext_forms(name, plain_ntt):
    """BFV and BGV with NTT-form and coefficient-form plaintexts (BGV's are transformed once, then take the fused path; BFV's
    NTT-form plaintexts multiply as the reference multiplies a coefficient-form ciphertext)"""
    n, mods, t, ctx, oc = case(name, KS_64)
    L, B = 3, 2
    rng = np.random.default_rng(400 + plain_ntt)
    elts, hkeys, keys, plains = terms(rng, n, mods, t, L, B, [1, 0, -1], [B, 1, 1], plain_ntt, ctx)
    x = rand_ct(rng, mods, n, 2, L, B)
    got = fused_diag(ctx, x, elts, keys, plains, plain_ntt)
    assert_words(got, chain_diag(ctx, name, x, elts, keys, plains, plain_ntt), f"{name} plain_ntt={plain_ntt} vs chain")
    assert_words(got, oracle_diag(oc, name, L, x, elts, hkeys, plains, plain_ntt), f"{name} plain_ntt={plain_ntt} vs oracle")


@pytest.mark.parametrize("name", ["CKKS", "BGV"])
@pytest.mark.parametrize("fusion", ["default", "no_fuse_ntt", "no_fuse_crt"])
def test_integer_path_exits(name, fusion, monkeypatch):
    """n = 8192 on the integer path: the exit fused into the 64-bit column passes (default), and the unfused exits"""
    for v in FUSE_SWITCHES:
        monkeypatch.delenv(v, raising=False)
    if fusion != "default":
        monkeypatch.setenv({"no_fuse_ntt": "SB200_KS_FUSE_NTT", "no_fuse_crt": "SB200_KS_FUSE_CRT"}[fusion], "0")
    n = 8192
    mods = O.coeff_modulus_create(n, [50, 40, 40, 40, 50])
    ctx, t = make(name, n, mods, KS_INT)
    L, B = 4, 2
    rng = np.random.default_rng(8192)
    elts, hkeys, keys, plains = terms(rng, n, mods, t, L, B, [0, 1, None], [1, B, 1], True, ctx)
    x, a = rand_ct(rng, mods, n, 2, L, B), rand_ct(rng, mods, n, 2, L, B)
    assert_words(fused_diag(ctx, x, elts, keys, plains, True), chain_diag(ctx, name, x, elts, keys, plains, True), f"{fusion} diagonal_sum")
    assert_words(fused_mpa(ctx, x, elts[1], keys[1], plains[1], a), chain_mpa(ctx, name, x, elts[1], keys[1], plains[1], a),
                 f"{fusion} apply_galois_multiply_plain_add")


@pytest.mark.parametrize("name", SCHEMES)
@pytest.mark.parametrize("algo", [KS_64, KS_INT])
def test_aliasing(name, algo):
    """addend = input, out = addend with four rotated terms accumulated into one destination, out = input rejected"""
    n, mods, t, ctx, oc = case(name, algo)
    L, B = 4, 2
    rng = np.random.default_rng(17 + algo)
    keys = {s: ctx.load_key(rand_key(rng, mods, n)) for s in (1, -1, 3, None)}
    x = rand_ct(rng, mods, n, 2, L, B)
    p = rand_plain(rng, mods, n, L, 1, t, True)
    d_x, d_p, out = dev(x), dev(p), dev(np.zeros_like(x))
    ctx.d_apply_galois_multiply_plain_add(d_x, elt_of(n, 1), keys[1], d_p, 1, d_x, out, L, B)
    sync()
    assert_words(host(out), chain_mpa(ctx, name, x, elt_of(n, 1), keys[1], p, x), "addend = input")
    cts = [rand_ct(rng, mods, n, 2, L, B) for _ in range(4)]
    ps = [rand_plain(rng, mods, n, L, B if i % 2 else 1, t, True) for i in range(4)]
    acc = rand_ct(rng, mods, n, 2, L, B)
    d_acc, want = dev(acc), acc.copy()
    for s, c, q in zip((1, -1, 3, None), cts, ps):
        ctx.d_apply_galois_multiply_plain_add(dev(c), elt_of(n, s), keys[s], dev(q), q.shape[0], d_acc, d_acc, L, B)
        want = chain_mpa(ctx, name, c, elt_of(n, s), keys[s], q, want)
    sync()
    assert_words(host(d_acc), want, "four rotated terms accumulated into one destination")
    before = host(d_x).copy()
    with pytest.raises(ValueError, match="must not alias"):
        ctx.d_apply_galois_multiply_plain_add(d_x, elt_of(n, 1), keys[1], d_p, 1, out, d_x, L, B)
    with pytest.raises(ValueError, match="must not alias"):
        ctx.d_diagonal_sum(d_x, [elt_of(n, 1)], [keys[1]], [d_p], [1], d_x, L, B)
    sync()
    assert_words(host(d_x), before, "input unchanged after the aliasing errors")


@pytest.mark.parametrize("name", SCHEMES)
@pytest.mark.parametrize("algo", [KS_64, KS_INT])
def test_chunks(name, algo):
    """several key-switching chunks with a ragged tail (LIMIT_KS_CHUNK), and host staging chunks with a ragged tail"""
    n, mods, t, _, _ = case(name, algo)
    ctx, _ = make(name, n, mods, algo)
    L, B = 4, 7
    rng = np.random.default_rng(31 + algo)
    plain_ntt = default_ntt(name)
    elts, hkeys, keys, plains = terms(rng, n, mods, t, L, B, [1, 0, 2, 4], [1, B, B, 1], plain_ntt, ctx)
    x, a = rand_ct(rng, mods, n, 2, L, B), rand_ct(rng, mods, n, 2, L, B)
    p1 = rand_plain(rng, mods, n, L, B, t, True)
    want_diag = chain_diag(ctx, name, x, elts, keys, plains, plain_ntt)
    want_mpa = chain_mpa(ctx, name, x, elts[0], keys[0], p1, a)
    ctx.set_limit(ctx.LIMIT_KS_CHUNK, 3)  # chunks of 3, 3, 1
    assert_words(fused_diag(ctx, x, elts, keys, plains, plain_ntt), want_diag, "diagonal_sum in key-switching chunks")
    assert_words(fused_mpa(ctx, x, elts[0], keys[0], p1, a), want_mpa, "apply_galois_multiply_plain_add in key-switching chunks")
    # staging chunks of 2, 2, 2, 1: per member the input, the output and the per-member plaintexts (and the addend)
    ctx.set_limit(ctx.LIMIT_HOST_STAGE_BYTES, 2 * 7 * L * n * 8)
    assert_words(ctx.apply_galois_multiply_plain_add(x, elts[0], keys[0], p1, a), want_mpa, "host staging chunks")
    ctx.set_limit(ctx.LIMIT_HOST_STAGE_BYTES, 2 * (4 * L * n + 2 * (L * n if plain_ntt else n)) * 8)
    assert_words(ctx.diagonal_sum(x, elts, keys, plains, plain_ntt), want_diag, "diagonal_sum in host staging chunks")


@pytest.mark.parametrize("bits", [60, 61])
@pytest.mark.parametrize("name", ["CKKS", "BGV"])
def test_worst_case_words(bits, name):
    """all-(q - 1) ciphertext, addend and key words, plaintext words up to 2^64 - 1 (the largest representative of each residue),
    at 60- and 61-bit primes: the epilogue reduces the plaintext on the way in and keeps every word canonical"""
    n = 4096
    mods = [int(q) for q in O.get_primes(2 * n, bits, 4)]
    ctx, t = make(name, n, mods)
    oc = O.Oracle(scheme_id(name), n, mods, t)
    L, B = 3, 2
    hkey = np.stack([max_ct(mods, n, 2, len(mods))] * (len(mods) - 1))
    key = ctx.load_key(hkey)
    x = max_ct(mods, n, 2, L, B)
    rng = np.random.default_rng(bits)
    reduced = [rand_plain(rng, mods, n, L, 1, t, True), max_ct(mods, n, 1, L)]
    for p in reduced:
        wide = unreduce(p, mods)
        assert (wide >= np.uint64(2 ** 63)).all()
        for step in (1, None):
            e = elt_of(n, step)
            got = fused_mpa(ctx, x, e, key, wide, x)
            assert_words(got, chain_mpa(ctx, name, x, e, key, wide, x), f"{bits}-bit vs chain")
            want = np.stack([oc.linear(0, L, x[b], oracle_term(oc, name, L, x[b], e, hkey, p[0], True)) for b in range(B)])
            assert_words(got, want, f"{bits}-bit vs oracle")
            assert all((got[:, :, i] < mods[i]).all() for i in range(L)), "canonical words"
        elts = [1, elt_of(n, 1), elt_of(n, -1)]
        keys = [None, key, key]
        got = fused_diag(ctx, x, elts, keys, [wide] * 3, True)
        assert_words(got, chain_diag(ctx, name, x, elts, keys, [wide] * 3, True), f"{bits}-bit diagonal_sum vs chain")


def test_large_n():
    """n = 65536, L = 31 (32 primes), three Galois keys: diagonal_sum with an identity term and three rotated terms, and one
    apply_galois_multiply_plain_add, against the chain"""
    n = 65536
    mods = O.coeff_modulus_create(n, [50] * 32)
    ctx, _ = make("CKKS", n, mods, 1)
    L, B = 31, 2
    rng = np.random.default_rng(65536)
    elts, hkeys, keys, plains = terms(rng, n, mods, 0, L, B, [0, 1, -1, 5], [1, B, 1, 1], True, ctx)
    x = rand_ct(rng, mods, n, 2, L, B)
    assert_words(fused_diag(ctx, x, elts, keys, plains, True), chain_diag(ctx, "CKKS", x, elts, keys, plains, True), "n=65536 diagonal_sum")
    a = rand_ct(rng, mods, n, 2, L, B)
    assert_words(fused_mpa(ctx, x, elts[1], keys[1], plains[1], a), chain_mpa(ctx, "CKKS", x, elts[1], keys[1], plains[1], a),
                 "n=65536 apply_galois_multiply_plain_add")


def test_fewer_launches_than_the_chain():
    """CKKS: one key switch per rotated term and one plain_sum pass, against the chain's extra product and add launches"""
    n, mods, t, ctx, _ = case("CKKS", KS_64)
    L, B = 4, 2
    rng = np.random.default_rng(3)
    elts, _, keys, plains = terms(rng, n, mods, t, L, B, [0, 1, -1, 2], [1, 1, B, 1], True, ctx)
    x = rand_ct(rng, mods, n, 2, L, B)
    d_x, out = dev(x), dev(np.zeros_like(x))
    d_p = [dev(p) for p in plains]
    sync()
    l0 = ctx.launch_count
    ctx.d_diagonal_sum(d_x, elts, keys, d_p, [p.shape[0] for p in plains], out, L, B)
    fused = ctx.launch_count - l0
    l0 = ctx.launch_count
    chain_diag(ctx, "CKKS", x, elts, keys, plains, True)
    chained = ctx.launch_count - l0
    assert fused < chained, (fused, chained)


def test_errors_leave_outputs_unchanged():
    """every check runs before the first launch, in the chain's order: level, element, key (context, digits), plaintext count,
    coefficient-form plaintexts in CKKS, count 0, NULL pointers, aliasing and overlap"""
    n, mods, t, ctx, _ = case("CKKS", KS_64)
    L, B = len(mods) - 1, 2
    rng = np.random.default_rng(5)
    key = ctx.load_key(rand_key(rng, mods, n))
    short = ctx.load_key(rand_key(rng, mods, n)[:2])  # 2 digits: too few at L = 5
    other, _ = make("CKKS", n, mods)
    foreign = other.load_key(rand_key(rng, mods, n))
    x = rand_ct(rng, mods, n, 2, L, B)
    p = rand_plain(rng, mods, n, L, 1, t, True)
    d_x, d_p, d_o, d_pc = dev(x), dev(p), dev(np.zeros_like(x)), dev(np.zeros((B, n), dtype=np.uint64))
    before = host(d_o).copy()
    e1 = elt_of(n, 1)

    def mpa(elt=e1, k=key, pc=1, plain=d_p, addend=d_x, out=d_o, level=L):
        ctx.d_apply_galois_multiply_plain_add(d_x, elt, k, plain, pc, addend, out, level, B)

    def diag(elts=(1, e1), keys=(None, key), plains=(d_p, d_p), counts=(1, 1), out=d_o, level=L, ntt=True):
        ctx.d_diagonal_sum(d_x, list(elts), list(keys), list(plains), list(counts), out, level, B, ntt)

    bad = [
        (lambda: mpa(elt=2), ValueError, "Galois element is not valid"),
        (lambda: mpa(elt=2 * n + 1), ValueError, "Galois element is not valid"),
        (lambda: mpa(k=short), ValueError, "inner dimension is too small"),
        (lambda: mpa(k=foreign), ValueError, "parameter mismatch"),
        (lambda: mpa(level=len(mods) + 1), None, None),
        (lambda: mpa(pc=3), ValueError, "plain_count must be 1 or batch"),
        (lambda: mpa(elt=2, pc=3), ValueError, "Galois element is not valid"),  # apply_galois's checks come first
        (lambda: mpa(k=None), ValueError, "null pointer"),
        (lambda: mpa(plain=None), ValueError, "null pointer"),
        (lambda: mpa(addend=None), ValueError, "null pointer"),
        (lambda: mpa(plain=d_o), ValueError, "must not"),
        (lambda: diag(elts=(1, 2)), ValueError, "Galois element is not valid"),
        (lambda: diag(keys=(None, short)), ValueError, "inner dimension is too small"),
        (lambda: diag(keys=(None, None)), ValueError, "null pointer"),
        (lambda: diag(counts=(1, 3)), ValueError, "plain_count must be 1 or batch"),
        (lambda: diag(elts=(2, e1), keys=(key, key), counts=(1, 3)), ValueError, "Galois element is not valid"),
        (lambda: diag(plains=(d_pc, d_pc), ntt=False), ValueError, "unsupported operation for scheme type"),
        (lambda: diag(elts=(), keys=(), plains=(), counts=()), ValueError, "cannot be empty"),
        (lambda: diag(plains=(d_p, None)), ValueError, "null pointer"),
        (lambda: diag(plains=(d_p, d_o)), ValueError, "must not"),
        (lambda: diag(level=0), None, None),
    ]
    for f, exc, msg in bad:
        with pytest.raises(exc or Exception, match=msg):
            f()
        sync()
        assert_words(host(d_o), before, f"output unchanged after {msg}")
    with pytest.raises(Exception):
        ctx.diagonal_sum(x, [e1, 4], [key, key], [p, p])
    with pytest.raises(Exception):
        ctx.apply_galois_multiply_plain_add(x, e1, short, p, x)


@pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsealref.so not present")
@pytest.mark.parametrize("name", SCHEMES)
def test_against_reference(name):
    """the reference's own rotate / multiply_plain / add_inplace chain on ciphertexts, with its Galois keys"""
    n = 4096
    scheme = scheme_id(name)
    mods = R.coeff_modulus_create(n, [50, 40, 40, 50])
    t = 0 if name == "CKKS" else int(R.plain_modulus_batching(n, 20))
    rc = R.RefContext(scheme, n, mods, t)
    ctx = sb().Context(scheme, n, mods, t)
    L, B = len(mods) - 1, 2
    rng = np.random.default_rng(77)
    steps = [0, 1, -1, 4]
    elts = [1 if s == 0 else rc.galois_elt_from_step(s) for s in steps]
    keys = [None if e == 1 else ctx.load_key(rc.galois_key(e)) for e in elts]
    plain_ntt = name != "BFV"
    plains = [rand_plain(rng, mods, n, L, 1 if i % 2 else B, t, plain_ntt) for i in range(len(steps))]
    x, a = rand_ct(rng, mods, n, 2, L, B), rand_ct(rng, mods, n, 2, L, B)
    got = ctx.diagonal_sum(x, elts, keys, plains, plain_ntt)

    def ref_mul(ct, p):
        # BFV: multiply_plain_normal of a coefficient-form plaintext; CKKS / BGV: the NTT-form product
        return rc.plain_op_coeff(0, L, ct, p, ct_is_ntt=False) if name == "BFV" else rc.multiply_plain(L, ct, p)

    for b in range(B):
        acc = None
        for s, p in zip(steps, plains):
            term = x[b] if s == 0 else rc.rotate(L, x[b], s)
            term = ref_mul(term, p[0] if p.shape[0] == 1 else p[b])
            acc = term if acc is None else rc.linear(0, L, acc, term)
        assert_words(got[b], acc, f"diagonal_sum member {b}")
    if name != "BFV":
        p = rand_plain(rng, mods, n, L, 1, t, True)
        one = ctx.apply_galois_multiply_plain_add(x, elts[1], keys[1], p, a)
        for b in range(B):
            assert_words(one[b], rc.linear(0, L, a[b], rc.multiply_plain(L, rc.rotate(L, x[b], 1), p[0])),
                         f"apply_galois_multiply_plain_add member {b}")


@pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsealref.so not present")
def test_ckks_matrix_times_vector_decodes():
    """an 8 x 8 matrix times a vector on CKKS slots (the vector repeated across every slot): decrypted and decoded by the reference,
    every slot j holds (M v)[j mod 8] within the encoding's tolerance"""
    n, d = 4096, 8
    mods = R.coeff_modulus_create(n, [60, 40, 40, 60])
    rc = R.RefContext(R.CKKS, n, mods)
    ctx = sb().Context(sb().CKKS, n, mods)
    L, scale = len(mods) - 1, 2.0 ** 40
    rng = np.random.default_rng(8)
    M, v = rng.uniform(-1, 1, (d, d)), rng.uniform(-1, 1, d)
    slots = n // 2
    j = np.arange(slots)
    ct = rc.encrypt_zero_symmetric(L)
    pv = rc.ckks_encode(L, v[j % d].astype(np.complex128), scale)
    ct[0] = np.stack([(ct[0][i].astype(object) + pv[i].astype(object)) % mods[i] for i in range(L)]).astype(np.uint64)
    elts = [1 if i == 0 else rc.galois_elt_from_step(i) for i in range(d)]
    keys = [None if e == 1 else ctx.load_key(rc.galois_key(e)) for e in elts]
    diags = [rc.ckks_encode(L, M[j % d, (j + i) % d].astype(np.complex128), scale)[None] for i in range(d)]
    y = ctx.diagonal_sum(ct, elts, keys, diags)
    got = rc.ckks_decode(L, rc.decrypt(L, y, True), scale * scale).real
    want = (M @ v)[j % d]
    assert np.abs(got - want).max() < 1e-3, np.abs(got - want).max()


@pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsealref.so not present")
def test_bfv_matrix_times_vector_decrypts_exactly():
    """an 8 x 8 matrix times a vector mod t on BFV slots (each row of the slot matrix holds the vector repeated): decrypted by the
    reference, every slot j holds (M v)[j mod 8] mod t exactly"""
    n, d = 4096, 8
    mods = R.coeff_modulus_create(n, [50, 40, 40, 50])
    t = int(R.plain_modulus_batching(n, 20))
    rc = R.RefContext(R.BFV, n, mods, t)
    ctx = sb().Context(sb().BFV, n, mods, t)
    L = len(mods) - 1
    rng = np.random.default_rng(9)
    M, v = rng.integers(0, t, (d, d)), rng.integers(0, t, d)
    j = np.arange(n) % (n // 2)  # the slot's column within its row
    ct = rc.bfv_encrypt(v[j % d].astype(np.uint64))
    elts = [1 if i == 0 else rc.galois_elt_from_step(i) for i in range(d)]
    keys = [None if e == 1 else ctx.load_key(rc.galois_key(e)) for e in elts]
    diags = [rc.batch_codec(M[j % d, (j + i) % d].astype(np.uint64), False)[None] for i in range(d)]
    y = ctx.diagonal_sum(ct, elts, keys, diags, plain_is_ntt=False)
    dec, budget = rc.bfv_decrypt(L, y)
    assert budget > 0
    want = np.array([int(sum(int(M[r, c]) * int(v[c]) for c in range(d)) % t) for r in range(d)], dtype=np.uint64)[j % d]
    assert_words(dec, want, "decrypted M v mod t")


def test_cpp_diagonal_sum_against_seal_evaluator():
    """tests/cpp/shim_diagsum_test.cpp: Evaluator::apply_galois_multiply_plain_add_inplace and diagonal_sum against seal::Evaluator's
    chains -- words, metadata, exception types and messages, the NAF fallback, a one-byte key cache and DeviceGaloisKeys"""
    exe = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref", "bin", "shim_diagsum_test")
    if not os.path.exists(exe):
        pytest.skip("shim_diagsum_test not built (reference sources absent at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert "shim_diagsum_test ok" in r.stdout
