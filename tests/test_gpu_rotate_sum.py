"""Sums of rotations: sb200_apply_galois_add (out = addend + apply_galois(in)) and sb200_rotate_sum (y_{j+1} = y_j +
apply_galois(y_j, elt_j)), both entry points, word for word against the chained device calls (sb200_apply_galois, then a
two-operand sb200_add_many), against the plain-C oracle (tests/oracle.py: apply_galois + linear) and against the reference's own
rotate / apply_galois + add (oracle/_ref); a BFV slot sum decrypted by the reference; and the C++ members
(tests/cpp/shim_rotsum_test.cpp) against seal::Evaluator."""
import os
import subprocess

import numpy as np
import pytest

import oracle as O
import refseal as R
from common import assert_words, max_ct, rand_ct

pytestmark = pytest.mark.gpu

KS_64, KS_INT = 0, 2  # SB200_LIMIT_KS_ALGORITHM
SCHEMES = ("CKKS", "BFV", "BGV")


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
    return 2 * n - 1 if step is None else O.galois_elt_from_step(n, step)


def chain_add(ctx, x, elt, key, addend):
    """the chained device calls: apply_galois into a temporary, then a two-operand add_many"""
    B, _, L, n = x.shape
    d_x, d_a = dev(x), dev(addend)
    t, out = dev(np.zeros_like(x)), dev(np.zeros_like(x))
    ctx.d_apply_galois(d_x, elt, key, t, L, B)
    ctx.d_add_many([d_a, t], out, L, B, [2, 2])
    sync()
    return host(out)


def chain_sum(ctx, x, elts, keys):
    y = x.copy()
    for e, k in zip(elts, keys):
        y = chain_add(ctx, y, e, k, y)
    return y


def fused_add(ctx, x, elt, key, addend):
    """the stream entry point (out a fresh slab, then accumulate into the addend) and the host form; all equal, inputs unchanged"""
    B, _, L, n = x.shape
    d_x, d_a, out = dev(x), dev(addend), dev(np.zeros_like(x))
    ctx.d_apply_galois_add(d_x, elt, key, d_a, out, L, B)
    ctx.d_apply_galois_add(d_x, elt, key, d_a, d_a, L, B)  # out = addend: accumulate
    sync()
    got = host(out)
    assert_words(host(d_a), got, "accumulated into the addend vs a fresh output")
    assert_words(host(d_x), x, "input unchanged")
    assert_words(ctx.apply_galois_add(x, elt, key, addend), got, "host form vs stream form")
    return got


def oracle_add(oc, L, x, elt, hkey, addend):
    return np.stack([oc.linear(0, L, addend[b], oc.apply_galois(L, x[b], elt, hkey)) for b in range(x.shape[0])])


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


@pytest.mark.parametrize("name", SCHEMES)
@pytest.mark.parametrize("algo", [KS_64, KS_INT])
@pytest.mark.parametrize("level", ["top", "middle", "last"])
@pytest.mark.parametrize("step", [1, -1, 3, "n/4-1", None])
def test_apply_galois_add_matrix(name, algo, level, step):
    """every scheme, both key-switching paths, three levels, steps 1, -1, 3, n/4 - 1 and the element 2n - 1, against the chain and
    the oracle"""
    n, mods, t, ctx, oc = case(name, algo)
    L = {"top": len(mods) - 1, "middle": 3, "last": 1}[level]
    s = n // 4 - 1 if step == "n/4-1" else step
    elt = elt_of(n, s)
    rng = np.random.default_rng(hash((name, algo, level, str(step))) & 0xFFFF)
    hkey = rand_key(rng, mods, n)
    key = ctx.load_key(hkey)
    B = 3
    x, a = rand_ct(rng, mods, n, 2, L, B), rand_ct(rng, mods, n, 2, L, B)
    got = fused_add(ctx, x, elt, key, a)
    assert_words(got, chain_add(ctx, x, elt, key, a), f"{name} L={L} vs chain")
    assert_words(got, oracle_add(oc, L, x, elt, hkey, a), f"{name} L={L} vs oracle")


@pytest.mark.parametrize("name", SCHEMES)
@pytest.mark.parametrize("algo", [KS_64, KS_INT])
def test_aliasing(name, algo):
    """addend = input (y + rotate(y)), out = addend with K = 4 rotated terms accumulated into one destination, out = input rejected"""
    n, mods, t, ctx, oc = case(name, algo)
    L, B = len(mods) - 1, 2
    rng = np.random.default_rng(17 + algo)
    keys = {s: ctx.load_key(rand_key(rng, mods, n)) for s in (1, -1, 3, None)}
    x = rand_ct(rng, mods, n, 2, L, B)
    d_x, out = dev(x), dev(np.zeros_like(x))
    ctx.d_apply_galois_add(d_x, elt_of(n, 1), keys[1], d_x, out, L, B)
    sync()
    assert_words(host(out), chain_add(ctx, x, elt_of(n, 1), keys[1], x), "addend = input")
    terms = [rand_ct(rng, mods, n, 2, L, B) for _ in range(4)]
    acc = rand_ct(rng, mods, n, 2, L, B)
    d_acc, want = dev(acc), acc.copy()
    for s, c in zip((1, -1, 3, None), terms):
        ctx.d_apply_galois_add(dev(c), elt_of(n, s), keys[s], d_acc, d_acc, L, B)
        want = chain_add(ctx, c, elt_of(n, s), keys[s], want)
    sync()
    assert_words(host(d_acc), want, "four rotated terms accumulated into one destination")
    before = host(d_x).copy()
    with pytest.raises(ValueError, match="must not alias"):
        ctx.d_apply_galois_add(d_x, elt_of(n, 1), keys[1], out, d_x, L, B)
    sync()
    assert_words(host(d_x), before, "output unchanged after the aliasing error")


@pytest.mark.parametrize("name", SCHEMES)
@pytest.mark.parametrize("algo", [KS_64, KS_INT])
def test_chunks(name, algo):
    """several key-switching chunks with a ragged tail (LIMIT_KS_CHUNK), and host staging chunks with a ragged tail"""
    n, mods, t, _, _ = case(name, algo)
    ctx, _ = make(name, n, mods, algo)
    L, B = len(mods) - 1, 7
    rng = np.random.default_rng(31 + algo)
    keys = [ctx.load_key(rand_key(rng, mods, n)) for _ in range(3)]
    elts = [elt_of(n, s) for s in (1, 2, 4)]
    x, a = rand_ct(rng, mods, n, 2, L, B), rand_ct(rng, mods, n, 2, L, B)
    want_add = chain_add(ctx, x, elts[0], keys[0], a)
    want_sum = chain_sum(ctx, x, elts, keys)
    ctx.set_limit(ctx.LIMIT_KS_CHUNK, 3)  # chunks of 3, 3, 1
    assert_words(fused_add(ctx, x, elts[0], keys[0], a), want_add, "apply_galois_add in key-switching chunks")
    d = dev(x)
    ctx.d_rotate_sum(d, elts, keys, d, L, B)
    sync()
    assert_words(host(d), want_sum, "rotate_sum in key-switching chunks, in place")
    ctx.set_limit(ctx.LIMIT_HOST_STAGE_BYTES, 2 * 3 * 2 * L * n * 8)  # staging chunks of 2, 2, 2, 1 (apply_galois_add: 3 slabs)
    assert_words(ctx.apply_galois_add(x, elts[0], keys[0], a), want_add, "apply_galois_add in host staging chunks")
    assert_words(ctx.rotate_sum(x, elts, keys), want_sum, "rotate_sum in host staging chunks")


@pytest.mark.parametrize("bits", [60, 61])
@pytest.mark.parametrize("name", SCHEMES)
def test_worst_case_words(bits, name):
    """every input, addend and key word q - 1 at 60- and 61-bit primes: the epilogue's two csubs keep every word canonical"""
    n = 4096
    mods = [int(q) for q in O.get_primes(2 * n, bits, 4)]
    ctx, t = make(name, n, mods)
    oc = O.Oracle(scheme_id(name), n, mods, t)
    L, B = 3, 2
    hkey = np.stack([max_ct(mods, n, 2, len(mods))] * (len(mods) - 1))
    key = ctx.load_key(hkey)
    x = max_ct(mods, n, 2, L, B)
    for step in (1, None):
        got = fused_add(ctx, x, elt_of(n, step), key, x)
        assert_words(got, chain_add(ctx, x, elt_of(n, step), key, x), f"{bits}-bit all q - 1 vs chain")
        assert_words(got, oracle_add(oc, L, x, elt_of(n, step), hkey, x), f"{bits}-bit all q - 1 vs oracle")
        assert all((got[:, :, i] < mods[i]).all() for i in range(L)), "canonical words"


def test_large_n():
    """n = 65536, L = 31 (32 primes): apply_galois_add and a two-step rotate_sum against the chain"""
    n = 65536
    mods = O.coeff_modulus_create(n, [50] * 32)
    ctx, _ = make("CKKS", n, mods, 1)
    L = 31
    rng = np.random.default_rng(65536)
    keys = [ctx.load_key(rand_key(rng, mods, n)) for _ in range(2)]
    elts = [elt_of(n, 1), elt_of(n, 2)]
    x, a = rand_ct(rng, mods, n, 2, L, 1), rand_ct(rng, mods, n, 2, L, 1)
    assert_words(fused_add(ctx, x, elts[0], keys[0], a), chain_add(ctx, x, elts[0], keys[0], a), "n=65536 apply_galois_add")
    d, out = dev(x), dev(np.zeros_like(x))
    ctx.d_rotate_sum(d, elts, keys, out, L, 1)
    sync()
    assert_words(host(out), chain_sum(ctx, x, elts, keys), "n=65536 rotate_sum")


@pytest.mark.parametrize("name", SCHEMES)
@pytest.mark.parametrize("count", [1, 2, 8, "row"])
def test_rotate_sum_counts(name, count):
    """rotate_sum with the elements of steps 1, 2, 4, ... for count in {1, 2, 8, a full row}, out = in and out != in, against the
    chain of apply_galois + add"""
    n, mods, t, ctx, oc = case(name, KS_64)
    count = n // 2 if count == "row" else count
    steps = [1 << j for j in range(count.bit_length() - 1)]
    L, B = 2, 2
    rng = np.random.default_rng(900 + count)
    hkeys = [rand_key(rng, mods, n) for _ in steps]
    keys = [ctx.load_key(h) for h in hkeys]
    elts = [elt_of(n, s) for s in steps]
    x = rand_ct(rng, mods, n, 2, L, B)
    want = chain_sum(ctx, x, elts, keys)
    if len(steps) <= 3:
        y = x.copy()
        for e, h in zip(elts, hkeys):
            y = oracle_add(oc, L, y, e, h, y)
        assert_words(want, y, "chain vs oracle")
    assert_words(ctx.rotate_sum(x, elts, keys), want, "host form")
    d, out = dev(x), dev(np.zeros_like(x))
    ctx.d_rotate_sum(d, elts, keys, out, L, B)
    ctx.d_rotate_sum(d, elts, keys, d, L, B)  # in place
    sync()
    assert_words(host(out), want, "stream form, out != in")
    assert_words(host(d), want, "stream form, in place")


def test_errors_leave_outputs_unchanged():
    """every check runs before the first launch: level, element, key (context, digits), NULL pointers, aliasing"""
    n, mods, t, ctx, _ = case("CKKS", KS_64)
    L, B = len(mods) - 1, 2
    rng = np.random.default_rng(5)
    key = ctx.load_key(rand_key(rng, mods, n))
    short = ctx.load_key(rand_key(rng, mods, n)[:2])  # 2 digits: too few at L = 5
    other, _ = make("CKKS", n, mods)
    foreign = other.load_key(rand_key(rng, mods, n))
    x = rand_ct(rng, mods, n, 2, L, B)
    d_x, d_o = dev(x), dev(np.zeros_like(x))
    before = host(d_o).copy()
    e1 = elt_of(n, 1)
    bad = [
        (lambda: ctx.d_apply_galois_add(d_x, 2, key, d_x, d_o, L, B), ValueError, "Galois element is not valid"),
        (lambda: ctx.d_apply_galois_add(d_x, 2 * n + 1, key, d_x, d_o, L, B), ValueError, "Galois element is not valid"),
        (lambda: ctx.d_apply_galois_add(d_x, e1, short, d_x, d_o, L, B), ValueError, "inner dimension is too small"),
        (lambda: ctx.d_apply_galois_add(d_x, e1, foreign, d_x, d_o, L, B), ValueError, "parameter mismatch"),
        (lambda: ctx.d_apply_galois_add(d_x, e1, key, d_x, d_o, len(mods) + 1, B), None, None),
        (lambda: ctx.d_apply_galois_add(d_x, e1, None, d_x, d_o, L, B), ValueError, "null pointer"),
        (lambda: ctx.d_apply_galois_add(d_x, e1, key, None, d_o, L, B), ValueError, "null pointer"),
        (lambda: ctx.d_rotate_sum(d_x, [e1, 2], [key, key], d_o, L, B), ValueError, "Galois element is not valid"),
        (lambda: ctx.d_rotate_sum(d_x, [e1, e1], [key, short], d_o, L, B), ValueError, "inner dimension is too small"),
        (lambda: ctx.d_rotate_sum(d_x, [e1, e1], [key, None], d_o, L, B), ValueError, "null pointer"),
        (lambda: ctx.d_rotate_sum(d_x, [e1], [key], d_o, 0, B), None, None),
    ]
    for f, exc, msg in bad:
        with pytest.raises(exc or Exception, match=msg):
            f()
        sync()
        assert_words(host(d_o), before, f"output unchanged after {msg}")
    with pytest.raises(Exception):
        ctx.rotate_sum(x, [e1, 4], [key, key])
    with pytest.raises(Exception):
        ctx.apply_galois_add(x, e1, short, x)
    d = dev(x)
    ctx.d_rotate_sum(d, [], [], d_o, L, B)  # steps = 0 copies
    sync()
    assert_words(host(d_o), x, "steps = 0 copies the input")


@pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsealref.so not present")
@pytest.mark.parametrize("name", SCHEMES)
def test_against_reference(name):
    """the reference's own apply_galois / rotate + add on ciphertexts it encrypted, with its Galois keys"""
    n = 4096
    scheme = scheme_id(name)
    mods = R.coeff_modulus_create(n, [50, 40, 40, 50])
    t = 0 if name == "CKKS" else int(R.plain_modulus_batching(n, 20))
    rc = R.RefContext(scheme, n, mods, t)
    ctx = sb().Context(scheme, n, mods, t)
    L, B = len(mods) - 1, 2
    rng = np.random.default_rng(77)
    steps = [1, 2, 4]
    elts = [rc.galois_elt_from_step(s) for s in steps]
    keys = [ctx.load_key(rc.galois_key(e)) for e in elts]
    x, a = rand_ct(rng, mods, n, 2, L, B), rand_ct(rng, mods, n, 2, L, B)
    got = ctx.apply_galois_add(x, elts[0], keys[0], a)
    sums = ctx.rotate_sum(x, elts, keys)
    for b in range(B):
        assert_words(got[b], rc.linear(0, L, a[b], rc.apply_galois(L, x[b], elts[0])), f"apply_galois_add member {b}")
        y = x[b]
        for s in steps:
            y = rc.linear(0, L, y, rc.rotate(L, y, s))
        assert_words(sums[b], y, f"rotate_sum member {b}")


@pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsealref.so not present")
def test_bfv_slot_sum_decrypts_to_the_total():
    """encrypt random BFV slots with the reference, sum every slot (rotate_sum over a row, then the column swap added), decrypt:
    every slot holds the total mod t"""
    n = 4096
    mods = R.coeff_modulus_create(n, [50, 40, 40, 50])
    t = int(R.plain_modulus_batching(n, 20))
    rc = R.RefContext(R.BFV, n, mods, t)
    ctx = sb().Context(sb().BFV, n, mods, t)
    L = len(mods) - 1
    rng = np.random.default_rng(4096)
    slots = rng.integers(0, t, n, dtype=np.uint64)
    ct = rc.bfv_encrypt(slots)
    steps = [1 << j for j in range((n // 2).bit_length() - 1)]
    elts = [rc.galois_elt_from_step(s) for s in steps]
    keys = [ctx.load_key(rc.galois_key(e)) for e in elts]
    y = ctx.rotate_sum(ct, elts, keys)
    y = ctx.apply_galois_add(y, 2 * n - 1, ctx.load_key(rc.galois_key(2 * n - 1)), y)
    dec, budget = rc.bfv_decrypt(L, y)
    assert budget > 0
    total = int(sum(int(v) for v in slots) % t)
    assert (dec == total).all(), f"slots {dec[:4]} vs total {total}"


def test_cpp_rotate_sum_against_seal_evaluator():
    """tests/cpp/shim_rotsum_test.cpp: Evaluator::apply_galois_add_inplace and rotate_sum_inplace against seal::Evaluator's chains --
    words, metadata, exception types and messages, the NAF fallback, a small key cache and DeviceGaloisKeys"""
    exe = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref", "bin", "shim_rotsum_test")
    if not os.path.exists(exe):
        pytest.skip("shim_rotsum_test not built (reference sources absent at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert "shim_rotsum_test ok" in r.stdout
