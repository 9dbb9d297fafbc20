"""Key generation on an H100 (-m gpu; seal_b200/csrc/sb_prng.cu: op_generate_public_key / op_generate_kswitch_key): public,
relinearization and Galois keys from a given secret key, word for word against the reference's KeyGenerator under seeded
Blake2xb / Shake256 factories (oracle/ref_keygen.cpp) and against the restatement of tests/keygen_ref.py; device handles against
uploaded words in both key-switching modes; fresh entropy through complete BFV / CKKS computations; chunking; the errors; and
the C++ stand-in seal_b200::KeyGenerator (tests/cpp/shim_keygen_test.cpp)."""
import os
import subprocess

import numpy as np
import pytest

import keygen_ref as K
import oracle as O
import refprng as P
import refseal as R

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not (K.ref_available() and P.ref_available()),
                               reason="oracle/_ref/libsealref_{keygen,prng}.so not present")


def sb():
    import seal_b200

    return seal_b200


def to_np(x):
    return x.cpu().numpy().view(np.uint64)


def make(scheme, n, bits, prng=P.BLAKE2XB, seed=0x6B67):
    S = sb()
    mods = R.coeff_modulus_create(n, bits)
    t = R.plain_modulus_batching(n, 20) if scheme != O.CKKS else 0
    rk = K.RefKeygen(scheme, n, mods, t, seed=seed, prng=prng)
    ctx = S.Context(scheme, n, mods, t)
    sk = rk.secret_key()
    return rk, ctx, ctx.load_secret_key(sk), sk, mods, t


SHAPES = [(O.CKKS, 1024, [60, 60]), (O.BFV, 4096, [36, 36, 37]), (O.BGV, 8192, [60] * 5), (O.CKKS, 16384, [30] * 17),
          (O.BFV, 32768, [60, 60, 60])]


@needs_ref
@pytest.mark.parametrize("prng", [P.BLAKE2XB, P.SHAKE256])
@pytest.mark.parametrize("scheme,n,bits", SHAPES)
def test_keys_vs_reference(scheme, n, bits, prng):
    """public key, relinearization key and Galois keys of a positive step, a negative step and the column / conjugate element,
    host words and the words behind the device handle, against the reference's KeyGenerator"""
    rk, ctx, skd, sk, mods, t = make(scheme, n, bits, prng)
    seeds = rk.boot_seeds(rk.k - 1)
    words, pkh = ctx.generate_public_key(skd, seeds[0], bootstrap_prng=prng)
    assert pkh is not None and (words == rk.public_key()).all()
    for elt in (0, ctx.galois_elt_from_step(1), ctx.galois_elt_from_step(-3), 2 * n - 1):
        words, _ = ctx.generate_kswitch_key(skd, elt, seeds, bootstrap_prng=prng, device=False)
        assert (words == rk.kswitch_key(elt)).all(), f"galois_elt {elt}"


@needs_ref
@pytest.mark.parametrize("scheme", [O.BFV, O.CKKS, O.BGV])
def test_ciphertext_prng_shake256_vs_restatement(scheme):
    """ciphertext_prng = 2 (c_1 expanded with SHAKE256, a reference built with SEAL_DEFAULT_PRNG Shake256): against the
    restatement, whose blake2xb arm the CPU tests hold to the reference"""
    n, bits = 1024, [40, 40, 50]
    rk, ctx, skd, sk, mods, t = make(scheme, n, bits, P.SHAKE256)
    ko = K.KeygenOracle(scheme, n, mods, t)
    seeds = np.arange(8 * (rk.k - 1), dtype=np.uint64).reshape(rk.k - 1, 8) * np.uint64(0x9E3779B97F4A7C15)
    for boot in (P.BLAKE2XB, P.SHAKE256):
        pk, _ = ctx.generate_public_key(skd, seeds[1], bootstrap_prng=boot, ciphertext_prng=P.SHAKE256, device=False)
        assert (pk == ko.public_key(sk, seeds[1], boot, P.SHAKE256)).all()
        for elt in (0, 2 * n - 1):
            words, _ = ctx.generate_kswitch_key(skd, elt, seeds, bootstrap_prng=boot, ciphertext_prng=P.SHAKE256, device=False)
            assert (words == ko.kswitch_key(sk, elt, seeds, boot, P.SHAKE256)).all()


@needs_ref
def test_relin_key_headline_shape():
    """the relinearization key at n = 65536, k = 32 (31 digits, about 1 GB of words) against the reference"""
    rk, ctx, skd, sk, mods, t = make(O.CKKS, 65536, [30] * 32)
    words, h = ctx.generate_kswitch_key(skd, 0, rk.boot_seeds(31))
    assert h is not None and (words == rk.kswitch_key(0)).all()


@pytest.mark.parametrize("algo", [0, 2])
def test_handles_equal_uploaded_words(algo):
    """relinearize, multiply_relinearize and apply_galois of a batch of 16 (the tensor-core product kernel's minimum) give the
    same words with the generated handle as with sb200_kswitch_key_create of the generated host words, in both key-switching
    modes"""
    S = sb()
    n = 4096
    mods = O.coeff_modulus_create(n, [30] * 8)
    k, L, B = len(mods), len(mods) - 1, 16
    ctx = S.Context(S.CKKS, n, mods)
    ctx.set_limit(ctx.LIMIT_KS_ALGORITHM, algo)
    rng = np.random.default_rng(algo + 11)
    sk = np.stack([rng.integers(0, q, n, dtype=np.uint64) for q in mods])
    skd = ctx.load_secret_key(sk)
    rw, rh = ctx.generate_kswitch_key(skd, 0)
    elt = ctx.galois_elt_from_step(5)
    gw, gh = ctx.generate_kswitch_key(skd, elt)
    ru, gu = ctx.load_key(rw), ctx.load_key(gw)

    def rnd(size):
        return np.stack([np.stack([np.stack([rng.integers(0, mods[i], n, dtype=np.uint64) for i in range(L)])
                                   for _ in range(size)]) for _ in range(B)])

    a, b, c3 = rnd(2), rnd(2), rnd(3)
    assert (ctx.relinearize(c3, rh) == ctx.relinearize(c3, ru)).all()
    assert (ctx.multiply_relinearize(a, b, rh) == ctx.multiply_relinearize(a, b, ru)).all()
    assert (ctx.apply_galois(a, elt, gh) == ctx.apply_galois(a, elt, gu)).all()


def _fresh(ctx, skd, L, B):
    import torch

    z = torch.zeros((B, 2, L, ctx.n), dtype=torch.int64, device="cuda")
    ctx.d_encrypt_zero_symmetric(skd, z, L, B)
    torch.cuda.synchronize()
    return to_np(z)


def test_fresh_entropy_bfv_multiply_relinearize_rotate():
    """seeds=None: two calls give different keys; BFV multiply + relinearize + rotate_rows with the generated keys decrypts to
    the expected slots"""
    S = sb()
    n = 8192
    mods = O.coeff_modulus_create(n, [50, 50, 50, 60])
    t = R.plain_modulus_batching(n, 20)
    ctx = S.Context(S.BFV, n, mods, t)
    rng = np.random.default_rng(7)
    # a ternary secret key in NTT form, as KeyGenerator samples it
    s = rng.integers(-1, 2, n)
    sk = ctx.transform_to_ntt(np.stack([np.where(s < 0, s + q, s).astype(np.uint64) for q in mods])[None])[0]
    skd = ctx.load_secret_key(sk)
    w1, rk = ctx.generate_kswitch_key(skd, 0)
    w2, _ = ctx.generate_kswitch_key(skd, 0, device=False)
    assert not (w1 == w2).all()
    _, gk = ctx.generate_kswitch_key(skd, ctx.galois_elt_from_step(1), host=False)
    L = len(mods) - 1
    a, b = rng.integers(0, t, n, dtype=np.uint64), rng.integers(0, t, n, dtype=np.uint64)
    ct = ctx.add_plain_coeff(_fresh(ctx, skd, L, 2), ctx.batch_encode(np.stack([a, b])))
    out = ctx.rotate(ctx.multiply_relinearize(ct[0], ct[1], rk), 1, gk)
    got = ctx.batch_decode(ctx.decrypt(out, skd)).reshape(2, n // 2)
    ab = ((a.astype(object) * b.astype(object)) % t).astype(np.uint64).reshape(2, n // 2)
    assert (got == np.roll(ab, -1, axis=1)).all()


def test_fresh_entropy_ckks_and_oracle_key_switching():
    """CKKS: multiply + relinearize + rescale + rotate with fresh generated keys decodes within the usual tolerance, and
    relinearizing with the generated handle equals the CPU oracle's key switching with the same key words"""
    S = sb()
    n, scale = 8192, 2.0 ** 40
    mods = O.coeff_modulus_create(n, [60, 40, 40, 60])
    L = len(mods) - 1
    ctx, oc = S.Context(S.CKKS, n, mods), O.Oracle(O.CKKS, n, mods)
    rng = np.random.default_rng(3)
    s = rng.integers(-1, 2, n)
    sk = ctx.transform_to_ntt(np.stack([np.where(s < 0, s + q, s).astype(np.uint64) for q in mods])[None])[0]
    skd = ctx.load_secret_key(sk)
    rw, rk = ctx.generate_kswitch_key(skd, 0)
    _, gk = ctx.generate_kswitch_key(skd, ctx.galois_elt_from_step(1), host=False)
    x, y = rng.uniform(-1, 1, n // 2), rng.uniform(-1, 1, n // 2)
    pt = ctx.ckks_encode(np.stack([x, y]), L, scale)
    ct = _fresh(ctx, skd, L, 2)
    q = np.array(mods[:L], dtype=np.uint64)[:, None]
    ct[:, 0] = ct[:, 0] + pt
    ct[:, 0] -= np.where(ct[:, 0] >= q, q, np.uint64(0))
    prod = ctx.multiply_relinearize(ct[0], ct[1], rk)
    assert (prod == oc.multiply_relin(L, ct[0], ct[1], rw)).all()
    out = ctx.rotate(ctx.rescale_to_next(prod), 1, gk)
    got = ctx.ckks_decode(ctx.decrypt(out, skd), scale * scale / mods[L - 1])
    assert np.abs(got.real - np.roll(x * y, -1)).max() < 1e-3


def test_chunked_digits_give_the_same_words():
    """a 1 MiB scratch budget cuts the 7 digits of n = 2048, k = 8 into chunks of 3, 3 and 1 (three bootstrap-stream launches):
    the words equal those of one chunk"""
    S = sb()
    n = 2048
    mods = O.coeff_modulus_create(n, [30] * 8)
    ctx = S.Context(S.BGV, n, mods, R.plain_modulus_batching(n, 20))
    rng = np.random.default_rng(5)
    skd = ctx.load_secret_key(np.stack([rng.integers(0, q, n, dtype=np.uint64) for q in mods]))
    seeds = rng.integers(0, 2 ** 63, (7, 8), dtype=np.uint64)
    for elt in (0, 2 * n - 1):
        whole, _ = ctx.generate_kswitch_key(skd, elt, seeds, device=False)
        ctx.set_limit(ctx.LIMIT_SCRATCH_BYTES, 1 << 20)
        ctx.profile(True)
        cut, h = ctx.generate_kswitch_key(skd, elt, seeds)
        launches = {name: cnt for name, _, cnt, _ in ctx.profile_read()}
        ctx.profile(False)
        ctx.set_limit(ctx.LIMIT_SCRATCH_BYTES, 8 << 30)
        assert launches.get("enc_bootstrap_stream") == 3 and launches.get("enc_combine:kswitch") == 3, launches
        assert (cut == whole).all()


def test_errors():
    S = sb()
    n = 1024
    mods = O.coeff_modulus_create(n, [40, 40, 40])
    ctx, other = S.Context(S.CKKS, n, mods), S.Context(S.CKKS, n, mods)
    rng = np.random.default_rng(1)
    sk = np.stack([rng.integers(0, q, n, dtype=np.uint64) for q in mods])
    skd, foreign = ctx.load_secret_key(sk), other.load_secret_key(sk)
    for elt in (2, 4, 2 * n, 2 * n + 1):
        with pytest.raises(ValueError, match="Galois element is not valid"):
            ctx.generate_kswitch_key(skd, elt)
    with pytest.raises(ValueError, match="secret key is not valid"):
        ctx.generate_kswitch_key(foreign, 0)
    with pytest.raises(ValueError, match="secret key is not valid"):
        ctx.generate_public_key(foreign)
    for bad in (0, 3):
        with pytest.raises(ValueError, match="prng_type"):
            ctx.generate_kswitch_key(skd, 0, bootstrap_prng=bad)
        with pytest.raises(ValueError, match="prng_type"):
            ctx.generate_kswitch_key(skd, 0, ciphertext_prng=bad)
        with pytest.raises(ValueError, match="prng_type"):
            ctx.generate_public_key(skd, bootstrap_prng=bad)
    with pytest.raises(ValueError, match="null pointer"):
        ctx.generate_kswitch_key(skd, 0, host=False, device=False)
    with pytest.raises(ValueError, match="null pointer"):
        ctx.generate_public_key(skd, host=False, device=False)
    # one prime: no key switching (the public key still exists)
    one = S.Context(S.CKKS, n, mods[:1])
    sk1 = one.load_secret_key(sk[:1].copy())
    with pytest.raises(RuntimeError, match="keyswitching is not supported by the context"):
        one.generate_kswitch_key(sk1, 0)
    pk, _ = one.generate_public_key(sk1)
    assert pk.shape == (2, 1, n)
    # the encryption entry points still reject the key level
    import torch

    z = torch.zeros((1, 2, 3, n), dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError, match="parms_id is not valid"):
        ctx.d_encrypt_zero_symmetric(skd, z, 3, 1)


SHIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref", "bin", "shim_keygen_test")


@pytest.mark.skipif(not os.path.exists(SHIM), reason="oracle/_ref/bin/shim_keygen_test not built (oracle/keygen.mk, needs the reference sources)")
def test_cpp_keygenerator_against_reference():
    """seal_b200::KeyGenerator against seal::KeyGenerator(context, secret_key) under both seeded factories and all three schemes:
    every create_* overload with a destination, the default Galois set, duplicates, the errors; words and save() bytes"""
    r = subprocess.run([SHIM], capture_output=True, text=True, timeout=900)
    print(r.stdout, r.stderr)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "PASS" in r.stdout
