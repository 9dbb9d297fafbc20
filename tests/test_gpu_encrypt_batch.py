"""Encryption of device-resident plaintexts on an H100 (-m gpu): sb200_encrypt_symmetric / sb200_encrypt_asymmetric
(seal_b200/csrc/sb_prng.cu).  The fused entry points must give the words of the composition they replace -- sb200_encrypt_zero_*_prng
followed by the evaluator's add_plain on c_0, each of which is checked against the reference elsewhere -- with the plaintext
term added inside the kernels that write c_0 (symmetric) or in one pass over the batch (public key), in chunks of the scratch
budget that do not change the words.  They must also give seal::Encryptor's words (oracle/ref_encrypt.cpp), and the C++
members on PlaintextBatch / CiphertextBatch must match the seal:: classes (tests/cpp/shim_encrypt_test.cpp)."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle as O

pytestmark = pytest.mark.gpu


def sb():
    import seal_b200

    return seal_b200


def to_np(x):
    return x.cpu().numpy().view(np.uint64)


def make(scheme, n, qbits, tbits=20):
    """context, secret key (uniform ternary, NTT form at the key level), public key made on the device, t, moduli"""
    import torch

    S = sb()
    allm = O.coeff_modulus_create(n, list(qbits) + ([tbits] if scheme != "ckks" else []))
    mods, t = (allm, 0) if scheme == "ckks" else (allm[:-1], int(allm[-1]))
    sid = {"ckks": S.CKKS, "bfv": S.BFV, "bgv": S.BGV}[scheme]
    ctx = S.Context(sid, n, mods, t)
    k = len(mods)
    rng = np.random.default_rng(0x5EC + n + k)
    tern = rng.integers(-1, 2, n)
    s = np.stack([np.where(tern < 0, np.uint64(int(q) - 1), tern.astype(np.uint64)) for q in mods]).astype(np.uint64)
    d = torch.from_numpy(s.view(np.int64).copy()).cuda()
    ctx.d_ntt_forward(d, k, 1, 1)
    torch.cuda.synchronize()
    sk = ctx.load_secret_key(to_np(d))
    _, pk = ctx.generate_public_key(sk, seed=np.arange(8, dtype=np.uint64) + np.uint64(77), host=False)
    return ctx, sk, pk, t, [int(q) for q in mods]


def first_level(ctx):
    return ctx.k - 1 if ctx.k > 1 else 1


def plaintexts(scheme, B, L, n, mods, t, seed=1):
    """CKKS: [B][L][n] words below each prime (a valid NTT-form plaintext); BFV / BGV: [B][n] words < t, with the lift edges
    0, t - 1, (t + 1) / 2 and (t + 1) / 2 - 1 among them"""
    rng = np.random.default_rng(seed)
    if scheme == "ckks":
        return np.stack([np.stack([rng.integers(0, mods[j], n, dtype=np.uint64) for j in range(L)]) for _ in range(B)])
    p = rng.integers(0, t, (B, n), dtype=np.uint64)
    h = (t + 1) // 2
    p[:, :4] = np.array([0, t - 1, h, h - 1], dtype=np.uint64)
    p[:, -4:] = np.array([h - 1, h, t - 1, 0], dtype=np.uint64)
    return p


def seeds_for(B, salt=0):
    s = (np.arange(B * 8, dtype=np.uint64).reshape(B, 8) + np.uint64(salt)) * np.uint64(0x9E3779B97F4A7C15)
    s[:, 0] ^= np.uint64(0xC0FFEE)
    return s


def dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def zeros(B, L, n):
    import torch

    return torch.zeros((B, 2, L, n), dtype=torch.int64, device="cuda")


def composed_symmetric(ctx, sk, plain, L, B, seeds, save_seed=False, bprng=1, cprng=1):
    out = zeros(B, L, ctx.n)
    pub = ctx.d_encrypt_zero_symmetric(sk, out, L, B, seeds, save_seed=save_seed, want_public_seeds=True, bootstrap_prng=bprng,
                                       ciphertext_prng=cprng)
    add_plain(ctx, out, plain, L, B)
    return out, pub


def composed_asymmetric(ctx, pk, plain, L, B, seeds, prng=1):
    out = zeros(B, L, ctx.n)
    ctx.d_encrypt_zero_asymmetric(pk, out, L, B, seeds, prng=prng)
    add_plain(ctx, out, plain, L, B)
    return out


def add_plain(ctx, out, plain, L, B):
    S = sb()
    if ctx.scheme == S.CKKS:
        ctx.d_add_plain_ntt(out, plain, out, L, 2, B, B)
    else:
        ctx.d_add_plain_coeff_n(out, plain, out, L, 2, B, B)


SHAPES = [("ckks", 4096, [50, 50, 50], 20), ("bfv", 4096, [50, 50, 50], 20), ("bfv", 4096, [50, 50, 50], 40),
          ("bgv", 4096, [50, 50, 50], 20), ("bgv", 4096, [50, 50, 50], 40), ("ckks", 32768, [60] * 3, 20),
          ("bfv", 32768, [60] * 3, 38)]


@pytest.mark.parametrize("scheme,n,qbits,tbits", SHAPES)
def test_fused_equals_composed(scheme, n, qbits, tbits):
    """Both entry points give the composition's words, with a distinct seed per batch member, for blake2xb and shake256 bootstrap
    PRNGs, c_1 expanded with either type, BFV with and without save_seed (the same public seeds), CKKS at the first and a lower
    level, t of 20 and 38+ bits with plaintext words at the lift edges, and n = 4096 and 32768 with 60-bit primes"""
    import torch

    ctx, sk, pk, t, mods = make(scheme, n, qbits, tbits)
    B = 3
    levels = [first_level(ctx)] + ([1] if scheme == "ckks" else [])
    for L in levels:
        plain = dev(plaintexts(scheme, B, L, n, mods, t, seed=L))
        seeds = seeds_for(B, L)
        for bprng, cprng in ((1, 1), (2, 1), (2, 2)):
            for save_seed in ((False, True) if scheme == "bfv" else (False,)):
                out = zeros(B, L, n)
                pub = ctx.d_encrypt_symmetric(sk, plain, out, L, B, seeds, save_seed=save_seed, want_public_seeds=True,
                                              bootstrap_prng=bprng, ciphertext_prng=cprng)
                want, wpub = composed_symmetric(ctx, sk, plain, L, B, seeds, save_seed, bprng, cprng)
                torch.cuda.synchronize()
                assert (to_np(out) == to_np(want)).all(), f"symmetric L={L} prng=({bprng},{cprng}) save_seed={save_seed}"
                assert (pub == wpub).all()
        for prng in (1, 2):
            out = zeros(B, L, n)
            ctx.d_encrypt_asymmetric(pk, plain, out, L, B, seeds, prng=prng)
            want = composed_asymmetric(ctx, pk, plain, L, B, seeds, prng)
            torch.cuda.synchronize()
            assert (to_np(out) == to_np(want)).all(), f"asymmetric L={L} prng={prng}"


@pytest.mark.parametrize("scheme", ["ckks", "bfv", "bgv"])
def test_launch_counts(scheme):
    """The symmetric fused call launches exactly the kernels of sb200_encrypt_zero_symmetric_prng; the public-key one adds one
    launch to sb200_encrypt_zero_asymmetric_prng (two for BGV: the plaintext's lift-and-transform, then the add)"""
    import torch

    ctx, sk, pk, t, mods = make(scheme, 8192, [50, 50, 50])
    B, L = 4, first_level(ctx)
    plain, seeds = dev(plaintexts(scheme, B, L, ctx.n, mods, t)), seeds_for(B)
    out = zeros(B, L, ctx.n)
    for save_seed in (False, True):
        ctx.d_encrypt_symmetric(sk, plain, out, L, B, seeds, save_seed=save_seed)  # warm: lazily built tables
        c0 = ctx.launch_count
        ctx.d_encrypt_zero_symmetric(sk, out, L, B, seeds, save_seed=save_seed)
        c1 = ctx.launch_count
        ctx.d_encrypt_symmetric(sk, plain, out, L, B, seeds, save_seed=save_seed)
        c2 = ctx.launch_count
        assert c2 - c1 == c1 - c0 > 0
    ctx.d_encrypt_asymmetric(pk, plain, out, L, B, seeds)
    c0 = ctx.launch_count
    ctx.d_encrypt_zero_asymmetric(pk, out, L, B, seeds)
    c1 = ctx.launch_count
    add_plain(ctx, out, plain, L, B)
    c2 = ctx.launch_count
    ctx.d_encrypt_asymmetric(pk, plain, out, L, B, seeds)
    c3 = ctx.launch_count
    torch.cuda.synchronize()
    assert c3 - c2 == (c1 - c0) + (c2 - c1)
    if scheme != "bgv":
        assert c2 - c1 == 1  # the add alone; BGV adds its lift-and-transform (one forward transform) in front of it
    else:
        ctx.profile(True)
        add_plain(ctx, out, plain, L, B)
        torch.cuda.synchronize()
        names = [e[0] for e in ctx.profile_read()]
        ctx.profile(False)
        assert names.count("bgv_add_plain") == 1 and all(x in ("plain_lift_ntt", "bgv_add_plain") or x.startswith("plain_lift_ntt")
                                                         for x in names), names


@pytest.mark.parametrize("scheme", ["ckks", "bfv", "bgv"])
def test_chunking_keeps_words(scheme):
    """With SB200_LIMIT_SCRATCH_BYTES at its 1 MiB floor, n = 4096 with 3 primes cuts 13 ciphertexts into 6 + 6 + 1 (symmetric)
    and six chunks of 2 plus one of 1 (public key): the words of the new and of both zero-plaintext entry points equal a single-chunk run"""
    import torch

    S = sb()
    ctx, sk, pk, t, mods = make(scheme, 4096, [50, 50, 50])
    B, L, n = 13, first_level(ctx), ctx.n
    plain, seeds = dev(plaintexts(scheme, B, L, n, mods, t)), seeds_for(B, 9)

    def run_all():
        outs = [zeros(B, L, n) for _ in range(4)]
        c0 = ctx.launch_count
        p1 = ctx.d_encrypt_symmetric(sk, plain, outs[0], L, B, seeds, save_seed=True, want_public_seeds=True)
        p2 = ctx.d_encrypt_zero_symmetric(sk, outs[1], L, B, seeds, save_seed=True, want_public_seeds=True)
        ctx.d_encrypt_asymmetric(pk, plain, outs[2], L, B, seeds)
        ctx.d_encrypt_zero_asymmetric(pk, outs[3], L, B, seeds)
        torch.cuda.synchronize()
        return [to_np(o) for o in outs] + [p1, p2], ctx.launch_count - c0

    whole, launches_whole = run_all()
    ctx.set_limit(S.Context.LIMIT_SCRATCH_BYTES, 1 << 20)
    try:
        chunked, launches_chunked = run_all()
    finally:
        ctx.set_limit(S.Context.LIMIT_SCRATCH_BYTES, 8 << 30)
    assert launches_chunked > launches_whole  # the batch was cut
    for i, (a, b) in enumerate(zip(whole, chunked)):
        assert (a == b).all(), f"output {i} depends on the chunking"


@pytest.mark.parametrize("scheme,tbits", [("bfv", 20), ("bfv", 40), ("bgv", 20), ("bgv", 40)])
def test_round_trip(scheme, tbits):
    """BFV and BGV: decrypt(encrypt(m)) == m for both key types, plaintext words at the lift edges included"""
    ctx, sk, pk, t, mods = make(scheme, 4096, [50, 50, 50], tbits)
    B, L = 5, first_level(ctx)
    m = plaintexts(scheme, B, L, ctx.n, mods, t, seed=3)
    plain, seeds = dev(m), seeds_for(B, 3)
    for ct in (ctx.encrypt_symmetric(sk, m, seeds), ctx.encrypt_asymmetric(pk, m, seeds)):
        assert ct.shape == (B, 2, L, ctx.n)
        assert (ctx.decrypt(ct, sk) == m).all()
    out = zeros(B, L, ctx.n)
    ctx.d_encrypt_symmetric(sk, plain, out, L, B, seeds, save_seed=True)
    assert (ctx.decrypt(to_np(out), sk) == m).all()


@pytest.mark.parametrize("scheme", ["ckks", "bfv", "bgv"])
def test_errors(scheme):
    """Wrong BFV / BGV level, the key level (symmetric), d_plain == d_out, NULL pointers, a key of another context, PRNG types 0 and
    3: SB200_E_INVALID_ARG / SB200_E_POINTER before anything is written"""
    import torch

    ctx, sk, pk, t, mods = make(scheme, 4096, [50, 50, 50])
    other, osk, opk, _, _ = make(scheme, 4096, [50, 50, 50])
    B, L, n = 2, first_level(ctx), ctx.n
    plain, seeds = dev(plaintexts(scheme, B, L, n, mods, t)), seeds_for(B)
    out = zeros(B, L, n)
    sentinel = out.clone()

    def untouched():
        torch.cuda.synchronize()
        assert torch.equal(out, sentinel)

    if scheme != "ckks":
        for bad_L in (1, ctx.k):
            o = zeros(B, bad_L, n)
            with pytest.raises(ValueError, match="first level"):
                ctx.d_encrypt_asymmetric(pk, plain, o, bad_L, B, seeds)
        with pytest.raises(ValueError, match="first level"):
            ctx.d_encrypt_symmetric(sk, plain, zeros(B, 1, n), 1, B, seeds)
    with pytest.raises(ValueError, match="parms_id is not valid"):
        ctx.d_encrypt_symmetric(sk, plain, zeros(B, ctx.k, n), ctx.k, B, seeds)
    with pytest.raises(ValueError, match="alias"):
        ctx.d_encrypt_symmetric(sk, out, out, L, B, seeds)
    with pytest.raises(ValueError, match="alias"):
        ctx.d_encrypt_asymmetric(pk, out, out, L, B, seeds)
    untouched()
    with pytest.raises(ValueError, match="null pointer"):
        ctx.d_encrypt_symmetric(sk, 0, out, L, B, seeds)
    with pytest.raises(ValueError, match="null pointer"):
        ctx.d_encrypt_asymmetric(pk, 0, out, L, B, seeds)
    with pytest.raises(ValueError, match="null pointer"):
        ctx.d_encrypt_symmetric(sk, plain, 0, L, B, seeds)
    with pytest.raises(ValueError, match="secret key is not valid"):
        ctx.d_encrypt_symmetric(osk, plain, out, L, B, seeds)
    with pytest.raises(ValueError, match="public key is not valid"):
        ctx.d_encrypt_asymmetric(opk, plain, out, L, B, seeds)
    for bad in (0, 3):
        with pytest.raises(ValueError, match="prng_type is invalid"):
            ctx.d_encrypt_symmetric(sk, plain, out, L, B, seeds, bootstrap_prng=bad)
        with pytest.raises(ValueError, match="prng_type is invalid"):
            ctx.d_encrypt_symmetric(sk, plain, out, L, B, seeds, ciphertext_prng=bad)
        with pytest.raises(ValueError, match="prng_type is invalid"):
            ctx.d_encrypt_asymmetric(pk, plain, out, L, B, seeds, prng=bad)
    untouched()


# ---- word-for-word parity with seal::Encryptor (oracle/ref_encrypt.cpp) ----
_REF_ENC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref", "libsealref_encrypt.so")
needs_ref = pytest.mark.skipif(not os.path.exists(_REF_ENC), reason="oracle/_ref/libsealref_encrypt.so not present")


def ref_encrypt(sid, n, mods, t, key, asym, seed, prng, save_seed, plain, L, scale=1.0):
    """seal::Encryptor::encrypt (asym) / encrypt_symmetric of one plaintext under a factory of type prng seeded with seed:
    [2][L][n], or (c_0 [L][n], seed [8]) of the Serializable object when save_seed"""
    lib = C.CDLL(_REF_ENC)
    u64p = C.POINTER(C.c_uint64)
    lib.sealenc_encrypt.restype = C.c_long
    lib.sealenc_encrypt.argtypes = [C.c_int, C.c_size_t, u64p, C.c_size_t, C.c_uint64, u64p, C.c_int, u64p, C.c_int, C.c_int, u64p,
                                    C.c_size_t, C.c_size_t, C.c_double, u64p, u64p]
    lib.sealenc_last_error.restype = C.c_char_p

    def p(a):
        return a.ctypes.data_as(u64p)

    m = np.array(mods, dtype=np.uint64)
    key, seed, plain = (np.ascontiguousarray(x, dtype=np.uint64) for x in (key, seed, plain))
    out, out_seed = np.zeros((2, L, n), dtype=np.uint64), np.zeros(8, dtype=np.uint64)
    r = lib.sealenc_encrypt(sid, n, p(m), len(mods), t, p(key), int(asym), p(seed), prng, int(save_seed), p(plain), plain.size, L, scale,
                            p(out), p(out_seed))
    assert r == L, lib.sealenc_last_error().decode()
    return (out[0], out_seed) if save_seed else out


PARITY = [("ckks", 4096, [50, 50, 50], 20), ("bfv", 4096, [50, 50, 50], 20), ("bfv", 4096, [50, 50, 50], 40),
          ("bgv", 4096, [50, 50, 50], 20), ("bgv", 4096, [50, 50, 50], 40), ("bfv", 4096, [30, 30, 30, 30], 40),
          ("bgv", 4096, [30, 30, 30, 30], 40), ("ckks", 32768, [60] * 3, 20), ("bfv", 32768, [60] * 3, 38)]


@needs_ref
@pytest.mark.parametrize("scheme,n,qbits,tbits", PARITY)
def test_parity_vs_reference(scheme, n, qbits, tbits):
    """Both entry points against seal::Encryptor word for word, a distinct seed per batch member: blake2xb and shake256 bootstrap
    PRNGs; BFV with save_seed (c_0 and the public seeds against the reference's Serializable object); CKKS at the first and the
    lowest level; t of 20 to 40 bits with words at the lift edges, t above every q_j (30-bit primes); n = 4096 and 32768 with
    60-bit primes.  ciphertext_prng = 2: c_1 is tests/refprng.py's SHAKE256 expansion and c_0 the restated encryption of zero plus
    the reference's plaintext term."""
    import torch

    import refprng as P

    S = sb()
    allm = O.coeff_modulus_create(n, list(qbits) + ([tbits] if scheme != "ckks" else []))
    mods, t = ([int(q) for q in allm], 0) if scheme == "ckks" else ([int(q) for q in allm[:-1]], int(allm[-1]))
    sids = {"ckks": (P.CKKS, S.CKKS, O.CKKS), "bfv": (P.BFV, S.BFV, O.BFV), "bgv": (P.BGV, S.BGV, O.BGV)}[scheme]
    rc = P.RefPrngContext(sids[0], n, mods, t, seed=0xA11CE, prng=P.BLAKE2XB)
    sk_host, pk_host = rc.secret_key(), rc.public_key()
    ctx = S.Context(sids[1], n, mods, t)
    sk, pk = ctx.load_secret_key(sk_host), ctx.load_public_key(pk_host)
    po = P.PrngOracle(O.Oracle(sids[2], n, mods, t))
    k, B = len(mods), 3
    qcol = np.array(mods, dtype=np.uint64)[:, None]
    for L in [first_level(ctx)] + ([1] if scheme == "ckks" and k > 2 else []):
        m = plaintexts(scheme, B, L, n, mods, t, seed=L + 5)
        plain, seeds = dev(m), seeds_for(B, L + 11)
        for prng in (1, 2):
            for save_seed in ((False, True) if scheme == "bfv" else (False,)):
                out = zeros(B, L, n)
                pub = ctx.d_encrypt_symmetric(sk, plain, out, L, B, seeds, save_seed=save_seed, want_public_seeds=True, bootstrap_prng=prng)
                torch.cuda.synchronize()
                got = to_np(out)
                for b in range(B):
                    want = ref_encrypt(sids[0], n, mods, t, sk_host, False, seeds[b], prng, save_seed, m[b], L, 2.0 ** 20)
                    if save_seed:
                        assert (got[b][0] == want[0]).all() and (pub[b] == want[1]).all(), f"seeded L={L} prng={prng} member {b}"
                    else:
                        assert (got[b] == want).all(), f"symmetric L={L} prng={prng} member {b}"
            out = zeros(B, L, n)
            ctx.d_encrypt_asymmetric(pk, plain, out, L, B, seeds, prng=prng)
            torch.cuda.synchronize()
            got = to_np(out)
            for b in range(B):
                want = ref_encrypt(sids[0], n, mods, t, pk_host, True, seeds[b], prng, False, m[b], L, 2.0 ** 20)
                assert (got[b] == want).all(), f"public key L={L} prng={prng} member {b}"
        # c_1 expanded with SHAKE256: the plaintext term is the reference's (its c_0 minus its encryption of zero, restated)
        for save_seed in ((False, True) if scheme == "bfv" else (False,)):
            out = zeros(B, L, n)
            ctx.d_encrypt_symmetric(sk, plain, out, L, B, seeds, save_seed=save_seed, bootstrap_prng=2, ciphertext_prng=2)
            torch.cuda.synchronize()
            got = to_np(out)
            q = qcol[:L]
            for b in range(B):
                ref_ct = ref_encrypt(sids[0], n, mods, t, sk_host, False, seeds[b], 2, False, m[b], L, 2.0 ** 20)
                z1 = po.encrypt_zero_symmetric(sk_host, seeds[b], False, 2, 1, L=L)
                term = (ref_ct[0] + q - z1[0]) % q
                z2 = po.encrypt_zero_symmetric(sk_host, seeds[b], save_seed, 2, 2, L=L)
                assert (got[b][1] == z2[1]).all(), f"c_1, ciphertext_prng 2, member {b}"
                assert (got[b][0] == (z2[0] + term) % q).all(), f"c_0, ciphertext_prng 2, member {b}"


@needs_ref
def test_cpp_encryptor_decryptor_encoders_against_seal():
    """tests/cpp/shim_encrypt_test.cpp: the PlaintextBatch / CiphertextBatch members of seal_b200::Encryptor, Decryptor and the
    encoders against the seal:: classes under seeded Blake2xb and Shake256 factories, and CKKS, BFV and BGV chains on the device"""
    import subprocess

    exe = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref", "bin", "shim_encrypt_test")
    if not os.path.exists(exe):
        pytest.skip("shim_encrypt_test not built (reference sources absent at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert "shim_encrypt_test ok" in r.stdout
