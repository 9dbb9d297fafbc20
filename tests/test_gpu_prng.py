"""The device's PRNG paths on an H100 (-m gpu; seal_b200/csrc/sb_prng.cu): seed-compressed ciphertexts and key-switching keys
of either PRNG type (blake2xb, shake256) loaded on the device, and encryption with SHAKE256 PRNGs, word for word against the
reference's own loaders and Encryptor (oracle/ref_prng.cpp) and against the restatement of tests/refprng.py."""
import os
import subprocess

import numpy as np
import pytest

import oracle as O
import refprng as P

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not P.ref_available(), reason="oracle/_ref/libsealref_prng.so not present")


def sb():
    import seal_b200

    return seal_b200


def to_np(x):
    return x.cpu().numpy().view(np.uint64)


@needs_ref
@pytest.mark.parametrize("scheme,n,bits", [("ckks", 8192, [60, 60, 60, 60]), ("bfv", 4096, [36, 36, 37]), ("ckks", 32768, [60] * 3),
                                          ("bfv", 32768, [60] * 3)])
def test_mixed_prng_seeded_loads_vs_reference(scheme, n, bits):
    """Ciphertext::load of one batch mixing blake2xb-seeded, shake256-seeded (the reference's seeded streams retyped), unseeded and
    zlib-compressed shake256-seeded members: every word equals the reference's own load, and the shake256 members' c_1 equals the
    restatement's expansion (SHAKE256 stream + sample_poly_uniform); 60-bit primes reject about one stream word in 16"""
    import torch

    import refseal as R

    mods = O.coeff_modulus_create(n, bits)
    t = R.plain_modulus_batching(n, 20) if scheme == "bfv" else 0
    sid = P.BFV if scheme == "bfv" else P.CKKS
    rcs = [P.RefPrngContext(sid, n, mods, t, seed=s, prng=P.BLAKE2XB) for s in (0x5EA1, 0xBEEF)]  # same parameters, two seeds
    ctx = sb().Context(sid, n, mods, t)
    po = P.PrngOracle(O.Oracle(O.BFV if scheme == "bfv" else O.CKKS, n, mods, t))
    L = len(mods) - 1
    s1, s2 = rcs[0].seeded_ct_stream(), rcs[1].seeded_ct_stream()
    plain = R.RefContext(sid, n, mods, t).ct_save(L, rcs[1].ct_load(s2), scheme != "bfv", 1.0)
    streams = [P.with_prng_type(s1, 2), s1, plain, P.zlib_stream(P.with_prng_type(s2, 2)), s2, P.with_prng_type(s2, 2)]
    want = [rcs[0].ct_load(s) for s in streams]
    dev = torch.zeros((len(streams), 2, L, n), dtype=torch.int64, device="cuda")
    infos = ctx.d_load_ciphertexts(streams, dev, L, 2)
    torch.cuda.synchronize()
    got = to_np(dev)
    assert [i.seeded for i in infos] == [2, 1, 0, 2, 1, 2]
    assert [i.compr_mode for i in infos] == [0, 0, 0, 1, 0, 0]
    for b, (g, w) in enumerate(zip(got, want)):
        assert (g == w).all(), f"member {b} vs the reference's load"
    for b in (0, 5):
        seed = np.frombuffer(streams[b], dtype=np.uint64, count=8, offset=infos[b].seed_offset)
        assert (po.expand_seed(L, seed, P.SHAKE256) == got[b][1]).all(), f"member {b} vs the restatement"
    assert not (got[0][1] == got[1][1]).all()  # same seed, different PRNG


@needs_ref
@pytest.mark.parametrize("scheme,n,bits", [("ckks", 8192, [50, 50, 50, 51]), ("bfv", 4096, [36, 36, 37]), ("bgv", 4096, [40, 40, 40]),
                                          ("ckks", 2048, [54])])
def test_encrypt_zero_with_shake256_vs_reference(scheme, n, bits):
    """sb200_encrypt_zero_symmetric_prng / _asymmetric_prng with SHAKE256 PRNGs against the reference's Encryptor on parameters that
    carry Shake256PRNGFactory(seed): symmetric (bootstrap 2, both save_seed variants), public-key (first data level, lowest level, key
    level), other seeds of the batch against the restatement.  ciphertext_prng = 2: c_1 equals the reference's load of a (c_0,
    public seed, shake256) stream built from the device output, and the whole ciphertext equals the restatement.  Invalid types
    (0, 3) are SB200_E_INVALID_ARG."""
    import torch

    import refseal as R

    S = sb()
    mods = O.coeff_modulus_create(n, bits)
    t = R.plain_modulus_batching(n, 20) if scheme != "ckks" else 0
    sid = {"ckks": (P.CKKS, S.CKKS, O.CKKS), "bfv": (P.BFV, S.BFV, O.BFV), "bgv": (P.BGV, S.BGV, O.BGV)}[scheme]
    seed0 = 0xC0FFEE
    rc = P.RefPrngContext(sid[0], n, mods, t, seed=seed0, prng=P.SHAKE256)
    po = P.PrngOracle(O.Oracle(sid[2], n, mods, t))
    ctx = S.Context(sid[1], n, mods, t)
    sk_host, pk_host = rc.secret_key(), rc.public_key()
    sk, pk = ctx.load_secret_key(sk_host), ctx.load_public_key(pk_host)
    k = len(mods)
    L = k - 1 if k > 1 else 1
    batch = 3
    seeds = np.zeros((batch, 8), dtype=np.uint64)
    seeds[0, 0] = seed0
    seeds[1] = np.arange(1, 9, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    seeds[2, 7] = 5
    ref_seeded = rc.seeded_ct_stream()
    info = S.ciphertext_inspect(ref_seeded)
    for save_seed in (False, True):
        out = torch.zeros((batch, 2, L, n), dtype=torch.int64, device="cuda")
        pub = ctx.d_encrypt_zero_symmetric(sk, out, L, batch, seeds, save_seed=save_seed, want_public_seeds=True, bootstrap_prng=2)
        torch.cuda.synchronize()
        got = to_np(out)
        want0 = rc.ct_load(ref_seeded) if save_seed else rc.encrypt_zero_symmetric()
        assert (got[0] == want0).all(), f"ciphertext 0 vs the reference, save_seed={save_seed}"
        for b in range(batch):
            assert (got[b] == po.encrypt_zero_symmetric(sk_host, seeds[b], save_seed, 2, 1)).all(), f"ciphertext {b} vs the restatement"
            assert (pub[b] == P.stream(P.SHAKE256, seeds[b], 8)).all()
        # c_1 expanded with SHAKE256 as well
        out = torch.zeros((batch, 2, L, n), dtype=torch.int64, device="cuda")
        pub = ctx.d_encrypt_zero_symmetric(sk, out, L, batch, seeds, save_seed=save_seed, want_public_seeds=True, bootstrap_prng=2,
                                           ciphertext_prng=2)
        torch.cuda.synchronize()
        got = to_np(out)
        for b in range(batch):
            assert (got[b] == po.encrypt_zero_symmetric(sk_host, seeds[b], save_seed, 2, 2)).all(), f"ciphertext_prng 2, {b}"
            if save_seed or scheme != "bfv":  # the seeded wire form: c_1 is what the seed expands into
                st = bytearray(P.with_prng_type(ref_seeded, 2))
                st[info.data_offset:info.data_offset + L * n * 8] = got[b][0].tobytes()
                st[info.seed_offset:info.seed_offset + 64] = pub[b].tobytes()
                assert (rc.ct_load(bytes(st))[1] == got[b][1]).all(), f"c_1 vs the reference's load, ciphertext {b}"
    if k > 2:
        out = torch.zeros((1, 2, 1, n), dtype=torch.int64, device="cuda")
        ctx.d_encrypt_zero_symmetric(sk, out, 1, 1, seeds[:1], bootstrap_prng=2)
        torch.cuda.synchronize()
        assert (to_np(out)[0] == rc.encrypt_zero_symmetric(L=1)).all()
    for Lv in sorted({L, 1, k}):
        out = torch.zeros((batch, 2, Lv, n), dtype=torch.int64, device="cuda")
        ctx.d_encrypt_zero_asymmetric(pk, out, Lv, batch, seeds, prng=2)
        torch.cuda.synchronize()
        got = to_np(out)
        assert (got[0] == rc.encrypt_zero_asymmetric(L=Lv)).all(), f"level {Lv} vs the reference"
        for b in range(1, batch):
            assert (got[b] == po.encrypt_zero_asymmetric(pk_host, seeds[b], 2, L=Lv)).all(), f"level {Lv}, ciphertext {b}"
    out = torch.zeros((1, 2, L, n), dtype=torch.int64, device="cuda")
    for bad in (0, 3):
        with pytest.raises(ValueError, match="prng_type is invalid"):
            ctx.d_encrypt_zero_symmetric(sk, out, L, 1, seeds[:1], bootstrap_prng=bad)
        with pytest.raises(ValueError, match="prng_type is invalid"):
            ctx.d_encrypt_zero_symmetric(sk, out, L, 1, seeds[:1], ciphertext_prng=bad)
        with pytest.raises(ValueError, match="prng_type is invalid"):
            ctx.d_encrypt_zero_asymmetric(pk, out, L, 1, seeds[:1], prng=bad)


@needs_ref
@pytest.mark.parametrize("n,bits", [(4096, [30] * 18), (8192, [50, 50, 50, 51])])
def test_seeded_key_streams_vs_reference(n, bits):
    """RelinKeys / GaloisKeys as KeyGenerator::create_relin_keys() / create_galois_keys() return them (seeded: c_0 and the seed of
    c_1 per digit), of either prng_type, uncompressed and zlib-compressed, loaded on the device (c_1 expanded at the key level).
    relinearize / apply_galois with the loaded key equal the oracle with the key words of the reference's KSwitchKeys::load and the
    library with those words uploaded directly, in both key-switching modes (17 digits: the integer path prepares an expanded key)"""
    S = sb()
    mods = O.coeff_modulus_create(n, bits)
    k, L = len(mods), len(mods) - 1
    rc = P.RefPrngContext(P.CKKS, n, mods, prng=P.BLAKE2XB)
    ctx = S.Context(S.CKKS, n, mods)
    oc = O.Oracle(O.CKKS, n, mods)
    rng = np.random.default_rng(n + k)
    c3 = np.stack([np.stack([rng.integers(0, mods[i], n, dtype=np.uint64) for i in range(L)]) for _ in range(3)])[None]
    c2 = np.ascontiguousarray(c3[:, :2])
    elt = ctx.galois_elt_from_step(1)
    for prng in (1, 2):
        for compr in (0, 1):
            for galois_elt, index in ((0, 0), (elt, (elt - 1) // 2)):
                raw = P.kswitch_with_prng_type(rc.seeded_kswitch_keys_stream(galois_elt), prng)
                data = P.zlib_stream(raw) if compr else raw
                want_key = rc.kswitch_keys_load(data, index)
                key = ctx.load_key_stream(data, index)
                direct = ctx.load_key(want_key)
                want = oc.relinearize(L, c3[0], want_key) if galois_elt == 0 else oc.apply_galois(L, c2[0], galois_elt, want_key)
                for mode in (0, 2):
                    ctx.set_limit(S.Context.LIMIT_KS_ALGORITHM, mode)
                    run = (lambda kk: ctx.relinearize(c3, kk)) if galois_elt == 0 else (lambda kk: ctx.apply_galois(c2, galois_elt, kk))
                    got = run(key)
                    case = f"prng {prng}, compr {compr}, galois_elt {galois_elt}, mode {mode}"
                    assert (got[0] == want).all(), case + ": vs the oracle with the reference-loaded key"
                    assert (got == run(direct)).all(), case + ": vs the reference-loaded key uploaded directly"
                ctx.set_limit(S.Context.LIMIT_KS_ALGORITHM, 1)


SHIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref", "bin", "shim_prng_test")


@pytest.mark.skipif(not os.path.exists(SHIM), reason="oracle/_ref/bin/shim_prng_test not built (oracle/prng.mk, needs the reference sources)")
def test_cpp_encryptor_under_shake256_factory():
    """seal_b200::Encryptor against seal::Encryptor with Shake256PRNGFactory(seed) on the parameters: secret- and public-key
    encryption, all three schemes, words and metadata (tests/cpp/shim_prng_test.cpp)"""
    r = subprocess.run([SHIM], capture_output=True, text=True, timeout=600)
    print(r.stdout, r.stderr)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "PASS" in r.stdout
