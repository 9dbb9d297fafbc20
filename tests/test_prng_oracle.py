"""CPU checks of the test infrastructure behind the device's PRNG paths (tests/refprng.py): the FIPS 202 SHAKE256 of
oracle/shake256.c against Python's hashlib (independent of the reference), both PRNG streams against the reference's
Blake2xbPRNG / Shake256PRNG, and the restatement of what the reference samples from a stream -- seed expansion, symmetric and
public-key encryption, seeded key-switching keys -- against the reference under a Shake256PRNGFactory and against the existing
blake2xb oracle."""
import hashlib

import numpy as np
import pytest

import oracle as O
import refprng as P

needs_ref = pytest.mark.skipif(not P.ref_available(), reason="oracle/_ref/libsealref_prng.so not present")
SEED = np.arange(1, 9, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)


def _setup(scheme, n, bits, prng, seed0=0x5EA1):
    mods = O.coeff_modulus_create(n, bits)
    t = 0
    if scheme != "ckks":
        import refseal as R

        t = R.plain_modulus_batching(n, 20)
    sid = {"ckks": P.CKKS, "bfv": P.BFV, "bgv": P.BGV}[scheme]
    rc = P.RefPrngContext(sid, n, mods, t, seed=seed0, prng=prng)
    oc = O.Oracle({"ckks": O.CKKS, "bfv": O.BFV, "bgv": O.BGV}[scheme], n, mods, t)
    return mods, rc, oc, P.PrngOracle(oc)


def test_shake256_matches_hashlib():
    """the FIPS 202 empty-message vector, messages of one block, exactly the rate and several blocks, and whole Shake256PRNG
    buffers SHAKE256(seed || counter, 4096 bytes) for counters 0, 1, 2 and 37"""
    assert P.shake256(b"", 32).hex().startswith("46b9dd2b0ba88d13")
    assert P.shake256(b"", 32) == hashlib.shake_256(b"").digest(32)
    for m in (b"abc", bytes(range(136)), bytes(range(200)) * 3):
        assert P.shake256(m, 300) == hashlib.shake_256(m).digest(300)
    s = P.stream(P.SHAKE256, SEED, 512 * 38)
    for counter in (0, 1, 2, 37):
        want = hashlib.shake_256(SEED.tobytes() + np.uint64(counter).tobytes()).digest(4096)
        assert s[512 * counter:512 * (counter + 1)].tobytes() == want, counter


@needs_ref
def test_prng_streams_match_reference():
    """both streams against UniformRandomGenerator::generate of the reference's PRNGs, across several buffer refills"""
    for seed in (np.zeros(8, dtype=np.uint64), SEED):
        for prng in (P.BLAKE2XB, P.SHAKE256):
            assert P.stream(prng, seed, 512 * 5 + 3).tobytes() == P.ref_stream(prng, seed, 4096 * 5 + 24), prng


@pytest.mark.parametrize("scheme,n,bits", [("ckks", 4096, [40, 40, 40, 40]), ("bfv", 4096, [36, 36, 37]), ("bgv", 4096, [40, 40, 40])])
def test_restatement_matches_the_blake2xb_oracle(scheme, n, bits):
    """on the blake2xb stream the restatement gives the words of oracle/seal_oracle.c (pinned against the reference by
    test_oracle.py): seed expansion, both symmetric variants, public-key encryption at every level kind"""
    mods = O.coeff_modulus_create(n, bits)
    t = 65537 if scheme != "ckks" else 0
    oc = O.Oracle({"ckks": O.CKKS, "bfv": O.BFV, "bgv": O.BGV}[scheme], n, mods, t)
    po = P.PrngOracle(oc)
    k = len(mods)
    rng = np.random.default_rng(3)
    sk = np.stack([rng.integers(0, q, n, dtype=np.uint64) for q in mods])
    pk = np.stack([np.stack([rng.integers(0, q, n, dtype=np.uint64) for q in mods]) for _ in range(2)])
    assert (po.expand_seed(k - 1, SEED, 1) == oc.expand_seed(k - 1, SEED)).all()
    for save_seed in (False, True):
        assert (po.encrypt_zero_symmetric(sk, SEED, save_seed, 1, 1) == oc.encrypt_zero_symmetric(sk, SEED, save_seed)).all()
    for L in sorted({k - 1, 1, k}):
        assert (po.encrypt_zero_asymmetric(pk, SEED, 1, L=L) == oc.encrypt_zero_asymmetric(pk, SEED, L=L)).all(), L


@needs_ref
@pytest.mark.parametrize("scheme,n,bits", [("ckks", 4096, [40, 40, 40]), ("ckks", 8192, [60, 60, 60]), ("bfv", 4096, [36, 36, 37])])
def test_expand_seed_shake256_matches_reference_load(scheme, n, bits):
    """the restatement's expansion on a Shake256PRNG against the reference loading a seeded stream whose prng_type names shake256
    (UniformRandomGeneratorInfo::make_prng reads the type from the stream); 60-bit primes reject about one word in 16.  The zlib
    form of the same stream loads to the same words."""
    import seal_b200 as S

    for seed0 in (0x5EA1, 77):
        _, rc, _, po = _setup(scheme, n, bits, P.BLAKE2XB, seed0)
        data = P.with_prng_type(rc.seeded_ct_stream(), P.SHAKE256)
        info = S.ciphertext_inspect(data)
        assert info.seeded == 2
        L = info.coeff_modulus_size
        full = rc.ct_load(data)
        seed = np.frombuffer(data, dtype=np.uint64, count=8, offset=info.seed_offset)
        assert (po.expand_seed(L, seed, P.SHAKE256) == full[1]).all()
        assert not (po.expand_seed(L, seed, P.BLAKE2XB) == full[1]).all()  # the type byte matters
        assert (rc.ct_load(P.zlib_stream(data)) == full).all()


@needs_ref
@pytest.mark.parametrize("scheme,n,bits", [("ckks", 4096, [40, 40, 40, 40]), ("bfv", 4096, [36, 36, 37]), ("bgv", 4096, [40, 40, 40]),
                                          ("ckks", 2048, [54])])
def test_encryption_under_shake256_factory_matches_reference(scheme, n, bits):
    """symmetric (both save_seed variants) and public-key encryption with SHAKE256 bootstrap / encryption PRNGs against the
    reference's Encryptor on parameters carrying Shake256PRNGFactory(seed); c_1 is expanded with the reference build's default
    PRNG (blake2xb).  The ciphertext_prng = 2 arm: c_1 equals the reference's load of the seeded stream retyped to shake256."""
    import seal_b200 as S

    mods, rc, oc, po = _setup(scheme, n, bits, P.SHAKE256)
    sk, pk = rc.secret_key(), rc.public_key()
    seed = np.zeros(8, dtype=np.uint64)
    seed[0] = 0x5EA1
    k = len(mods)
    assert (po.encrypt_zero_symmetric(sk, seed, False, 2, 1) == rc.encrypt_zero_symmetric()).all()
    assert not (po.encrypt_zero_symmetric(sk, seed, False, 1, 1) == rc.encrypt_zero_symmetric()).all()
    data = rc.seeded_ct_stream()
    assert S.ciphertext_inspect(data).seeded == 1  # the default factory names c_1's PRNG
    assert (po.encrypt_zero_symmetric(sk, seed, True, 2, 1) == rc.ct_load(data)).all()
    retyped = rc.ct_load(P.with_prng_type(data, P.SHAKE256))
    assert (po.encrypt_zero_symmetric(sk, seed, True, 2, 2)[1] == retyped[1]).all()
    if k > 2:
        assert (po.encrypt_zero_symmetric(sk, seed, False, 2, 1, L=1) == rc.encrypt_zero_symmetric(L=1)).all()
    for L in sorted({k - 1 if k > 1 else 1, 1, k}):
        assert (po.encrypt_zero_asymmetric(pk, seed, 2, L=L) == rc.encrypt_zero_asymmetric(L=L)).all(), L


@needs_ref
@pytest.mark.parametrize("prng", [1, 2])
def test_seeded_kswitch_keys_expand_like_the_reference(prng):
    """KeyGenerator::create_relin_keys() / create_galois_keys() objects are seeded: every member carries c_0 and the seed of c_1,
    which KSwitchKeys::load expands at the key level.  The restatement's expansion at the key level gives the reference's c_1 of
    every digit, for either prng_type (shake256: the members retyped), uncompressed and zlib-compressed."""
    n, bits = 4096, [40, 40, 40, 40]
    mods, rc, oc, po = _setup("ckks", n, bits, P.BLAKE2XB)
    k = len(mods)
    elt = O.galois_elt_from_step(n, 1)
    for galois_elt, index in ((0, 0), (elt, (elt - 1) // 2)):
        raw = P.kswitch_with_prng_type(rc.seeded_kswitch_keys_stream(galois_elt), prng)
        key = rc.kswitch_keys_load(raw, index)
        assert key.shape == (k - 1, 2, k, n)
        assert (rc.kswitch_keys_load(P.zlib_stream(raw), index) == key).all()
        members = P.kswitch_members(raw, index)
        assert len(members) == k - 1
        for j, (off, info) in enumerate(members):
            assert info.seeded == prng and info.data_words == k * n
            seed = np.frombuffer(raw, dtype=np.uint64, count=8, offset=off + info.seed_offset)
            c0 = np.frombuffer(raw, dtype=np.uint64, count=k * n, offset=off + info.data_offset).reshape(k, n)
            assert (key[j, 0] == c0).all()
            assert (po.expand_seed(k, seed, prng) == key[j, 1]).all(), (galois_elt, j)
