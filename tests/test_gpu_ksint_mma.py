"""The product step of the integer key-switching path on the INT8 tensor cores (-m gpu; ks32_mac_mma in
seal_b200/csrc/sb_ksint.cu).  It splits every 29-bit word into four u8 limbs and sums the limb-pair products in s32 class
accumulators; the words it writes must be the integer-pipe kernels' words, bit for bit, for every input, including the
words that make the class sums largest (p - 1, and low limbs all 0xFF)."""
import numpy as np
import pytest

import oracle as O

pytestmark = pytest.mark.gpu


def sb():
    import seal_b200

    return seal_b200


def words(rng, primes, shape, kind):
    """[S][*shape] canonical residues modulo each auxiliary prime"""
    out = np.empty((len(primes),) + shape, dtype=np.uint32)
    for t, p in enumerate(primes):
        if kind == "random":
            out[t] = rng.integers(0, p, shape, dtype=np.uint32)
        elif kind == "max":
            out[t] = p - 1
        else:  # low three limbs 0xFF, a random top limb that keeps the word below p
            out[t] = (rng.integers(0, p >> 24, shape, dtype=np.uint32) << 24) | 0xFFFFFF
    return out


@pytest.fixture(scope="module")
def ctx():
    S = sb()
    n = 4096  # the deepest levels the integer path takes (64 digits) exist at this size only
    return S.Context(S.CKKS, n, O.coeff_modulus_create(n, [50, 50, 51]))


# L: 3 .. 32 digits run on the tensor cores (one K step; L = 32: nine output tiles, no zero digit), 33 .. 63 take the integer-pipe
# kernels; B: ragged tiles of 16, and chunks below 16 ciphertexts, which take the integer-pipe kernels
@pytest.mark.parametrize("kind", ["random", "max", "ff"])
@pytest.mark.parametrize("L,B", [(3, 140), (8, 1), (8, 15), (8, 16), (8, 17), (31, 1), (31, 17), (31, 40), (32, 17), (33, 16),
                                 (41, 16), (63, 15)])
def test_product_kernels_word_identical(ctx, kind, L, B):
    primes = ctx.ksint_primes()
    S, n = len(primes), ctx.n
    rng = np.random.default_rng(1000 * L + B)
    dh = words(rng, primes, (L, B, n), kind)
    key = words(rng, primes, (L, 2, L + 1, n), kind)
    acc_int, ran_int = ctx.ksint_product(dh, key, 0)
    acc_mma, ran_mma = ctx.ksint_product(dh, key, 1)
    assert ran_int in (0, 1)
    assert ran_mma == (2 if L <= 32 and B >= 16 else ran_int), "the tensor-core kernel runs for L <= 32 digits, B >= 16"
    assert np.array_equal(acc_mma, acc_int), "tensor-core and integer-pipe products differ"
    # numpy: the exact sums (< L p^2 < 2^64) modulo p_t on the first 128 coefficients; the kernels leave values in [0, 2p)
    xs = slice(0, 128)
    for t, p in enumerate(primes):
        d = dh[t][:, :, xs].astype(np.uint64)  # [L][B][x]
        k = key[t][..., xs].astype(np.uint64)  # [L][2][L+1][x]
        ref = np.zeros((B, 2, L + 1, 128), dtype=np.uint64)
        for J in range(L):
            ref += d[J][:, None, None, :] * k[J][None]
        got = acc_mma[:, :, :, t, xs]
        assert (got < 2 * p).all()
        assert np.array_equal(got.astype(np.uint64) % np.uint64(p), ref % np.uint64(p)), f"prime {p}"


def test_product_rejects_levels_past_max_digits(ctx):
    primes = ctx.ksint_primes()
    L = 65
    dh = np.zeros((len(primes), L, 1, ctx.n), dtype=np.uint32)
    key = np.zeros((len(primes), L, 2, L + 1, ctx.n), dtype=np.uint32)
    with pytest.raises(ValueError):
        ctx.ksint_product(dh, key, 1)


def _rand_ct(rng, mods, batch, parts, L, n):
    return np.stack([np.stack([np.stack([rng.integers(0, mods[i], n, dtype=np.uint64) for i in range(L)])
                               for _ in range(parts)]) for _ in range(batch)])


def test_headline_shape_relinearize_and_rotation_same_words(monkeypatch):
    """the headline shape (n = 65536, 32 primes), device-resident, three key-switching chunks with a ragged tail (17, 17, 3), with
    the tensor-core product and without it: relinearize and one rotation give identical words.  The profile's integer
    multiply-accumulate counter shows which kernels ran: with the tensor cores only the 3-ciphertext chunk takes the integer-pipe
    kernels"""
    import torch

    S = sb()
    n = 65536
    mods = O.coeff_modulus_create(n, [55] * 32)
    k, L = len(mods), len(mods) - 1
    rng = np.random.default_rng(65536)
    key = np.stack([np.stack([np.stack([rng.integers(0, mods[i], n, dtype=np.uint64) for i in range(k)]) for _ in range(2)])
                    for _ in range(L)])
    batch = 37
    c3 = torch.from_numpy(_rand_ct(rng, mods, batch, 3, L, n).view(np.int64)).cuda()
    c2 = c3[:, :2].contiguous()
    elt = O.galois_elt_from_step(n, 1)
    got, macs32 = {}, {}
    for mma in ("0", "1"):
        monkeypatch.setenv("SB200_KS_MAC_MMA", mma)
        ctx = S.Context(S.CKKS, n, mods)
        rk = ctx.load_key(key)
        ctx.set_limit(ctx.LIMIT_KS_ALGORITHM, 2)
        ctx.set_limit(ctx.LIMIT_KS_CHUNK, 17)
        S5 = len(ctx.ksint_primes())
        rel, rot = torch.empty_like(c2), torch.empty_like(c2)
        ctx.profile(True)
        ctx.d_relinearize(c3, rk, rel, L, batch)
        torch.cuda.synchronize()
        macs32[mma] = sum(r[7] for r in ctx.profile_read_work32() if r[0] == "ks32_mac")
        ctx.profile(False)
        ctx.d_apply_galois(c2, elt, rk, rot, L, batch)
        torch.cuda.synchronize()
        got[mma] = (rel.cpu(), rot.cpu())
        del rk, ctx
    per_ct = 2.0 * (L + 1) * L * S5 * n  # integer multiply-accumulates of one ciphertext's products
    assert macs32["0"] == 37 * per_ct and macs32["1"] == 3 * per_ct, macs32
    assert torch.equal(got["0"][0], got["1"][0]), "relinearize: tensor-core product differs"
    assert torch.equal(got["0"][1], got["1"][1]), "apply_galois: tensor-core product differs"
