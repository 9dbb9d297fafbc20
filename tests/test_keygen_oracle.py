"""CPU: the Python restatement of KeyGenerator's public and key-switching keys (tests/keygen_ref.py: key-level symmetric
encryptions of zero in NTT form plus (q_{k-1} mod q_j) s'_j on row j of digit j) against the reference's create_public_key /
create_relin_keys / create_galois_keys({elt}) under a seeded Blake2xbPRNGFactory and a seeded Shake256PRNGFactory, for BFV, CKKS
and BGV at small n.  The GPU tests hold the device to the same keys."""
import numpy as np
import pytest

import keygen_ref as K
import oracle as O
import refprng as P
import refseal as R

needs_ref = pytest.mark.skipif(not (K.ref_available() and P.ref_available()),
                               reason="oracle/_ref/libsealref_{keygen,prng}.so not present")


def setup(scheme, n, bits, prng, seed=0x6B67):
    mods = R.coeff_modulus_create(n, bits)
    t = R.plain_modulus_batching(n, 20) if scheme != O.CKKS else 0
    rk = K.RefKeygen(scheme, n, mods, t, seed=seed, prng=prng)
    return rk, K.KeygenOracle(scheme, n, mods, t), rk.secret_key()


@needs_ref
@pytest.mark.parametrize("prng", [P.BLAKE2XB, P.SHAKE256])
@pytest.mark.parametrize("scheme", [O.BFV, O.CKKS, O.BGV])
@pytest.mark.parametrize("n,bits", [(256, [30, 30, 40]), (512, [60, 60, 60, 60])])
def test_restatement_matches_reference(scheme, prng, n, bits):
    rk, ko, sk = setup(scheme, n, bits, prng)
    seeds = rk.boot_seeds(rk.k - 1)
    assert (ko.public_key(sk, seeds[0], prng) == rk.public_key()).all()
    # relinearization, a positive and a negative step, the column / conjugate element
    for elt in (0, 3, pow(3, n // 2 - 1, 2 * n), 2 * n - 1):
        want = rk.kswitch_key(elt)
        assert want.shape == (rk.k - 1, 2, rk.k, n)
        assert (ko.kswitch_key(sk, elt, seeds, prng) == want).all(), f"galois_elt {elt}"


@needs_ref
def test_factor_term_is_what_makes_the_key():
    """without the (q_{k-1} mod q_j) s'_j term every digit would be a plain encryption of zero: the term sits on row j of digit j
    only, and the rows it does not touch equal the public key's (same bootstrap seed, same level)"""
    rk, ko, sk = setup(O.CKKS, 256, [30, 30, 30, 40], P.BLAKE2XB)
    pk, key = rk.public_key(), rk.kswitch_key(0)
    for j in range(rk.k - 1):
        assert (key[j, 1] == pk[1]).all()
        for i in range(rk.k):
            assert (key[j, 0, i] == pk[0, i]).all() == (i != j)


def test_galois_table_matches_the_rotation_tables():
    """the restated NTT-form Galois table is a permutation, the identity for elt 1, and composes as the group does"""
    n = 64
    assert (K.galois_table_ntt(n, 1) == np.arange(n)).all()
    for elt in (3, 5, 2 * n - 1):
        t = K.galois_table_ntt(n, elt)
        assert sorted(t) == list(range(n))
    a, b = K.galois_table_ntt(n, 3), K.galois_table_ntt(n, 5)
    assert (a[b] == K.galois_table_ntt(n, 15)).all() or (b[a] == K.galois_table_ntt(n, 15)).all()
