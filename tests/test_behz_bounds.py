"""The 128-bit sums of BFV multiplication, in Python integers (no GPU).

behz_lift_kernel and behz_floor_sk_kernel (seal_b200/csrc/sb_bfv.cu) compute the three FastBConv dot products of the BEHZ steps as
unreduced 128-bit sums and reduce once at the end:
  q -> Bsk   sum_{i < L}  t_i ((q / q_i) mod P),    t_i < q_i    (the lift, rns.cpp:1086-1131, and fast_floor, :1041-1084)
  B -> q_j   sum_{i < |B|} t_i ((B / B_i) mod q_j), t_i < B_i    (fastbconv_sk, rns.cpp:932-976)
  B -> m_sk  sum_{i < |B|} t_i ((B / B_i) mod m_sk)                (the same, for the Shenoy-Kumaresan correction)
Coefficient primes and the auxiliary 61-bit primes are below 2^61, so every term is below 2^122 and at most 64 terms cannot wrap.
The library rejects BFV multiplication at levels whose base B would hold more than 64 primes (check_bfv_multiply_level).  These
tests restate the auxiliary base, check the worst cases of all three sums at every level the library accepts, and show that the
limit is needed: without it the B -> m_sk sum reaches 2^128 at a level whose shared memory still fits."""
import pytest

import oracle as O
from common import ntt_primes_below, product

MAX_BASE = 64  # kBfvMultiplyMaxBase (seal_b200/csrc/sb_engine.cuh)
WORD_MAX = (1 << 61) - 1  # the largest word below 2^61: any coefficient prime is at most this
SMEM_OPTIN = 232448  # bytes of dynamic shared memory a block may opt into on H100 (227 KB)
THREADS = 128  # kBehzThreads


def aux_list(n, count):
    """[m_sk, gamma, B_0, B_1, ...]: 61-bit primes = 1 mod 2n, largest first (rns.cpp:626-632)"""
    return ntt_primes_below(61, n, count)


def base_size(q, L, t):
    """|B| of the level with the first L primes of q: L, plus one prime when K n t q^2 < q prod(B) m_sk needs it
    (rns.cpp:605-612)"""
    return L + 1 if 32 + t.bit_length() + product(q[:L]).bit_length() >= 61 * L + 61 else L


def bsk(n, q, L, t):
    nB = base_size(q, L, t)
    aux = aux_list(n, nB + 2)
    return aux[2:2 + nB] + [aux[0]]


def sk_to_msk_worst(B, m_sk):
    """sum_i (B_i - 1) ((B / B_i) mod m_sk): the B -> m_sk sum with every t_i at its largest value"""
    total = 0
    for i, b in enumerate(B):
        rest = 1
        for j, c in enumerate(B):
            if j != i:
                rest = rest * c % m_sk
        total += (b - 1) * rest
    return total


@pytest.mark.parametrize("n", [2, 1024, 4096, 32768])
def test_auxiliary_base_vs_oracle(n):
    """the restated auxiliary list and |B| rule equal the oracle's base Bsk at every level up to 64 primes, for a small, a 60-bit
    and a power-of-two plain modulus"""
    assert aux_list(n, 8) == O.get_primes(2 * n, 61, 8)
    for bits in ([60] * 64, [30] * 64):
        q = O.coeff_modulus_create(n, bits)
        for t in (65537, 1 << 59, ntt_primes_below(60, n, 1)[0]):
            for L in range(1, 65):
                assert bsk(n, q, L, t) == O.behz_base(n, q[:L], t), (n, bits[0], t, L)


@pytest.mark.parametrize("L", [1, 2, 3])
def test_base_size_rule_both_sides(L):
    """n = 4096, 60-bit primes: a plain modulus of b* = 61 L + 61 - 32 - bits(Q_L) bits enlarges B by one prime, one of b* - 1
    bits does not (the smallest margin of the rule)"""
    n = 4096
    q = O.coeff_modulus_create(n, [60] * 4)
    b_star = 61 * L + 61 - 32 - product(q[:L]).bit_length()
    assert 2 <= b_star - 1 and b_star <= 60, b_star
    for bits, want in ((b_star, L + 1), (b_star - 1, L)):
        t = (1 << (bits - 1)) + 1
        assert base_size(q, L, t) == want and len(O.behz_base(n, q[:L], t)) == want + 1, (L, bits)


@pytest.mark.parametrize("logn", range(1, 18))
def test_fastbconv_sums_below_2_128_at_every_accepted_level(logn):
    """for every |B| <= 64 (every level BFV multiplication accepts: |B| is L or L + 1), the worst case of each dot product is
    below 2^128; the coefficient primes are any words below 2^61"""
    n = 1 << logn
    aux = aux_list(n, MAX_BASE + 2)
    m_sk = aux[0]
    for nB in range(1, MAX_BASE + 1):
        B = aux[2:2 + nB]
        P_max = max(B + [m_sk])
        L = nB  # the longest level with this base
        lift = L * (WORD_MAX - 1) * (P_max - 1)
        sk_q = sum(b - 1 for b in B) * (WORD_MAX - 1)
        sk_m = sk_to_msk_worst(B, m_sk)
        for name, s in (("q -> Bsk", lift), ("B -> q", sk_q), ("B -> m_sk", sk_m)):
            assert s < 2 ** 128, f"n = {n}, |B| = {nB}: the {name} sum reaches {s / 2 ** 128:.4f} * 2^128"
    assert lift >= 2 ** 127.9 and sk_q >= 2 ** 127.9, "at |B| = 64 the term-count bound is nearly tight"


def test_sk_to_msk_sum_wraps_without_the_limit():
    """n = 512 and |B| = 110 (a level of 110 primes of 60 bits): the B -> m_sk worst case reaches 2^128 while the floor kernel's
    shared memory still fits, so neither the shared memory nor the constants would have stopped a silent wrap"""
    n, nB = 512, 110
    q = O.coeff_modulus_create(n, [60] * 40) + ntt_primes_below(59, n, 70)
    assert len(set(q)) == nB and base_size(q, nB, 65537) == nB
    aux = aux_list(n, nB + 2)
    s = sk_to_msk_worst(aux[2:2 + nB], aux[0])
    assert s >= 2 ** 128, f"the B -> m_sk sum at |B| = {nB} is {s / 2 ** 128:.4f} * 2^128"
    L, nS = nB, nB + 1
    smem = (max(L, nS) + nS) * THREADS * 8  # behz_floor_sk_kernel
    assert smem <= SMEM_OPTIN, smem
