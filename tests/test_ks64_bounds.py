"""The 128-bit digit sums of the 64-bit key-switching path in Python integers (ks_mac_kernel / ks_local_mac_kernel,
seal_b200/csrc/sb_engine.cu).  A level of L digits adds L products of canonical words at output prime I, each at most
(q_I - 1)^2.  Below 2^60 that fits 128 bits for every level a context can have (L <= 255); the context accepts primes up to
2^61, where 65 products already wrap, so levels with L (q_max - 1)^2 >= 2^128 reduce the sums once every kKsSumWindow digits."""
from common import ntt_primes_below
from test_plain_sum_bounds import primes_below

WINDOW = 64  # kKsSumWindow (seal_b200/csrc/sb_engine.cu)
MAX_DIGITS = 255  # a context has at most 256 primes, the last one special


def window(q):
    """the largest w with a carried residue plus w products of words q - 1 below 2^128"""
    return (2**128 - 1 - (q - 1)) // (q - 1) ** 2


def worst(q, w, carry=True):
    return (q - 1) * carry + w * (q - 1) ** 2


def needs_window(qs, L):
    """ks_sum_needs_window: L (q_max - 1)^2 >= 2^128 over the L data primes and the special prime qs[-1]"""
    qmax = max(qs[:L] + [qs[-1]])
    return (qmax - 1) ** 2 > (2**128 - 1) // L


def test_window_values():
    """the window is 64 at the largest 61-bit primes and at least 64 at every prime below 2^61 (the context's bound), so one
    compile-time value serves every level; at 60 bits it is at least 255, more digits than any level has"""
    for n in (1024, 4096):
        for q in ntt_primes_below(61, n, 3):
            assert window(q) == WINDOW, (n, q)
    assert window(2**61 - 1) == WINDOW  # bounds every prime below 2^61
    for q in primes_below(2**60, 3) + [2**60 - 1]:
        assert window(q) >= MAX_DIGITS, q


def test_window_fits_and_one_more_overflows():
    """64 products plus a residue fit at the largest 61-bit primes, 65 products alone do not; 255 products of the largest 60-bit
    and 57-bit primes fit without any reduction"""
    for q in ntt_primes_below(61, 1024, 2) + ntt_primes_below(61, 4096, 2):
        assert worst(q, WINDOW) < 2**128
        assert worst(q, WINDOW + 1, carry=False) >= 2**128, q
    for bits in (57, 60):
        q = ntt_primes_below(bits, 1024, 1)[0]
        assert worst(q, MAX_DIGITS, carry=False) < 2**128, bits


def test_window_selection():
    """the levels that take the WINDOW instantiations: past 64 digits of the largest 61-bit primes, never at 60 bits or below"""
    q61 = ntt_primes_below(61, 1024, 256)
    assert not needs_window(q61, 64) and needs_window(q61[:66], 65) and needs_window(q61, 255)
    for bits in (57, 60):
        qs = ntt_primes_below(bits, 1024, 256)
        assert not needs_window(qs, 255), bits
    # one 61-bit prime among 60-bit ones: the largest prime decides
    q60 = ntt_primes_below(60, 1024, 255)
    assert needs_window(q60 + [q61[0]], 255) and not needs_window([q61[0]] + q60, 64)


def kernel_sum(q, xs, ks, reduce):
    """one 128-bit digit sum of the kernels, restated: products of canonical words, reduced every WINDOW digits when `reduce`,
    the accumulator kept to 128 bits as the hardware does"""
    acc = 0
    for J, (x, k) in enumerate(zip(xs, ks)):
        acc = (acc + x * k) % 2**128
        if reduce and (J + 1) % WINDOW == 0:
            acc %= q
    return acc % q


def test_windowed_sum_is_exact_and_the_unreduced_one_wraps():
    """the constant-digit extreme (every digit q_min - 1, every key word q_I - 1) at 65 and 255 digits of the largest 61-bit
    primes: the windowed sum is the exact one, the unreduced sum is not; at 64 digits both are exact"""
    for n in (1024, 4096):
        qs = ntt_primes_below(61, n, 256)
        qmin, q = min(qs), max(qs)
        for L in (64, 65, 255):
            xs, ks = [qmin - 1] * L, [q - 1] * L
            exact = L * (qmin - 1) * (q - 1) % q
            assert kernel_sum(q, xs, ks, True) == exact, (n, L)
            assert (kernel_sum(q, xs, ks, False) == exact) == (L <= WINDOW), (n, L)
