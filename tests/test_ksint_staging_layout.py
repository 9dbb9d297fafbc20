"""Shared-memory access patterns of the linear row buffers of the 32-bit local passes (ks32_local in sb_ksint.cu).  A row's
4096-word block arrives and leaves by bulk copies, so its buffer holds the words in order; the first pass of the forward transform
and the last pass of the inverse access it as tid + 256 e, the other two ends as 16 consecutive words per lane in four 16-byte
groups, visited in the order h ^ hx (hx = (tid >> 1) & 3).  The exchanges between passes use the swizzled tile checked by
test_host_logic.py::test_ksint_swizzle_conflict_free."""


def _hx(t):
    return (t >> 1) & 3


def test_linear_lane_pattern_conflict_free():
    """tid + 256 e: 32 distinct banks per warp-wide 4-byte access, and every word of the block exactly once"""
    seen = []
    for warp in range(8):
        tids = [warp * 32 + l for l in range(32)]
        for e in range(16):
            words = [t + 256 * e for t in tids]
            assert len({w % 32 for w in words}) == 32
            seen += words
    assert sorted(seen) == list(range(4096))


def test_linear_group_pattern_conflict_free():
    """16 tid + 4 (h ^ hx): 8 distinct 16-byte bank groups per quarter-warp for each h, every lane visits its own four groups once,
    and the block is covered exactly once"""
    seen = []
    for t in range(256):
        groups = [16 * t + 4 * (h ^ _hx(t)) for h in range(4)]
        assert sorted(groups) == [16 * t + 4 * h for h in range(4)]
        seen += [w + i for w in groups for i in range(4)]
    assert sorted(seen) == list(range(4096))
    for q in range(32):
        grp = range(8 * q, 8 * q + 8)
        for h in range(4):
            assert len({((16 * t + 4 * (h ^ _hx(t))) // 4) % 8 for t in grp}) == 8


def test_xor_groups_is_the_visit_order():
    """xor_groups: a conditional swap of groups (0,1), (2,3) by bit 0 of x, then of (0,2), (1,3) by bit 1, puts group h ^ x at h --
    what the stores of the forward pass need and what undoes the loads of the inverse pass"""
    for x in range(4):
        a = list(range(4))
        if x & 1:
            a[0], a[1], a[2], a[3] = a[1], a[0], a[3], a[2]
        if x & 2:
            a[0], a[1], a[2], a[3] = a[2], a[3], a[0], a[1]
        assert a == [h ^ x for h in range(4)]
