"""The bin-to-lane assignment of k_front11a's half-warps WITHOUT a GPU (front_bin / front_pair of sora_b200/csrc/rx11a_kernels.cuh,
restated here): each of the 16 lanes of a half owns four bins, every bin of the 64 exactly once, the pilots in bin 0 of lanes 12-15 in
the order the tracker's width-16 shuffles read them, and the data bins as the (d, d + 3) pairs whose 64-QAM soft bits the kernel stores
as six 16-bit words."""
from test_cpu_packed_rot import _data_bin, _deint_inverse

def front_pair(hl, p):
    q = hl + 12 * p
    return 6 * (q // 3) + q % 3

def front_bin(hl, i):
    if hl < 12:
        return _data_bin(front_pair(hl, i >> 1) + 3 * (i & 1))
    j = hl - 12; m = 3 * j + i - 1
    return ((0x1507392B >> (8 * j)) & 0xFF) if i == 0 else (26 + m if m else 0)

def test_every_bin_once_per_half():
    bins = [front_bin(hl, i) for hl in range(16) for i in range(4)]
    assert sorted(bins) == list(range(64))
    assert [front_bin(hl, 0) for hl in range(12, 16)] == [43, 57, 7, 21]
    # bins 1-3 of lanes 12-15 are the zero bins, which the tracker leaves unrotated
    assert sorted(front_bin(hl, i) for hl in range(12, 16) for i in range(1, 4)) == [0] + list(range(27, 38))
    # every data bin is a subcarrier in -26..-1, 1..26 (rotated), none of the zero bins is
    k = lambda b: b if b < 32 else b - 64
    assert all(k(front_bin(hl, i)) != 0 and abs(k(front_bin(hl, i))) <= 26 for hl in range(12) for i in range(4))
    assert not any(k(front_bin(hl, i)) != 0 and abs(k(front_bin(hl, i))) <= 26 for hl in range(12, 16) for i in range(1, 4))

def test_64qam_pairs_of_the_half_warp_lanes():
    # the 24 pairs of lanes 0-11 are all the d in 0..47 with d % 6 < 3, and bit i of d lands at an even position with bit
    # (2 0 1 5 3 4)[i] of d + 3 right after it
    ds = sorted(front_pair(hl, p) for hl in range(12) for p in range(2))
    assert ds == [d for d in range(48) if d % 6 < 3]
    inv = _deint_inverse(288, 6); sigma = (2, 0, 1, 5, 3, 4)
    for d in ds:
        for i in range(6):
            assert inv[6 * d + i] % 2 == 0 and inv[6 * (d + 3) + sigma[i]] == inv[6 * d + i] + 1, (d, i)
