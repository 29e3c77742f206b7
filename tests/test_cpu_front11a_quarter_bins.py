"""The bin-to-lane assignment of k_front11a's quarter-warps WITHOUT a GPU (front_bin / front_pair / front_zero of
sora_b200/csrc/rx11a_kernels.cuh, restated here): each of the 8 lanes of a quarter owns eight bins, every bin of the 64 exactly once;
bins 0-5 of every lane are three (d, d + 3) data pairs whose 64-QAM soft bits the kernel stores as six 16-bit words, bin 6 holds the
pilots in lanes 0-3 in the order the tracker's width-8 shuffles read them, and the zero bins fill bin 6 of lanes 4-7 and bin 7."""
from test_cpu_packed_rot import _data_bin, _deint_inverse

def front_pair(ql, p):
    q = ql + 8 * p
    return 6 * (q // 3) + q % 3

def front_zero(m):
    return 26 + m if m else 0

def front_bin(ql, i):
    if i < 6:
        return _data_bin(front_pair(ql, i >> 1) + 3 * (i & 1))
    if i == 7:
        return front_zero(ql)
    return ((0x1507392B >> (8 * ql)) & 0xFF) if ql < 4 else front_zero(ql + 4)

def k(b):
    return b if b < 32 else b - 64

def test_every_bin_once_per_quarter():
    bins = [front_bin(ql, i) for ql in range(8) for i in range(8)]
    assert sorted(bins) == list(range(64))

def test_pilots_in_bin_6_of_lanes_0_to_3():
    # th1..th4 of the tracker are the shuffles from lanes 0, 1, 2, 3; 21 (sent negated) sits in lane 3
    assert [front_bin(ql, 6) for ql in range(4)] == [43, 57, 7, 21]

def test_rotated_bins():
    # the kernel rotates bins 0-5 of every lane and bin 6 of lanes 0-3: exactly the subcarriers -26..-1, 1..26
    rotated = [front_bin(ql, i) for ql in range(8) for i in range(8) if i < 6 or (i == 6 and ql < 4)]
    assert sorted(rotated) == sorted(b for b in range(64) if k(b) != 0 and abs(k(b)) <= 26)
    # and everything else is one of the twelve zero bins 0, 27..37
    zero = [front_bin(ql, 7) for ql in range(8)] + [front_bin(ql, 6) for ql in range(4, 8)]
    assert sorted(zero) == [0] + list(range(27, 38))

def test_data_bins_in_demapper_order():
    # bins 0-5 of every lane are data subcarriers; bin 2 p is d = front_pair(ql, p) and bin 2 p + 1 is d + 3
    for ql in range(8):
        for p in range(3):
            d = front_pair(ql, p)
            assert front_bin(ql, 2 * p) == _data_bin(d) and front_bin(ql, 2 * p + 1) == _data_bin(d + 3)

def test_64qam_pairs_of_the_quarter_warp_lanes():
    # the 24 pairs are all the d in 0..47 with d % 6 < 3, and bit i of d lands at an even position with bit (2 0 1 5 3 4)[i] of d + 3
    # right after it
    ds = sorted(front_pair(ql, p) for ql in range(8) for p in range(3))
    assert ds == [d for d in range(48) if d % 6 < 3]
    inv = _deint_inverse(288, 6); sigma = (2, 0, 1, 5, 3, 4)
    for d in ds:
        for i in range(6):
            assert inv[6 * d + i] % 2 == 0 and inv[6 * (d + 3) + sigma[i]] == inv[6 * d + i] + 1, (d, i)
