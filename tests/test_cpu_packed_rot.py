"""The per-bin path of k_front11a behind the FFT WITHOUT a GPU: the rotation-factor and hand-over helpers of sora_b200/csrc/fixed.cuh
against the scalar primitives they replace (tests/cpp/packed_rot_emu.cpp compiles the header for the host), and the properties of the
802.11a tables the kernel's bin-to-lane mapping and 16-bit soft-bit stores rely on.  The device build is checked bit for bit by the GPU
tests of the 802.11a receive chain (stage taps, all rates, channels, rails)."""
import ctypes as C, itertools, os, shutil, subprocess
import numpy as np, pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "packed_rot_emu.cpp"); CSRC = os.path.join(ROOT, "sora_b200", "csrc")

EDGES = np.array([-32768, -32767, -16385, -16384, -8193, -8192, -2049, -2048, -129, -128, -1, 0, 1, 127, 128, 2047, 2048, 8191, 8192,
                  16383, 16384, 32766, 32767], np.int64)
ROT_EDGES = EDGES[EDGES > -32768]                     # rotation-table halves are round(32767 cos / sin): never -32768

def words(re, im):
    return ((np.asarray(re, np.int64) & 0xFFFF) | ((np.asarray(im, np.int64) & 0xFFFF) << 16)).astype(np.uint32)

@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no host compiler")
    so = str(tmp_path_factory.mktemp("packed_rot_emu") / "packed_rot_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-DSB_HOST_EMU", "-I", CSRC, "-o", so, SRC])
    L = C.CDLL(so); P = C.c_void_p
    L.packed_rot.argtypes = [C.c_int, P, P, P, C.c_uint32, P, P]
    L.turn.argtypes = [P, C.c_uint32, P, P]
    return L

def _check(got, want, what):
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%s: %d mismatches, first at %d: got %08x want %08x" % (what, bad.size, bad[0], got[bad[0]], want[bad[0]])

def _rot_words(rng, n):
    """Random rotation-table-like words plus every table word (the host formula of tables.cuh, P = 3.141593)."""
    ph = 2 * 3.141593 * np.arange(65536) / 65536
    lround = lambda v: (np.sign(v) * np.floor(np.abs(v) + 0.5)).astype(np.int64)
    table = words(lround(32767.0 * np.cos(ph)), -lround(32767.0 * np.sin(ph)))
    return np.concatenate([words(rng.integers(-32767, 32768, n), rng.integers(-32767, 32768, n)), table])

@pytest.mark.parametrize("op,name", [(0, "rotation product"), (1, "equalise + phase compensation")])
def test_rotation_products(lib, op, name):
    rng = np.random.default_rng(30 + op)
    w = _rot_words(rng, 1 << 19)
    n = w.size
    a = words(rng.integers(-32768, 32768, n), rng.integers(-32768, 32768, n))
    ch = words(rng.integers(-32768, 32768, n), rng.integers(-32768, 32768, n))
    # every combination of the int16 edges for the data word and the channel, rotation halves at their edges
    g = np.array(list(itertools.product(EDGES, EDGES, ROT_EDGES, ROT_EDGES)), np.int64)
    a = np.concatenate([a, words(g[:, 0], g[:, 1])]); w = np.concatenate([w, words(g[:, 2], g[:, 3])])
    ch = np.concatenate([ch, words(g[:, 1], g[:, 0])])
    b, c = (w, w) if op == 0 else (ch, w)
    arrs = [np.ascontiguousarray(v, np.uint32) for v in (a, b, c)]
    got = np.zeros(a.size, np.uint32); want = np.zeros(a.size, np.uint32)
    lib.packed_rot(op, *[v.ctypes.data for v in arrs], a.size, got.ctypes.data, want.ctypes.data)
    _check(got, want, name)

def test_turn_pi_every_angle(lib):
    th = np.arange(-32768, 32768, dtype=np.int32)
    got = np.zeros(2 * th.size, np.int32); want = np.zeros(2 * th.size, np.int32)
    lib.turn(th.ctypes.data, th.size, got.ctypes.data, want.ctypes.data)
    _check(got.view(np.uint32), want.view(np.uint32), "turn_pi")

def _deint_inverse(ncbps, nbpsc):
    """inv[j] = coded-bit position k of received bit j (gen_deint_map of tables.cuh, inverted as sb200.cu uploads it)."""
    s = max(nbpsc // 2, 1); inv = [0] * ncbps
    for k in range(ncbps):
        i = (ncbps // 16) * (k % 16) + k // 16
        inv[s * (i // s) + (i + ncbps - (16 * i) // ncbps) % s] = k
    return inv

def _data_bin(d):
    return 38 + d + (d >= 5) + (d >= 18) if d < 24 else d - 23 + (d >= 30) + (d >= 43)

def test_lane_bins_and_64qam_pairs():
    # lanes 0-23 own data subcarriers d0 = 6 (l / 3) + l % 3 and d0 + 3, lanes 24-27 the pilots, the rest the zero bins: every bin once
    bins = []
    for l in range(32):
        j = l - 24
        if l < 24:
            d0 = 6 * (l // 3) + l % 3; bins += [_data_bin(d0), _data_bin(d0 + 3)]
        else:
            bins += [((0x1507392B >> (8 * j)) & 0xFF) if j < 4 else (0 if j == 4 else 22 + j), 30 + j]
    assert sorted(bins) == list(range(64))
    assert [bins[2 * l] for l in range(24, 28)] == [43, 57, 7, 21]
    assert sorted(_data_bin(d) for d in range(48)) == [b for b in range(1, 64) if not 27 <= b <= 37 and b not in (7, 21, 43, 57)]
    # at 64-QAM bit i of d0 lands at an even position and bit (2 0 1 5 3 4)[i] of d0 + 3 right after it (the six 16-bit stores)
    inv = _deint_inverse(288, 6); sigma = (2, 0, 1, 5, 3, 4)
    for l in range(24):
        d0 = 6 * (l // 3) + l % 3
        for i in range(6):
            assert inv[6 * d0 + i] % 2 == 0 and inv[6 * (d0 + 3) + sigma[i]] == inv[6 * d0 + i] + 1, (l, i)

def test_pilot_average_ranges():
    # avg = (th1 + th2 + th3 + th4) / 4 and del = ((th3 - th1) / 28 + (th4 - th2) / 28) >> 1 (C truncation) stay in int16 for int16 angles
    def tdiv(a, b): return int(a / b)
    for t in itertools.product((-32768, -32767, 0, 32767), repeat=4):
        avg = tdiv(sum(t), 4); dl = (tdiv(t[2] - t[0], 28) + tdiv(t[3] - t[1], 28)) >> 1
        assert -32768 <= avg <= 32767 and -32768 <= dl <= 32767
