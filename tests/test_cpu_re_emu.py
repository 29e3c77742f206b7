"""The four-lanes-per-code-block Viterbi kernel (k_viterbi_re, sora_b200/csrc/viterbi_k7_re.cuh) WITHOUT a GPU: its device source is
compiled for the host by tests/cpp/re_emu.cpp (the CUDA intrinsics in tests/cpp/warp_emu.h; the 32 lanes of a CTA run as 32 threads, and
every quad shuffle, __syncwarp and warp vote is a real exchange) and compared with the CPU oracle, bit for bit: clean and noisy code
words, wrap-around garbage, every traceback window size, code blocks of different lengths side by side, and code blocks that run out of whole
6-step chunks while a neighbour in the warp still has some (802.11n symbols).  Four lanes per code block, eight code blocks per warp: the
kernel the library runs below 16 384 code blocks."""
import ctypes as C, os, shutil, subprocess
import numpy as np, pytest
import oracle_py
from test_cpu_lane_emu import CR_12, CR_23, CR_34, N11N, _coded, check_ragged

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "re_emu.cpp"); CSRC = os.path.join(ROOT, "sora_b200", "csrc")
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="no host compiler")

def build_emu(tmp_path_factory):
    """Compile the emulator into a temporary directory; returns run(soft, cr, L, depth, look, lens=, nsofts=) -> (bytes, nraw)."""
    so = str(tmp_path_factory.mktemp("re_emu") / "re_emu.so")
    subprocess.check_call(["g++", "-O1", "-std=c++20", "-pthread", "-shared", "-fPIC", "-DSB_HOST_EMU", "-Wno-unknown-pragmas", "-I", CSRC, "-o", so, SRC])
    lib = C.CDLL(so)
    lib.re_emu_viterbi.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64,
                                   C.c_void_p, C.c_void_p, C.c_void_p]
    lib.re_emu_viterbi.restype = C.c_int
    def run(soft, cr, L, depth=256, look=24, lens=None, nsofts=None):
        soft = np.ascontiguousarray(soft, dtype=np.uint8); nb, ns = soft.shape
        stride = (ns + 15) // 16 * 16 + 16                              # the kernel fetches whole chunks: rows padded like the library's soft rows
        sp = np.zeros((nb, stride), np.uint8); sp[:, :ns] = soft
        ostride = L + 2 + 14
        out = np.zeros((nb, ostride), np.uint8); nraw = np.zeros(nb, np.uint32)
        lp = np.ascontiguousarray(lens, dtype=np.uint32) if lens is not None else None
        npp = np.ascontiguousarray(nsofts, dtype=np.uint32) if nsofts is not None else None
        rc = lib.re_emu_viterbi(sp.ctypes.data, stride, ns, nb, cr, L, depth, look, out.ctypes.data, ostride, nraw.ctypes.data,
                                lp.ctypes.data if lp is not None else None, npp.ctypes.data if npp is not None else None)
        assert rc == 0
        return out[:, :L + 2], nraw
    return run

@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build_emu(tmp_path_factory)

def test_code_words_clean_and_noisy(emu):
    rng = np.random.default_rng(3)
    for cr, rate in ((CR_12, (1, 2)), (CR_23, (2, 3)), (CR_34, (3, 4))):
        L = 300
        bits, coded = _coded(rng, 9, L, rate)
        for flip in (0.0, 0.06, 0.5):
            soft = np.where(coded > 0, rng.integers(5, 8, coded.shape), rng.integers(0, 3, coded.shape)).astype(np.uint8)
            soft = np.where(rng.random(coded.shape) < flip, rng.integers(0, 8, coded.shape), soft).astype(np.uint8)
            g, nraw = emu(soft, cr, L)
            assert (g == oracle_py.viterbi_blocks(soft, cr, L)).all(), (cr, flip)
            assert (nraw == L + 2).all()
            if flip == 0.0:
                assert (np.unpackbits(g, axis=1, bitorder="little")[:, :8 * L + 16] == bits[:, :8 * L + 16]).all()

def test_wrap_and_windows(emu):
    """Wrap-around garbage (all 7, all 0, alternating extremes, uniform noise) at short and long windows, lookahead 0 and at the limit,
    with nsoft a few groups past the flush point and a trailing partial group."""
    rng = np.random.default_rng(11)
    for cr, per, steps_per in ((CR_12, 2, 1), (CR_23, 3, 2), (CR_34, 4, 3)):
        for L in (1, 2, 17, 101):
            ngroups = -(-(8 * L + 22) // steps_per) + int(rng.integers(0, 5))
            ns = ngroups * per + int(rng.integers(0, per))
            pats = [rng.integers(0, 8, (4, ns)), np.full((1, ns), 7), np.zeros((1, ns), int), np.tile([0, 7, 7, 0, 7], ns)[None, :ns], rng.integers(3, 5, (2, ns))]
            soft = np.concatenate(pats).astype(np.uint8)
            for depth, look in ((256, 24), (192, 36), (8, 0), (16, 7), (64, 280 - 64), (256, 24)):
                g, _ = emu(soft, cr, L, depth, look)
                o = oracle_py.viterbi_blocks(soft, cr, L, depth, look)
                assert (g == o).all(), (cr, L, depth, look, np.argwhere(g != o)[:4])

def test_blocks_of_different_lengths_side_by_side(emu):
    """The receive chains hand every code block its own length and soft-byte count (FrameInfo): 37 blocks whose triggers and ends fall at
    different times; a short input (a truncated frame) among them decodes what it has, exactly the bytes the oracle produces."""
    rng = np.random.default_rng(5)
    for cr, per, steps_per in ((CR_12, 2, 1), (CR_23, 3, 2), (CR_34, 4, 3)):
        lens = np.array([1 + (37 * i) % 211 for i in range(37)], np.uint32)
        nsofts = np.array([-(-(8 * int(L) + 22) // steps_per) * per for L in lens], np.uint32)
        nsofts[7] = nsofts[7] // (2 * per) * per                          # truncated: half of the soft values of block 7 are missing
        ns = int(nsofts.max())
        soft = rng.integers(0, 8, (37, ns)).astype(np.uint8)
        g, nraw = emu(soft, cr, int(lens.max()), lens=lens, nsofts=nsofts)
        for i in range(37):
            L = int(lens[i]); n = int(nsofts[i])
            o, k = oracle_py.viterbi_blocks_n(soft[i:i + 1, :n], cr, L)
            assert nraw[i] == k[0] and (i == 7 or k[0] == L + 2), (cr, i, nraw[i], k[0], L)
            assert (g[i, :k[0]] == o[0, :k[0]]).all(), (cr, i, L)

@pytest.mark.parametrize("cr, ncbps", N11N)
def test_ragged_chunks_11n_symbols(emu, cr, ncbps):
    """A code block that runs out of whole 6-step chunks while a neighbour in its warp still has some must still decode its remaining
    whole groups and fire its last traceback window (802.11n frames: N_CBPS soft bytes per symbol, flush point in the last partial chunk)."""
    check_ragged(emu, cr, ncbps, 40 + ncbps + cr)

def test_ragged_chunks_two_blocks(emu):
    """L = 62 with 10 x 104 soft bytes beside L = 200 with 32 x 104 (rate 1/2, 802.11n window)."""
    rng = np.random.default_rng(62)
    soft = rng.integers(0, 8, (2, 32 * 104)).astype(np.uint8)
    lens = np.array([62, 200], np.uint32); nsofts = np.array([10 * 104, 32 * 104], np.uint32)
    g, nraw = emu(soft, CR_12, 200, 192, 36, lens=lens, nsofts=nsofts)
    for i in range(2):
        L = int(lens[i])
        assert nraw[i] == L + 2, "block %d L=%d: nraw %d, want %d" % (i, L, nraw[i], L + 2)
        assert (g[i, :L + 2] == oracle_py.viterbi_blocks(soft[i:i + 1, :nsofts[i]], CR_12, L, 192, 36)[0]).all(), i
