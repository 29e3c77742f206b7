"""The one-lane-per-code-block Viterbi kernel (sora_b200/csrc/viterbi_k7_lane.cuh) WITHOUT a GPU: its device source is compiled for the host
by tests/cpp/lane_emu.cpp (the CUDA intrinsics it uses are written out in C++ in tests/cpp/warp_emu.h; the 32 lanes of a CTA run as 32
threads and every warp vote is a real vote) and compared with the CPU oracle, bit for bit, on the cases the GPU tests use: clean and noisy
code words, wrap-around garbage, block lengths that end anywhere in the 6-step trellis phase / 8-step normalisation period / 6-column history
block, both traceback windows, code blocks of different lengths side by side (the receive chains' per-frame path), and code blocks that run
out of whole 6-step chunks while a neighbour in the warp still has some (802.11n symbols).  The GPU run of the same kernel is in
tests/test_gpu_rx11a.py and tests/test_gpu_zz_viterbi_ragged.py."""
import ctypes as C, os, shutil, subprocess
import numpy as np, pytest
import oracle_py
from sora_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "lane_emu.cpp"); CSRC = os.path.join(ROOT, "sora_b200", "csrc")
CR_12, CR_23, CR_34 = 0, 1, 2
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="no host compiler")

def build_emu(tmp_path_factory):
    """Compile the emulator into a temporary directory; returns run(soft, cr, L, depth, look, lens=, nsofts=) -> (bytes, nraw)."""
    so = str(tmp_path_factory.mktemp("lane_emu") / "lane_emu.so")
    subprocess.check_call(["g++", "-O1", "-std=c++20", "-pthread", "-shared", "-fPIC", "-DSB_HOST_EMU", "-Wno-unknown-pragmas", "-I", CSRC, "-o", so, SRC])
    lib = C.CDLL(so)
    lib.lane_emu_viterbi.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    lib.lane_emu_viterbi.restype = C.c_int
    def run(soft, cr, L, depth=256, look=24, lens=None, nsofts=None, hb=6):
        soft = np.ascontiguousarray(soft, dtype=np.uint8); nb, ns = soft.shape
        stride = (ns + 15) // 16 * 16 + 16                              # the kernel fetches whole chunks: rows padded like the library's soft rows
        sp = np.zeros((nb, stride), np.uint8); sp[:, :ns] = soft
        ostride = L + 2 + 14
        out = np.zeros((nb, ostride), np.uint8); nraw = np.zeros(nb, np.uint32)
        lp = np.ascontiguousarray(lens, dtype=np.uint32) if lens is not None else None
        npp = np.ascontiguousarray(nsofts, dtype=np.uint32) if nsofts is not None else None
        rc = lib.lane_emu_viterbi(sp.ctypes.data, stride, ns, nb, cr, L, depth, look, out.ctypes.data, ostride, nraw.ctypes.data,
                                  lp.ctypes.data if lp is not None else None, npp.ctypes.data if npp is not None else None, hb)
        assert rc == 0
        return out[:, :L + 2], nraw
    return run

@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build_emu(tmp_path_factory)

def _coded(rng, nblocks, L, rate):
    nbits = 8 * L + 16 + 6; nbits += (-nbits) % 48
    bits = rng.integers(0, 2, (nblocks, nbits)).astype(np.uint8); bits[:, 8 * L + 16:] = 0
    A, B = synth.conv_encode(bits)
    return bits, synth.puncture(A, B, rate)

HB = pytest.mark.parametrize("hb", (6, 8, 9))          # columns per history block: 6, 8, and 9 = 8 with the walk spread over the step loop

@HB
def test_code_words_clean_and_noisy(emu, hb):
    rng = np.random.default_rng(3)
    for cr, rate in ((CR_12, (1, 2)), (CR_23, (2, 3)), (CR_34, (3, 4))):
        L = 700
        bits, coded = _coded(rng, 5, L, rate)
        for flip in (0.0, 0.06, 0.5):
            soft = np.where(coded > 0, rng.integers(5, 8, coded.shape), rng.integers(0, 3, coded.shape)).astype(np.uint8)
            soft = np.where(rng.random(coded.shape) < flip, rng.integers(0, 8, coded.shape), soft).astype(np.uint8)
            g, nraw = emu(soft, cr, L, hb=hb)
            assert (g == oracle_py.viterbi_blocks(soft, cr, L)).all(), (cr, flip)
            assert (nraw == L + 2).all()
            if flip == 0.0:
                assert (np.unpackbits(g, axis=1, bitorder="little")[:, :8 * L + 16] == bits[:, :8 * L + 16]).all()

@HB
def test_wrap_and_ragged_stress(emu, hb):
    """tests/test_gpu_rx11a.py::test_viterbi_wrap_and_ragged_stress on the emulated kernel."""
    rng = np.random.default_rng(11)
    for cr, per in ((CR_12, 2), (CR_23, 3), (CR_34, 4)):
        steps_per = {2: 1, 3: 2, 4: 3}[per]
        for L in (1, 2, 3, 5, 17, 40, 101, 333, 1000):
            nbits = 8 * L + 16 + 6
            ngroups = -(-nbits // steps_per) + int(rng.integers(0, 5))
            ns = ngroups * per
            pats = [rng.integers(0, 8, (6, ns)), np.full((1, ns), 7), np.zeros((1, ns), int), np.tile([0, 7, 7, 0, 7], ns)[None, :ns], rng.integers(3, 5, (2, ns))]
            soft = np.concatenate(pats).astype(np.uint8)
            for depth, look in ((256, 24), (192, 36)):
                g, _ = emu(soft, cr, L, depth, look, hb=hb)
                o = oracle_py.viterbi_blocks(soft, cr, L, depth, look)
                assert (g == o).all(), (cr, L, depth, np.argwhere(g != o)[:4])

@HB
def test_blocks_of_different_lengths_side_by_side(emu, hb):
    """The receive chains hand every code block its own length and soft-byte count (FrameInfo): 37 blocks — a full warp and part of the next —
    whose triggers and ends fall at different times; a short input (a truncated frame) among them decodes what it has, like the oracle."""
    rng = np.random.default_rng(5)
    for cr, per, steps_per in ((CR_12, 2, 1), (CR_23, 3, 2), (CR_34, 4, 3)):
        lens = np.array([1 + (37 * i) % 411 for i in range(37)], np.uint32)
        nsofts = np.array([-(-(8 * int(L) + 22) // steps_per) * per for L in lens], np.uint32)
        nsofts[7] = nsofts[7] // (2 * per) * per                          # truncated: half of the soft values of block 7 are missing
        ns = int(nsofts.max())
        soft = rng.integers(0, 8, (37, ns)).astype(np.uint8)
        Lmax = int(lens.max())
        g, nraw = emu(soft, cr, Lmax, lens=lens, nsofts=nsofts, hb=hb)
        for i in range(37):
            L = int(lens[i]); n = int(nsofts[i])
            o = oracle_py.viterbi_blocks(soft[i:i + 1, :n], cr, L)[0]
            k = int(nraw[i])
            assert k <= L + 2 and (i == 7 or k == L + 2), (cr, i, k, L)
            assert (g[i, :k] == o[:k]).all(), (cr, i, L)

@HB
def test_short_windows(emu, hb):
    """Traceback windows shorter than a deferred walk lasts (the standalone decoder accepts any depth that is a multiple of 8): a trigger then
    finds the previous window's walk still in flight and has to finish it first; every window size must still give the oracle's bytes."""
    rng = np.random.default_rng(21)
    for cr, per in ((CR_12, 2), (CR_23, 3), (CR_34, 4)):
        L = 90; ns = (8 * L + 22 + 5) * per                               # more groups than the block needs, for every rate
        ns = ns // per * per
        soft = rng.integers(0, 8, (5, ns)).astype(np.uint8)
        for depth, look in ((8, 0), (8, 24), (16, 7), (64, 24), (128, 40), (248, 32)):
            g, _ = emu(soft, cr, L, depth, look, hb=hb)
            o = oracle_py.viterbi_blocks(soft, cr, L, depth, look)
            assert (g == o).all(), (cr, depth, look, np.argwhere(g != o)[:4])

# 802.11n soft bytes per OFDM symbol (N_CBPS, two streams) and code rate: MCS 8, 9, 11 (rate 1/2, 52 / 104 / 208 trellis steps per symbol)
# and 13 (rate 2/3, 416) are not whole 6-step chunks; MCS 10 and 14 (rate 3/4, 156 and 468) are.
N11N = ((CR_12, 104), (CR_12, 208), (CR_12, 416), (CR_23, 624), (CR_34, 208), (CR_34, 624))
GROUPS = {CR_12: (2, 1), CR_23: (3, 2), CR_34: (4, 3)}          # soft bytes and trellis steps per puncture group
RATES = {CR_12: (1, 2), CR_23: (2, 3), CR_34: (3, 4)}

def ragged_11n_blocks(rng, cr, ncbps, nblocks=40):
    """Code blocks the way k_front11n hands them over: whole symbols of ncbps soft bytes.  Short blocks whose flush point (8 L + 22 steps) lies
    past their last whole 6-step chunk, at every offset it can take there, alternate with long blocks, so that every warp of every kernel
    rendering holds both and the short ones run out of whole chunks while their neighbours go on.  Clean code words of varying confidence.
    Returns soft [nblocks, max nsoft], lens, nsofts and the sent bits."""
    per, gst = GROUPS[cr]
    spsym = ncbps // per * gst                                       # trellis steps per symbol
    shape = lambda L: (lambda S: (S, S // 6 * 6))(-(-(8 * L + 22) // spsym) * spsym)
    by_off = {}
    for L in range(1, 500):
        S, whole = shape(L)
        if 8 * L + 22 > whole: by_off.setdefault(8 * L + 22 - whole, []).append(L)
    short = [L for off in sorted(by_off) for L in by_off[off][:4]] or [5, 61, 62, 99]   # rate 3/4: no such length (whole chunks), plain ones
    lens = []
    for i in range(nblocks):
        lens.append(short[(i // 2) % len(short)] if i % 2 == 0 else 200 + 37 * (i % 5))
    lens = np.array(lens, np.uint32)
    nsofts = np.array([shape(int(L))[0] // gst * per for L in lens], np.uint32)
    ns = int(nsofts.max())
    soft = np.zeros((nblocks, ns), np.uint8); sent = []
    for i, L in enumerate(lens):
        S = int(nsofts[i]) // per * gst
        bits = rng.integers(0, 2, S).astype(np.uint8); bits[8 * int(L) + 16:] = 0
        A, B = synth.conv_encode(bits)
        coded = synth.puncture(A, B, RATES[cr])
        sv = np.where(coded > 0, rng.integers(4, 8, coded.shape), rng.integers(0, 4, coded.shape))
        soft[i, :len(coded)] = sv; sent.append(bits)
    return soft, lens, nsofts, sent

def check_ragged(run, cr, ncbps, seed, **kw):
    """run(soft, cr, Lmax, depth, look, lens=, nsofts=, **kw) -> (bytes, nraw): every block must equal the oracle in full."""
    soft, lens, nsofts, sent = ragged_11n_blocks(np.random.default_rng(seed), cr, ncbps)
    g, nraw = run(soft, cr, int(lens.max()), 192, 36, lens=lens, nsofts=nsofts, **kw)
    for i in range(len(lens)):
        L = int(lens[i]); n = int(nsofts[i])
        assert nraw[i] == L + 2, "block %d L=%d nsoft=%d: nraw %d, want %d" % (i, L, n, nraw[i], L + 2)
        o = oracle_py.viterbi_blocks(soft[i:i + 1, :n], cr, L, 192, 36)[0]
        assert (g[i, :L + 2] == o).all(), (i, L, np.argwhere(g[i, :L + 2] != o)[:4])
        assert (np.unpackbits(o, bitorder="little")[:8 * L + 16] == sent[i][:8 * L + 16]).all(), (i, L)

@HB
@pytest.mark.parametrize("cr, ncbps", N11N)
def test_ragged_chunks_11n_symbols(emu, hb, cr, ncbps):
    """A code block that runs out of whole 6-step chunks while a neighbour in its warp still has some must still decode its remaining
    whole groups and fire its last traceback window (802.11n frames: N_CBPS soft bytes per symbol, flush point in the last partial chunk)."""
    check_ragged(emu, cr, ncbps, 40 + ncbps + cr, hb=hb)

def test_ragged_chunks_two_blocks(emu):
    """The smallest case: L = 62 with 10 x 104 soft bytes beside L = 200 with 32 x 104 (rate 1/2, 802.11n window)."""
    rng = np.random.default_rng(62)
    soft = rng.integers(0, 8, (2, 32 * 104)).astype(np.uint8)
    lens = np.array([62, 200], np.uint32); nsofts = np.array([10 * 104, 32 * 104], np.uint32)
    for hb in (6, 8, 9):
        g, nraw = emu(soft, CR_12, 200, 192, 36, lens=lens, nsofts=nsofts, hb=hb)
        for i in range(2):
            L = int(lens[i])
            assert nraw[i] == L + 2, "hb %d block %d L=%d: nraw %d, want %d" % (hb, i, L, nraw[i], L + 2)
            assert (g[i, :L + 2] == oracle_py.viterbi_blocks(soft[i:i + 1, :nsofts[i]], CR_12, L, 192, 36)[0]).all(), (hb, i)
