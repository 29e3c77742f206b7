"""k_viterbi_re as persistent CTAs, WITHOUT a GPU (the device source compiled for the host by tests/cpp/re_emu_grid.cpp): a grid smaller than the
number of groups of code blocks, so that one CTA decodes several groups in a row and every group must start from the state a fresh CTA
starts from (metrics, ring position, traceback schedule, the ragged-block tail).  The last group is ragged (fewer code blocks than a warp
holds), the code blocks have different lengths, and one is truncated; every byte is compared with the CPU oracle."""
import ctypes as C, os, shutil, subprocess
import numpy as np, pytest
import oracle_py
from test_cpu_lane_emu import CR_12, CR_23, CR_34, check_ragged

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "re_emu_grid.cpp"); CSRC = os.path.join(ROOT, "sora_b200", "csrc")
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="no host compiler")

@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("re_emu_grid") / "re_emu_grid.so")
    subprocess.check_call(["g++", "-O1", "-std=c++20", "-pthread", "-shared", "-fPIC", "-DSB_HOST_EMU", "-Wno-unknown-pragmas", "-I", CSRC, "-o", so, SRC])
    lib = C.CDLL(so)
    lib.re_emu_viterbi_grid.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    lib.re_emu_viterbi_grid.restype = C.c_int
    def run(soft, cr, L, depth=256, look=24, lens=None, nsofts=None, ctas=1):
        soft = np.ascontiguousarray(soft, dtype=np.uint8); nb, ns = soft.shape
        stride = (ns + 15) // 16 * 16 + 16
        sp = np.zeros((nb, stride), np.uint8); sp[:, :ns] = soft
        ostride = L + 2 + 14
        out = np.zeros((nb, ostride), np.uint8); nraw = np.zeros(nb, np.uint32)
        lp = np.ascontiguousarray(lens, dtype=np.uint32) if lens is not None else None
        npp = np.ascontiguousarray(nsofts, dtype=np.uint32) if nsofts is not None else None
        rc = lib.re_emu_viterbi_grid(sp.ctypes.data, stride, ns, nb, cr, L, depth, look, out.ctypes.data, ostride, nraw.ctypes.data,
                                     lp.ctypes.data if lp is not None else None, npp.ctypes.data if npp is not None else None, ctas)
        assert rc == 0
        return out[:, :L + 2], nraw
    return run

@pytest.mark.parametrize("ctas", (1, 2))
def test_several_groups_per_cta(emu, ctas):
    """Three full groups and a ragged fourth, blocks of different lengths (one truncated), on one or two CTAs: CTA 0 decodes every group
    but the second one, so a long block's group is followed by shorter ones and the ragged group comes after a full one."""
    fr = 8                                                                # code blocks per CTA
    nb = 3 * fr + 5
    rng = np.random.default_rng(19 + 10 * ctas)
    for cr, per, steps_per in ((CR_12, 2, 1), (CR_23, 3, 2), (CR_34, 4, 3)):
        lens = np.array([1 + (53 * i) % 173 for i in range(nb)], np.uint32)
        lens[:fr] += 60                                                   # the first group is the longest: later groups must not inherit its state
        nsofts = np.array([-(-(8 * int(L) + 22) // steps_per) * per for L in lens], np.uint32)
        nsofts[fr + 3] = nsofts[fr + 3] // (2 * per) * per                # a truncated block in the second group
        soft = rng.integers(0, 8, (nb, int(nsofts.max()))).astype(np.uint8)
        g, nraw = emu(soft, cr, int(lens.max()), lens=lens, nsofts=nsofts, ctas=ctas)
        for i in range(nb):
            o, k = oracle_py.viterbi_blocks_n(soft[i:i + 1, :int(nsofts[i])], cr, int(lens[i]))
            assert nraw[i] == k[0] and (i == fr + 3 or k[0] == lens[i] + 2), (cr, i, nraw[i], k[0])
            assert (g[i, :k[0]] == o[0, :k[0]]).all(), (cr, ctas, i)

def test_uniform_blocks_one_cta(emu):
    """sb200_viterbi_k7's uniform parameters (no FrameInfo): 27 code blocks, rate 3/4, one CTA for all four groups."""
    rng = np.random.default_rng(29)
    L = 90; ns = -(-(8 * L + 22) // 3) * 4 + 8
    soft = rng.integers(0, 8, (27, ns)).astype(np.uint8)
    g, nraw = emu(soft, CR_34, L, 64, 30)
    assert (g == oracle_py.viterbi_blocks(soft, CR_34, L, 64, 30)).all() and (nraw == L + 2).all()

def test_ragged_chunks_11n_symbols_one_cta(emu):
    """802.11n frames whose blocks run out of whole 6-step chunks at different times (the tail path), all groups on one CTA."""
    check_ragged(emu, CR_12, 104, 144, ctas=1)
