"""The packed complex-int16 helpers of sora_b200/csrc/fixed.cuh (pk_*, the arithmetic of k_front11a) against the scalar primitives they
replace, WITHOUT a GPU: tests/cpp/packed_emu.cpp compiles the header for the host and both paths run on the same words.  Unary helpers see
every low half against edge high halves and the other way round; products and butterflies see random words plus every combination of the
int16 edges (-32768, -32767, -1, 0, 1, 32767, ...).  The device build of the same helpers is checked bit for bit by the GPU tests of the
802.11a receive chain (stage taps, golden captures, rail captures)."""
import ctypes as C, itertools, os, shutil, subprocess
import numpy as np, pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "packed_emu.cpp"); CSRC = os.path.join(ROOT, "sora_b200", "csrc")
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="no host compiler")

EDGES = np.array([-32768, -32767, -16385, -16384, -8193, -8192, -2049, -2048, -129, -128, -1, 0, 1, 127, 128, 2047, 2048, 8191, 8192,
                  16383, 16384, 32766, 32767], np.int64)

def words(re, im):
    return ((np.asarray(re, np.int64) & 0xFFFF) | ((np.asarray(im, np.int64) & 0xFFFF) << 16)).astype(np.uint32)

@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("packed_emu") / "packed_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-DSB_HOST_EMU", "-I", CSRC, "-o", so, SRC])
    L = C.CDLL(so)
    P = C.c_void_p
    L.packed_unary.argtypes = [C.c_int, P, C.c_uint32, P, P]
    L.packed_cmul.argtypes = [C.c_int, P, P, C.c_uint32, P, P]
    L.packed_butterfly.argtypes = [C.c_int, P, P, C.c_uint32, P, P]
    return L

def _run(fn, op, *arrays, n, out_len):
    arrays = [np.ascontiguousarray(a, np.uint32) for a in arrays]
    got = np.zeros(out_len, np.uint32); want = np.zeros(out_len, np.uint32)
    fn(op, *[a.ctypes.data for a in arrays], n, got.ctypes.data, want.ctypes.data)
    return got, want

def _check(got, want, what):
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%s: %d mismatches, first at %d: got %08x want %08x" % (what, bad.size, bad[0], got[bad[0]], want[bad[0]])

@pytest.mark.parametrize("op,name", [(0, "sra1"), (1, "sra2"), (2, "sra4"), (3, "mulj"), (4, "mulmj"), (5, "demap clamp")])
def test_unary_every_half(lib, op, name):
    allv = np.arange(-32768, 32768, dtype=np.int64)
    rng = np.random.default_rng(op)
    others = np.concatenate([EDGES, rng.integers(-32768, 32768, 9)])
    a = np.concatenate([words(allv, o) for o in others] + [words(o, allv) for o in others])
    got, want = _run(lib.packed_unary, op, a, n=a.size, out_len=a.size)
    _check(got, want, name)

@pytest.mark.parametrize("op,name", [(0, "cmul_q15"), (1, "cmul_tw"), (2, "cmul32 >> 8"), (3, "freq comp")])
def test_products(lib, op, name):
    rng = np.random.default_rng(10 + op)
    n = 1 << 20
    a = words(rng.integers(-32768, 32768, n), rng.integers(-32768, 32768, n)); b = words(rng.integers(-32768, 32768, n), rng.integers(-32768, 32768, n))
    g = np.array(list(itertools.product(EDGES, repeat=4)), np.int64)
    a = np.concatenate([a, words(g[:, 0], g[:, 1])]); b = np.concatenate([b, words(g[:, 2], g[:, 3])])
    got, want = _run(lib.packed_cmul, op, a, b, n=a.size, out_len=a.size)
    _check(got, want, name)

@pytest.mark.parametrize("op,name", [(0, "radix-4 butterfly"), (1, "dft4")])
def test_butterflies(lib, op, name):
    rng = np.random.default_rng(20 + op)
    n = 1 << 18
    x = words(rng.integers(-32768, 32768, 4 * n), rng.integers(-32768, 32768, 4 * n))
    w = words(rng.integers(-32768, 32768, 3 * n), rng.integers(-32768, 32768, 3 * n))
    # every input at an edge in both halves (all four inputs equal or alternating between two edges), twiddles at the edges too
    e = [int(v) for v in words(EDGES, EDGES[::-1])] + [int(v) for v in words(EDGES, EDGES)]
    ex = np.array([[p, q, p, q] for p in e for q in e] + [[p, q, q, p] for p in e for q in e], np.uint32)
    ew = np.array([[e[i % len(e)], e[(3 * i + 1) % len(e)], e[(7 * i + 2) % len(e)]] for i in range(len(ex))], np.uint32)
    x = np.concatenate([x, ex.ravel()]); w = np.concatenate([w, ew.ravel()])
    m = x.size // 4
    got, want = _run(lib.packed_butterfly, op, x, w, n=m, out_len=4 * m)
    _check(got, want, name)
