"""The transmitters' default out_stride against the library's own frame lengths, without a GPU: tests/cpp/tx_frames.cpp builds
sora_b200/csrc/tx_frames.cuh with the host compiler and returns, per rate and frame length, the smallest out_stride_samples the batch
call accepts.  For every rate (preamble, sample rate, MCS 8 .. 14) and every frame length the call accepts, the default stride of the
Python wrapper must be at least that minimum, so that a call with the default is never refused; the legacy transmitters' sample counts
must equal it exactly.  The Python rate tables must agree with the C ones."""
import ctypes as C, os, shutil, subprocess
import numpy as np, pytest
from sora_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E = api.Engine
LEADS = [0, 1, 3, 4, 5, 8, 20, 304, 400]

@pytest.fixture(scope="module")
def frames(tmp_path_factory):
    if shutil.which("g++") is None: pytest.skip("no host compiler")
    so = str(tmp_path_factory.mktemp("tx_frames") / "tx_frames.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "sora_b200", "csrc"),
                           "-o", so, os.path.join(ROOT, "tests", "cpp", "tx_frames.cpp")])
    L = C.CDLL(so)
    for f in (L.ndbps_11a, L.chips_11b, L.ndbps_11n): f.argtypes, f.restype = [C.c_uint32], C.c_uint32
    for f in (L.strides_11a, L.strides_11b, L.strides_11n, L.strides_11b_legacy, L.strides_11a_legacy):
        f.argtypes, f.restype = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p], C.c_int
    return L

def c_min(fn, a, b, n):
    """fn(a, b) over lengths 0 .. n - 1 -> int64 [n]"""
    out = np.zeros(n, np.uint64)
    assert fn(a, b, n, out.ctypes.data) == 0
    return out.astype(np.int64)

def test_rate_tables_agree(frames):
    assert {k: frames.ndbps_11a(k) for k in api._NDBPS_11A} == api._NDBPS_11A
    assert {k: frames.chips_11b(k) for k in api._CHIPS_11B} == api._CHIPS_11B
    assert {m: frames.ndbps_11n(m) for m in api._NDBPS_11N} == api._NDBPS_11N
    assert all(frames.ndbps_11n(m) for m in range(8, 15)) and frames.ndbps_11n(7) == 0 and frames.ndbps_11n(15) == 0
    assert frames.ndbps_11a(7000) == 0 and frames.chips_11b(6000) == 0

@pytest.mark.parametrize("lead", LEADS)
@pytest.mark.parametrize("rate", sorted(api._NDBPS_11A))
def test_tx11a_default_stride_is_accepted(frames, rate, lead):
    n = 4092                                           # MPDU 0 .. 4091 bytes (LENGTH is 12 bits, FCS included)
    got = np.array([E.tx11a_out_stride(L, rate, lead) for L in range(n)])
    assert (got >= c_min(frames.strides_11a, rate, lead, n)).all()

@pytest.mark.parametrize("lead", LEADS)
@pytest.mark.parametrize("rate", sorted(api._CHIPS_11B))
def test_tx11b_default_stride_is_accepted(frames, rate, lead):
    n = 4092                                           # MPDU 0 .. 4091 bytes
    got = np.array([E.tx11b_out_stride(L, rate, lead) for L in range(n)])
    assert (got >= c_min(frames.strides_11b, rate, lead, n)).all()

@pytest.mark.parametrize("lead", LEADS)
@pytest.mark.parametrize("mcs", range(8, 15))
def test_tx11n_default_stride_is_accepted(frames, mcs, lead):
    n = 4092                                           # MPDU 0 .. 4091 bytes
    got = np.array([E.tx11n_out_stride(L, mcs, lead) for L in range(n)])
    assert (got >= c_min(frames.strides_11n, mcs, lead, n)).all()

@pytest.mark.parametrize("short_preamble", [False, True])
@pytest.mark.parametrize("rate", sorted(api._CHIPS_11B))
def test_tx11b_legacy_nsamples_equal_the_library(frames, rate, short_preamble):
    sizes = np.arange(4, 4096)                         # PSDU 4 .. 4095 bytes, FCS included
    got = np.array([E.tx11b_legacy_nsamples(int(s), rate, short_preamble) for s in sizes])
    assert (got == c_min(frames.strides_11b_legacy, rate, int(short_preamble), 4096)[4:]).all()

@pytest.mark.parametrize("sample_rate_mhz", [40, 44])
@pytest.mark.parametrize("rate", sorted(api._NDBPS_11A))
def test_tx11a_legacy_nsamples_equal_the_library(frames, rate, sample_rate_mhz):
    sizes = np.arange(4, 4097)                         # PSDU 4 .. 4096 bytes, FCS included
    got = np.array([E.tx11a_legacy_nsamples(int(s), rate, sample_rate_mhz) for s in sizes])
    assert (got == c_min(frames.strides_11a_legacy, rate, sample_rate_mhz, 4097)[4:]).all()
