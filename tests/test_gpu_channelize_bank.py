"""GPU tests of the filter-bank channelizer (sb200_channelize_bank, pytest -m gpu): bit for bit against the numpy model of
tests/bank_model.py over lengths, grids, decimations, stackings, tap counts and full-scale input; the pointer residency, streams, launch
bookkeeping and argument checks of the C ABI; channel k against the device's sb200_channelize; and the captures of
test_cpu_channelize_bank.py taken apart and decoded on the device, all device-resident, against the CPU oracle."""
import ctypes as C
import numpy as np, pytest
import torch
import oracle_py
import wideband_inputs as W
import wideband_device as WD
import bank_model as B
from sora_b200 import api
from test_gpu_abi_residency import _matrix, _each, _fill
from test_cpu_channelize import CCA_WIDE, _full_scale
from test_cpu_channelize_bank import GRID, bank_rows_11a, bank_rows_11n, bank_rows_octet
from wideband_device import ddc_taps as _taps

pytestmark = pytest.mark.gpu
V, U32, U64 = C.c_void_p, C.c_uint32, C.c_uint64
TILE = 4096

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

def _same(eng, x, M, D, odd, taps):
    got = eng.channelize_bank(x, M, D, taps, odd=odd); want = B.bank(x, M, D, odd, taps)
    assert got.shape == want.shape and (got == want).all(), (M, D, odd, len(taps), [(k, np.argwhere((got[k] != want[k]).any(1))[:3].ravel()) for k in range(M) if (got[k] != want[k]).any()])

@pytest.mark.parametrize("n", [1, 126, TILE - 1, TILE, TILE + 1, 3 * TILE + 2, 10001])
def test_lengths(eng, n):
    """n_in of 1, below ntaps, around one tile and not a multiple of D; full-scale input with rails."""
    x = _full_scale(n, 10 + n)
    _same(eng, x, 8, 4, 1, _taps(255, n))
    _same(eng, x, 16, 2, 0, _taps(127, n + 1))

@pytest.mark.parametrize("M,D", GRID)
def test_grid(eng, M, D):
    """Every M = 2 .. 64 and every D | M, both stackings."""
    x = _full_scale(9000 + 37 * M + D, M * 64 + D)
    for odd in (0, 1):
        _same(eng, x, M, D, odd, _taps([31, 63, 127, 255][(M + D + odd) % 4], M + D + odd))

@pytest.mark.parametrize("ntaps", [1, 3, 5, 63, 65, 255, 257, 511, 1021, 1023])
def test_ntaps(eng, ntaps):
    """Tap counts 1 .. 1023, below, at and above multiples of M (halos up to 512 samples)."""
    x = _full_scale(3 * TILE + 999, ntaps)
    _same(eng, x, 64, 8, 1, _taps(ntaps, ntaps))
    _same(eng, x, 4, 1, 0, _taps(ntaps, ntaps + 1))

@pytest.mark.parametrize("M", [2, 8, 64])
def test_tap_sum_at_the_limit(eng, M):
    """sum |t| = 65535 on rail input: branch sums and butterflies at their extremes, outputs saturating, the int64 DFT path."""
    t = _taps(255, 40 + M, 65535); t[127] += 65535 - int(np.abs(t.astype(np.int64)).sum())
    assert np.abs(t.astype(np.int64)).sum() == 65535
    x = np.where(np.random.default_rng(41).random((12000, 2)) < 0.5, -32768, 32767).astype(np.int16)
    x[5000:5400] = np.where(t[np.arange(400) % 255] < 0, 32767, -32768)[:, None]   # runs whose products all take one sign
    for odd in (0, 1):
        _same(eng, x, M, min(M, 4), odd, t)

@pytest.mark.parametrize("M,D,ntaps", [(8, 4, 255), (64, 64, 1023), (2, 1, 63)])
def test_long_capture(eng, M, D, ntaps):
    """A capture of 4 x SMs tiles plus 777 samples, device-resident; its first, middle and last outputs against the model's windows."""
    n = 4 * WD.sms() * TILE + 777; x = _full_scale(n, M + ntaps); taps = _taps(ntaps, M)
    n_out = -(-n // D); stride = (n_out + 3) // 4 * 4
    d_in = torch.from_numpy(x).cuda(); d_out = torch.zeros((M, stride, 2), dtype=torch.int16, device="cuda")
    for odd in (0, 1):
        eng.channelize_bank_raw(d_in.data_ptr(), n, M, D, taps, d_out.data_ptr(), stride, odd=odd)
        mid = n_out // 2
        for m0, m1 in ((0, 300), (mid - 150, mid + 150), (n_out - 300, n_out)):
            got = d_out[:, m0:m1].cpu().numpy(); want = B.window(x, M, D, odd, taps, m0, m1)
            assert (got == want).all(), (M, D, odd, m0)


# ---- the C ABI ----------------------------------------------------------------------------------------------------------------------
def test_residency(eng):
    """iq and out each host or device; out rows wider than n_out: the bytes between and after them stay untouched."""
    x = _full_scale(5001, 50); M, D = 8, 2; n_out = 2501; stride = 2508; taps = _taps(127, 50)
    args = dict(iq=x, out=_fill(M * stride * 4 + 16))
    ref = _matrix(lambda p: eng.channelize_bank_raw(p["iq"], 5001, M, D, taps, p["out"], stride, odd=True), args, _each(*args))
    rows = ref["out"][:M * stride * 4].view(np.int16).reshape(M, stride, 2)
    assert (rows[:, :n_out] == B.bank(x, M, D, 1, taps)).all()
    assert (ref["out"][:M * stride * 4].reshape(M, stride * 4)[:, n_out * 4:] == 0xA5).all() and (ref["out"][M * stride * 4:] == 0xA5).all()

def test_caller_stream_one_launch_and_timing():
    e = api.Engine(0)
    try:
        x = _full_scale(50000, 60); taps = _taps(255, 60); n_out = 12500; stride = 12500
        d_in = torch.from_numpy(x).cuda(); d_out = torch.zeros((16, stride, 2), dtype=torch.int16, device="cuda")
        s = torch.cuda.Stream()
        for _ in range(2):
            n0 = e.launches
            with torch.cuda.stream(s):
                e.channelize_bank_raw(d_in.data_ptr(), 50000, 16, 4, taps, d_out.data_ptr(), stride, odd=True, stream=s.cuda_stream)
            assert e.launches - n0 == 1
            s.synchronize()
            assert e.last_kernel_ms() >= 0 and (d_out.cpu().numpy() == B.bank(x, 16, 4, 1, taps)).all()
    finally:
        e.close()

def _call(eng, iq, n, M, D, odd, taps, ntaps, out, stride):
    return eng._lib.sb200_channelize_bank(eng._h, V(iq), U64(n), U32(M), U32(D), U32(odd), V(taps), U32(ntaps), V(out), U64(stride), V(0))

def test_invalid_arguments_are_rejected(eng):
    x = _full_scale(1000, 70); out = np.zeros((64, 1000, 2), np.int16); t = _taps(127, 70)
    xp, op, tp = x.ctypes.data, out.ctypes.data, t.ctypes.data
    assert _call(eng, xp, 1000, 8, 4, 1, tp, 127, op, 252) == 0
    big = np.full(9, 7282, np.int16); t1025 = np.zeros(1025, np.int16); t1025[512] = 100
    bad = {"M 0": (xp, 1000, 0, 1, 0, tp, 127, op, 252), "M 1": (xp, 1000, 1, 1, 0, tp, 127, op, 252), "M 6": (xp, 1000, 6, 2, 0, tp, 127, op, 252),
           "M 128": (xp, 1000, 128, 4, 0, tp, 127, op, 252), "D 0": (xp, 1000, 8, 0, 0, tp, 127, op, 252), "D 3": (xp, 1000, 8, 3, 0, tp, 127, op, 336),
           "D 16 > M": (xp, 1000, 8, 16, 0, tp, 127, op, 252), "odd 2": (xp, 1000, 8, 4, 2, tp, 127, op, 252),
           "ntaps even": (xp, 1000, 8, 4, 0, tp, 126, op, 252), "ntaps 0": (xp, 1000, 8, 4, 0, tp, 0, op, 252),
           "ntaps 1025": (xp, 1000, 8, 4, 0, t1025.ctypes.data, 1025, op, 252), "tap sum": (xp, 1000, 8, 4, 0, big.ctypes.data, 9, op, 252),
           "stride < n_out": (xp, 1000, 8, 4, 0, tp, 127, op, 248), "stride % 4": (xp, 1000, 8, 4, 0, tp, 127, op, 254),
           "stride > 2^40": (xp, 1000, 8, 4, 0, tp, 127, op, 2 ** 40 + 4), "n_in > 2^40": (xp, 2 ** 40 + 1, 8, 4, 0, tp, 127, op, 2 ** 40),
           "null iq": (0, 1000, 8, 4, 0, tp, 127, op, 252), "null taps": (xp, 1000, 8, 4, 0, 0, 127, op, 252), "null out": (xp, 1000, 8, 4, 0, tp, 127, 0, 252)}
    n0 = eng.launches
    for name, a in bad.items():
        assert _call(eng, *a) == -1, name
    d = torch.zeros(2 * 1000 * 2 + 8, dtype=torch.int16, device="cuda")
    assert _call(eng, d.data_ptr() + 4, 999, 2, 2, 0, tp, 127, op, 500) == -1, "misaligned device input"
    assert _call(eng, xp, 1000, 2, 2, 0, tp, 127, d.data_ptr() + 4, 500) == -1, "misaligned device output"
    assert eng.launches == n0, "a refused call launched"
    big[0] -= 3
    assert _call(eng, xp, 1000, 8, 4, 0, big.ctypes.data, 9, op, 252) == 0                  # sum |t| = 65535 is accepted

@pytest.mark.parametrize("M", [4, 8, 16, 64])
def test_against_the_device_channelizer(eng, M):
    """Channel k of the bank against the device's sb200_channelize at phase_inc = (2k + o) 2^31 / M (16 channels per call at most),
    within 2 LSB where neither saturates."""
    x = np.random.default_rng(M).integers(-23170, 23171, (30000, 2)).astype(np.int16); taps = _taps(255, M)
    for odd in (0, 1):
        bank = eng.channelize_bank(x, M, 4 if M >= 4 else 2, taps, odd=odd).astype(np.int64)
        inc = B.phase_incs(M, odd)
        ch = np.concatenate([eng.channelize(x, inc[i:i + 16], 4 if M >= 4 else 2, taps) for i in range(0, M, 16)]).astype(np.int64)
        assert np.abs(bank - ch).max() <= 2, (M, odd)


# ---- end to end, device-resident ----------------------------------------------------------------------------------------------------
def _dev_bank(eng, x, odd):
    """The capture on the device, taken apart by the M = 8, D = 4 bank into device rows; returns (rows [8, stride, 2], stride, n_out)."""
    d_in = torch.from_numpy(np.ascontiguousarray(x)).cuda(); n = len(x); n_out = -(-n // 4)
    d_out = WD.dev_rows(8, n_out, 64); stride = d_out.shape[1]
    eng.channelize_bank_raw(d_in.data_ptr(), n, 8, 4, B.TAPS_BANK, d_out.data_ptr(), stride, odd=odd)
    return d_out, stride, n_out

@pytest.mark.parametrize("case", ["even", "odd"])
def test_bank_11a_on_the_device(case):
    """capture_11a through the even-stacked bank, and the eight-channel capture through the odd-stacked one, into sb200_rx11a_streams:
    equal to the oracle decoding the model's rows, on every field, event position and delivered byte."""
    iq, fcs, _ = W.capture_11a() if case == "even" else B.capture_11a_octet()
    rows, want = bank_rows_11a() if case == "even" else bank_rows_octet()
    e = api.Engine(0, cca_pwr_threshold=CCA_WIDE)
    try:
        d, stride, n_out = _dev_bank(e, iq, case == "odd")
        assert (d[:, :n_out].cpu().numpy() == rows).all()
        got = WD.rx11a(e, d, stride, n_out, 8)
    finally:
        e.close()
    for c, (o, _) in enumerate(WD.equal_11a(rows, got)):
        assert sum((o["status"] == oracle_py.E_FRAME_OK)) == len(want.get(c, [])), c

def test_bank_11n_on_the_device(eng):
    (a0, a1), fcs, _ = W.capture_11n(); r0, r1, want = bank_rows_11n()
    d0, stride, n_out = _dev_bank(eng, a0, False)
    d1, _, _ = _dev_bank(eng, a1, False)
    assert (d0[:, :n_out].cpu().numpy() == r0).all() and (d1[:, :n_out].cpu().numpy() == r1).all()
    for c, (o, _) in enumerate(WD.equal_11n(r0, r1, WD.rx11n(eng, d0, d1, stride, n_out, 8))):
        assert sum(o["status"] == oracle_py.E_FRAME_OK) == len(want.get(c, [])), (c, o)
