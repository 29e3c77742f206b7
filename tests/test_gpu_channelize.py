"""GPU tests of the wideband channelizer (sb200_channelize, pytest -m gpu): bit for bit against the numpy model of tests/wideband_inputs.py
over lengths, channel counts, decimations, tap counts, increments and full-scale input; the pointer residency, launch bookkeeping and
argument checks of the C ABI; and the wideband captures of test_cpu_channelize.py channelized and decoded on the device, all
device-resident, against the CPU oracle decoding the numpy-channelized streams."""
import ctypes as C
import numpy as np, pytest
import torch
import wideband_inputs as W
import wideband_device as WD
from sora_b200 import api
from test_gpu_abi_residency import _matrix, _each, _fill
from test_cpu_channelize import CCA_WIDE, TAPS_11A, TAPS_11B, _full_scale, channels_11a, channels_11b, channels_11n
from wideband_device import GROUP_CH, DDC_INCS as INCS, ddc_channels as _channels, ddc_taps as _taps, sms as _sms

pytestmark = pytest.mark.gpu
V, U32, U64 = C.c_void_p, C.c_uint32, C.c_uint64
TILE = 4096

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

def _same(eng, x, ch, d, taps):
    got = eng.channelize(x, ch, d, taps); want = W.channelize(x, ch, d, taps)
    assert got.shape == want.shape and (got == want).all(), [(i, np.argwhere((got[i] != want[i]).any(1))[:3].ravel()) for i in range(len(ch)) if (got[i] != want[i]).any()]

@pytest.mark.parametrize("n", [1, 126, TILE - 1, TILE, TILE + 1, 3 * TILE + 2, 10001])
def test_lengths(eng, n):
    """n_in of 1, ntaps - 1, around one tile, and lengths that are not a multiple of D; random full-scale input with rails."""
    x = _full_scale(n, 10 + n)
    _same(eng, x, _channels(4, n), 4, _taps(127, n))
    _same(eng, x, [(0, 0), (2 ** 31, 1 << 20)], 3, _taps(255, n + 1))

@pytest.mark.parametrize("d", range(1, 17))
def test_decimations_channels_and_taps(eng, d):
    """D = 1 .. 16, with K = 1 .. 16 and ntaps 1 .. 255 spread over them."""
    x = _full_scale(9000 + 37 * d, 20 + d)
    k = d; ntaps = [1, 3, 17, 31, 63, 101, 127, 255][d % 8]
    _same(eng, x, _channels(k, d), d, _taps(ntaps, d))

def test_increments_and_phases(eng):
    """Every increment of INCS (0, quarter and half turns, wrapped negatives, arbitrary) with zero and arbitrary phase0, 16 channels."""
    x = _full_scale(20000, 30)
    ch = [(inc, ph) for inc in INCS for ph in (0, 0xDEADBEEF)]
    _same(eng, x, ch, 4, TAPS_11A)

def test_tap_sum_at_the_limit(eng):
    """sum |t| = 65535 on rail input: the accumulator reaches its extremes without wrapping."""
    t = _taps(63, 40, 65535); t[31] += 65535 - int(np.abs(t.astype(np.int64)).sum())
    assert np.abs(t.astype(np.int64)).sum() == 65535
    x = np.where(np.random.default_rng(41).random((12000, 2)) < 0.5, -32768, 32767).astype(np.int16)
    x[5000:5200] = np.where(t[np.arange(200) % 63] < 0, 32767, -32768)[:, None]     # runs whose products all take one sign
    _same(eng, x, [(0, 0), (2 ** 30, 0), (2 ** 31, 0)], 2, t)


# ---- long captures: several channels per CTA (GROUP_CH) -----------------------------------------------------------------------------
def _long_case(eng, tiles, k, d, taps, seed):
    """A full-scale capture of `tiles` tiles plus 777 samples, channelized on the device; its first, middle and last outputs against
    the model (channelize_window)."""
    n = tiles * TILE + 777; x = _full_scale(n, seed); ch = GROUP_CH[:k]
    n_out = -(-n // d); stride = (n_out + 3) // 4 * 4
    d_in = torch.from_numpy(x).cuda(); d_out = torch.zeros((k, stride, 2), dtype=torch.int16, device="cuda")
    eng.channelize_raw(d_in.data_ptr(), n, ch, d, taps, d_out.data_ptr(), stride)
    mid = (tiles // 2) * TILE // d
    for m0, m1 in ((0, 700), (mid - 350, mid + 350), (n_out - 700, n_out)):
        got = d_out[:, m0:m1].cpu().numpy(); want = W.channelize_window(x, ch, d, taps, m0, m1)
        assert (got == want).all(), (d, len(taps), m0, [(i, int((got[i] != want[i]).any(1).sum())) for i in range(k) if (got[i] != want[i]).any()])

@pytest.mark.parametrize("d", range(1, 17))
def test_all_channels_in_one_cta(eng, d):
    """D = 1 .. 16 with 251 / 253 / 255 taps (the largest halo) and 4 .. 16 channels, all of them in every CTA."""
    _long_case(eng, 4 * _sms() + 3, [4, 7, 11, 16][d % 4], d, _taps([251, 253, 255][d % 3], 80 + d), 80 + d)

@pytest.mark.parametrize("d", [1, 4, 10, 15, 16])
def test_channel_groups(eng, d):
    """A capture of a third of 4 x SMs tiles: 16 channels in groups of several per CTA."""
    _long_case(eng, 4 * _sms() // 3, 16, d, _taps(255, 90 + d), 90 + d)


# ---- the C ABI ----------------------------------------------------------------------------------------------------------------------
def test_residency(eng):
    """iq and out each host or device; out rows are wider than n_out: the bytes between and after them stay untouched."""
    x = _full_scale(1001, 50); ch = _channels(3, 50); D = 3; n_out = 334; stride = 340
    args = dict(iq=x, out=_fill(3 * stride * 4 + 16))
    ref = _matrix(lambda p: eng.channelize_raw(p["iq"], 1001, ch, D, TAPS_11A, p["out"], stride), args, _each(*args))
    rows = ref["out"][:3 * stride * 4].view(np.int16).reshape(3, stride, 2)
    assert (rows[:, :n_out] == W.channelize(x, ch, D, TAPS_11A)).all()
    assert (ref["out"][:3 * stride * 4].reshape(3, stride * 4)[:, n_out * 4:] == 0xA5).all() and (ref["out"][3 * stride * 4:] == 0xA5).all()

def test_one_launch_and_timing():
    e = api.Engine(0)
    try:
        x = _full_scale(50000, 60)
        for _ in range(2):
            n0 = e.launches; e.channelize(x, _channels(5, 60), 4, TAPS_11A)
            assert e.launches - n0 == 1 and e.last_kernel_ms() >= 0
    finally:
        e.close()

def _call(eng, iq, n, ch, nch, d, taps, ntaps, out, stride):
    return eng._lib.sb200_channelize(eng._h, V(iq), U64(n), V(ch), U32(nch), U32(d), V(taps), U32(ntaps), V(out), U64(stride), V(0))

def test_invalid_arguments_are_rejected(eng):
    x = _full_scale(1000, 70); out = np.zeros((17, 1000, 2), np.int16)
    ch = (api.DdcChannel * 17)(*[api.DdcChannel(i << 24, 0) for i in range(17)])
    t = np.array(TAPS_11A); xp, op, cp, tp = x.ctypes.data, out.ctypes.data, C.addressof(ch), t.ctypes.data
    assert _call(eng, xp, 1000, cp, 4, 4, tp, 127, op, 252) == 0
    big = np.full(9, 7282, np.int16)                                                # sum |t| = 65538
    bad = {"nchannels 0": (xp, 1000, cp, 0, 4, tp, 127, op, 252), "nchannels 17": (xp, 1000, cp, 17, 4, tp, 127, op, 252),
           "decim 0": (xp, 1000, cp, 4, 0, tp, 127, op, 252), "decim 17": (xp, 1000, cp, 4, 17, tp, 127, op, 252),
           "ntaps even": (xp, 1000, cp, 4, 4, tp, 126, op, 252), "ntaps 257": (xp, 1000, cp, 4, 4, np.zeros(257, np.int16).ctypes.data, 257, op, 252),
           "tap sum": (xp, 1000, cp, 4, 4, big.ctypes.data, 9, op, 252), "stride < n_out": (xp, 1000, cp, 4, 4, tp, 127, op, 248),
           "stride % 4": (xp, 1000, cp, 4, 4, tp, 127, op, 254), "null iq": (0, 1000, cp, 4, 4, tp, 127, op, 252),
           "null channels": (xp, 1000, 0, 4, 4, tp, 127, op, 252), "null taps": (xp, 1000, cp, 4, 4, 0, 127, op, 252),
           "null out": (xp, 1000, cp, 4, 4, tp, 127, 0, 252)}
    for name, a in bad.items():
        assert _call(eng, *a) == -1, name
    d = torch.zeros(2 * 1000 * 2 + 8, dtype=torch.int16, device="cuda")
    assert _call(eng, d.data_ptr() + 4, 999, cp, 1, 4, tp, 127, op, 252) == -1, "misaligned device input"
    assert _call(eng, xp, 1000, cp, 1, 4, tp, 127, d.data_ptr() + 4, 252) == -1, "misaligned device output"
    big[0] -= 3
    assert _call(eng, xp, 1000, cp, 4, 4, big.ctypes.data, 9, op, 252) == 0                  # sum |t| = 65535 is accepted


# ---- end to end, device-resident ----------------------------------------------------------------------------------------------------
def _dev_channelize(eng, x, fcs, fs, taps):
    """The capture on the device, channelized into device rows; returns (device rows [K, stride, 2], stride, n_out)."""
    d_in = torch.from_numpy(np.ascontiguousarray(x)).cuda(); n = len(x); n_out = -(-n // 4)
    d_out = WD.dev_rows(len(fcs), n_out, 64); stride = d_out.shape[1]
    eng.channelize_raw(d_in.data_ptr(), n, [(W.phase_inc(f, fs), 0) for f in fcs], 4, taps, d_out.data_ptr(), stride)
    return d_out, stride, n_out

def test_wideband_11a_on_the_device():
    iq, fcs, _ = W.capture_11a(); rows, _ = channels_11a(); K = len(fcs)
    e = api.Engine(0, cca_pwr_threshold=CCA_WIDE)
    try:
        d, stride, n_out = _dev_channelize(e, iq, fcs, W.FS_11A_WIDE, TAPS_11A)
        assert (d[:, :n_out].cpu().numpy() == rows).all()
        got = WD.rx11a(e, d, stride, n_out, K)
    finally:
        e.close()
    for c, (o, _) in enumerate(WD.equal_11a(rows, got)): assert len(o) >= 3, (c, o)

def test_wideband_11b_on_the_device(eng):
    iq, fcs, _ = W.capture_11b(); rows, _ = channels_11b(); K = len(fcs)
    d, stride, n_out = _dev_channelize(eng, iq, fcs, W.FS_11B_WIDE, TAPS_11B)
    assert (d[:, :n_out].cpu().numpy() == rows).all()
    for c, (o, _) in enumerate(WD.equal_11b(rows, WD.rx11b(eng, d, stride, n_out, K))): assert len(o) >= 2, (c, o)

def test_wideband_11n_on_the_device(eng):
    (a0, a1), fcs, _ = W.capture_11n(); r0, r1, _ = channels_11n(); K = len(fcs)
    d0, stride, n_out = _dev_channelize(eng, a0, fcs, W.FS_11A_WIDE, TAPS_11A)
    d1, _, _ = _dev_channelize(eng, a1, fcs, W.FS_11A_WIDE, TAPS_11A)
    assert (d0[:, :n_out].cpu().numpy() == r0).all() and (d1[:, :n_out].cpu().numpy() == r1).all()
    for c, (o, _) in enumerate(WD.equal_11n(r0, r1, WD.rx11n(eng, d0, d1, stride, n_out, K))): assert len(o) >= 2, (c, o)
