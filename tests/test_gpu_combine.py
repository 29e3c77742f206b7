"""GPU tests of the wideband combiner (sb200_combine, pytest -m gpu): bit for bit against the numpy model of tests/combine_model.py over
lengths around a tile, channel counts, interpolations, tap counts, gains, increments and full-scale input; the pointer residency, stream,
launch bookkeeping and argument checks of the C ABI; and the transmit chains of test_cpu_combine.py on the device (transmitter ->
combiner -> channelizer -> stream receivers, all device-resident) against the CPU oracle on the same chain."""
import ctypes as C
import numpy as np, pytest
import torch
import oracle_py
import wideband_inputs as W
import wideband_device as WD
import combine_model as CM
from sora_b200 import api
from test_gpu_abi_residency import _matrix, _each, _fill
from test_cpu_channelize import CCA_WIDE, TAPS_11A, TAPS_11B
from test_cpu_combine import TAPS_UP, TAPS_UP_11B, GAIN_11A, frames_11a, frames_11b, frames_11n, wide_11a, wide_11b, wide_11n
from wideband_device import GAINS, DUC_INCS as INCS, duc_channels as _channels, duc_rows as _rows, duc_taps as _taps, sms as _sms

pytestmark = pytest.mark.gpu
V, U32, U64 = C.c_void_p, C.c_uint32, C.c_uint64

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

def _tile(K, U, ntaps):
    """Input samples per CTA that sb200_combine picks: 1024, 512 or 256, the largest whose shared memory fits 51200 bytes."""
    halo = ((ntaps // 2 + U - 1) // U + 3) // 4 * 4
    for ti in (1024, 512):
        if (K * (ti + 2 * halo) + U * ti + 4096) * 4 + 16 <= 51200: return ti
    return 256

def _same(eng, rows, ch, u, taps):
    got = eng.combine(rows, ch, u, taps); want = CM.combine(rows, ch, u, taps)
    assert got.shape == want.shape and (got == want).all(), np.argwhere((got != want).any(1))[:5].ravel()


@pytest.mark.parametrize("K,U,ntaps", [(4, 4, 127), (3, 5, 255), (16, 16, 255), (1, 1, 1)])
def test_lengths(eng, K, U, ntaps):
    """n_in of 1 .. 5 and around the tile the call picks for (K, U, ntaps), and several tiles + 777; full-scale input with rails."""
    ti = _tile(K, U, ntaps)
    for n in (1, 2, 3, 4, 5, ti - 1, ti, ti + 1, 3 * ti + 777):
        _same(eng, _rows(K, n, n), _channels(K, n), U, _taps(ntaps, U, n))

@pytest.mark.parametrize("u", range(1, 17))
def test_interpolations_channels_and_taps(eng, u):
    """U = 1 .. 16, with K = 1 .. 16 and ntaps 1 .. 255 spread over them; every gain and increment kind."""
    k = 17 - u; ntaps = [1, 3, 17, 31, 63, 101, 127, 255][u % 8]
    _same(eng, _rows(k, 2000 + 37 * u, 20 + u), _channels(k, u), u, _taps(ntaps, u, u))

def test_increments_phases_and_gains(eng):
    """Every increment of INCS with zero and arbitrary phase0, 16 channels, gains 0 .. 65535."""
    ch = [(inc, ph, GAINS[i % 8]) for i, (inc, ph) in enumerate((inc, ph) for inc in INCS for ph in (0, 0xDEADBEEF))]
    _same(eng, _rows(16, 6000, 30), ch, 4, TAPS_UP)

def test_the_limits_at_once(eng):
    """Every branch of the taps sums to exactly 65535 on rail input, and 16 channels at gain 65535 in phase: the accumulator reaches its
    extremes without wrapping and the final sat16 clips."""
    U = 4; t = np.zeros(63, np.int64)
    for r in range(U):
        idx = np.arange(r, 63, U); t[idx] = 65535 // len(idx); t[idx[0]] += 65535 - t[idx].sum()
    t = t.astype(np.int16); assert all(np.abs(t[r::U].astype(np.int64)).sum() == 65535 for r in range(U))
    x = np.where(np.random.default_rng(41).random((3000, 2)) < 0.5, -32768, 32767).astype(np.int16); x[1000:1100] = -32768
    rows = np.stack([x] * 16); ch = [(2 ** 30, 0, 65535)] * 16
    got = eng.combine(rows, ch, U, t)
    assert (got == CM.combine(rows, ch, U, t)).all() and (np.abs(got.astype(np.int64)) >= 32767).mean() > 0.5


# ---- long captures --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,U,ntaps", [(4, 4, 127), (16, 16, 255), (7, 1, 255), (16, 3, 101), (2, 15, 253)])
def test_long_captures(eng, K, U, ntaps):
    """At least 4 x SMs tiles plus 777 samples, on the device; the first, middle and last outputs against combine_window."""
    n = (4 * _sms() + 3) * _tile(K, U, ntaps) + 777; stride = (n + 3) // 4 * 4
    rows = np.zeros((K, stride, 2), np.int16); rows[:, :n] = _rows(K, n, 70 + U)
    ch = _channels(K, 70 + U); taps = _taps(ntaps, U, 70 + U)
    d_in = torch.from_numpy(rows).cuda(); d_out = torch.zeros((U * n, 2), dtype=torch.int16, device="cuda")
    eng.combine_raw(d_in.data_ptr(), stride, n, ch, U, taps, d_out.data_ptr())
    for n0, n1 in ((0, 700), (U * n // 2 - 350, U * n // 2 + 350), (U * n - 700, U * n)):
        got = d_out[n0:n1].cpu().numpy(); want = CM.combine_window(rows[:, :n], ch, U, taps, n0, n1)
        assert (got == want).all(), (n0, np.argwhere((got != want).any(1))[:5].ravel())


# ---- the C ABI ------------------------------------------------------------------------------------------------------------------------
def test_residency(eng):
    """rows and out each host or device; rows wider than n_in (the samples between them are not read), the bytes after out untouched."""
    K, n, stride, U = 3, 1001, 1008, 4
    rows = np.full((K, stride, 2), 0x5A5A, np.int16); rows[:, :n] = _rows(K, n, 50); ch = _channels(K, 50)
    args = dict(rows=rows, out=_fill(U * n * 4 + 16))
    ref = _matrix(lambda p: eng.combine_raw(p["rows"], stride, n, ch, U, TAPS_UP, p["out"]), args, _each(*args))
    assert (ref["out"][:U * n * 4].view(np.int16).reshape(-1, 2) == CM.combine(rows[:, :n], ch, U, TAPS_UP)).all()
    assert (ref["out"][U * n * 4:] == 0xA5).all()

def test_a_callers_stream(eng):
    K, n, U = 4, 30001, 4; rows = _rows(K, n + 3, 51)[:, :n + 3]; ch = _channels(K, 51)
    d_in = torch.from_numpy(np.ascontiguousarray(rows)).cuda(); s = torch.cuda.Stream(); s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        d_out = torch.zeros((U * n, 2), dtype=torch.int16, device="cuda")
        eng.combine_raw(d_in.data_ptr(), n + 3, n, ch, U, TAPS_UP, d_out.data_ptr(), s.cuda_stream)
        got = d_out.cpu().numpy()
    assert (got == CM.combine(rows[:, :n], ch, U, TAPS_UP)).all()

def test_one_launch_and_timing():
    e = api.Engine(0)
    try:
        rows = _rows(5, 50000, 60)
        for _ in range(2):
            n0 = e.launches; e.combine(rows, _channels(5, 60), 4, TAPS_UP)
            assert e.launches - n0 == 1 and e.last_kernel_ms() > 0
    finally:
        e.close()

def _call(eng, rows, stride, n, ch, nch, u, taps, ntaps, out):
    return eng._lib.sb200_combine(eng._h, V(rows), U64(stride), U64(n), V(ch), U32(nch), U32(u), V(taps), U32(ntaps), V(out), V(0))

def test_invalid_arguments_are_rejected(eng):
    x = _rows(17, 1000, 70); out = np.zeros((4 * 1000, 2), np.int16)
    ch = (api.DucChannel * 17)(*[api.DucChannel(i << 24, 0, 4096) for i in range(17)])
    hot = (api.DucChannel * 2)(api.DucChannel(0, 0, 4096), api.DucChannel(0, 0, 65536))
    t = np.array(TAPS_UP); xp, op, cp, tp = x.ctypes.data, out.ctypes.data, C.addressof(ch), t.ctypes.data
    assert _call(eng, xp, 1000, 1000, cp, 4, 4, tp, 127, op) == 0
    branch = np.zeros(9, np.int16); branch[0::4] = 21845; branch[0] = 21846          # taps 0, 4, 8: 65536; the total is legal elsewhere
    assert np.abs(branch.astype(np.int64)).sum() == 65536
    ok_total = np.zeros(9, np.int16); ok_total[0::4] = 21845; ok_total[1::4] = 21845 // 2     # every branch <= 65535, the total above it
    n0 = eng.launches
    bad = {"nchannels 0": (xp, 1000, 1000, cp, 0, 4, tp, 127, op), "nchannels 17": (xp, 1000, 1000, cp, 17, 4, tp, 127, op),
           "interp 0": (xp, 1000, 1000, cp, 4, 0, tp, 127, op), "interp 17": (xp, 1000, 1000, cp, 4, 17, tp, 127, op),
           "ntaps even": (xp, 1000, 1000, cp, 4, 4, tp, 126, op), "ntaps 257": (xp, 1000, 1000, cp, 4, 4, np.zeros(257, np.int16).ctypes.data, 257, op),
           "branch sum": (xp, 1000, 1000, cp, 4, 4, branch.ctypes.data, 9, op), "gain 65536": (xp, 1000, 1000, C.addressof(hot), 2, 4, tp, 127, op),
           "stride < n_in": (xp, 996, 1000, cp, 4, 4, tp, 127, op), "stride % 4": (xp, 1002, 1000, cp, 4, 4, tp, 127, op),
           "stride > 2^40": (xp, (1 << 40) + 4, 1000, cp, 4, 4, tp, 127, op), "interp * n_in > 2^40": (xp, (1 << 38) + 4, (1 << 38) + 4, cp, 1, 4, tp, 127, op),
           "null rows": (0, 1000, 1000, cp, 4, 4, tp, 127, op), "null channels": (xp, 1000, 1000, 0, 4, 4, tp, 127, op),
           "null taps": (xp, 1000, 1000, cp, 4, 4, 0, 127, op), "null out": (xp, 1000, 1000, cp, 4, 4, tp, 127, 0)}
    for name, a in bad.items():
        assert _call(eng, *a) == -1, name
    d = torch.zeros(4 * 1000 * 2 + 8, dtype=torch.int16, device="cuda")
    assert _call(eng, d.data_ptr() + 4, 1000, 999, cp, 1, 4, tp, 127, op) == -1, "misaligned device rows"
    assert _call(eng, xp, 1000, 1000, cp, 1, 4, tp, 127, d.data_ptr() + 4) == -1, "misaligned device output"
    assert eng.launches == n0, "a refused call launched"
    assert _call(eng, xp, 1000, 1000, cp, 4, 4, ok_total.ctypes.data, 9, op) == 0                 # the limit is per branch, not on the total
    branch[0] -= 1
    assert _call(eng, xp, 1000, 1000, cp, 4, 4, branch.ctypes.data, 9, op) == 0                   # a branch at 65535 is accepted
    assert _call(eng, xp, 1000, 1000, C.addressof(hot), 1, 4, tp, 127, op) == 0              # only the first channel, gain 4096


# ---- end to end, device-resident: transmitter -> combiner -> channelizer -> stream receivers -------------------------------------------
def _dev_chain(eng, rows, n, ch, taps_up, taps_down):
    """rows (device [K, stride, 2]) -> combined on the device (interp 4) -> channelized (decim 4) into device rows; returns (y, rows, stride)."""
    K = len(ch); y = torch.zeros((4 * n, 2), dtype=torch.int16, device="cuda")
    eng.combine_raw(rows.data_ptr(), rows.shape[1], n, ch, 4, taps_up, y.data_ptr())
    back = WD.dev_rows(K, n, 64); stride = back.shape[1]
    eng.channelize_raw(y.data_ptr(), 4 * n, [(a, b) for a, b, _ in ch], 4, taps_down, back.data_ptr(), stride)
    return y, back, stride

def test_round_trip_11a_on_the_device():
    rows_h, mpdus, plan = frames_11a(); K, n = rows_h.shape[:2]
    y_h, back_h, _ = wide_11a()
    ch = [(W.phase_inc(f, W.FS_11A_WIDE), 0, g) for f, g in zip(W.CH_11A, GAIN_11A)]
    e = api.Engine(0, cca_pwr_threshold=CCA_WIDE)
    try:
        rows = WD.dev_rows(K, n)
        for c, pl in enumerate(plan):
            for (t, rate, seed), m in zip(pl, mpdus[c]):
                f = WD.tx11a(e, m, rate, seed); rows[c, t:t + len(f)] = f.to(torch.int16) * 20
        assert (rows[:, :n].cpu().numpy() == rows_h).all()
        y, back, stride = _dev_chain(e, rows, n, ch, TAPS_UP, TAPS_11A)
        assert (y.cpu().numpy() == y_h).all() and (back[:, :n].cpu().numpy() == back_h).all()
        got = WD.rx11a(e, back, stride, n, K)
    finally:
        e.close()
    for c, (o, _) in enumerate(WD.equal_11a(back_h, got)):
        assert len(o) == 3 and (o["status"] == oracle_py.E_FRAME_OK).all(), (c, o)

def test_round_trip_11b_on_the_device(eng):
    rows_h, mpdus, plan = frames_11b(); K, n = rows_h.shape[:2]
    y_h, back_h, _ = wide_11b()
    ch = [(W.phase_inc(f, W.FS_11B_WIDE), 0, 4096) for f in W.CH_11B]
    rows = WD.dev_rows(K, n)
    for c, pl in enumerate(plan):
        for (t, rate), m in zip(pl, mpdus[c]):
            f = WD.tx11b(eng, m, rate); rows[c, t:t + len(f)] = f.to(torch.int16) * 64
    assert (rows[:, :n].cpu().numpy() == rows_h).all()
    y, back, stride = _dev_chain(eng, rows, n, ch, TAPS_UP_11B, TAPS_11B)
    assert (y.cpu().numpy() == y_h).all() and (back[:, :n].cpu().numpy() == back_h).all()
    for c, (o, _) in enumerate(WD.equal_11b(back_h, WD.rx11b(eng, back, stride, n, K))): assert len(o) == 2, (c, o)

def test_round_trip_11n_on_the_device(eng):
    r0_h, r1_h, mpdus, plan = frames_11n(); K, n = r0_h.shape[:2]
    (y0_h, y1_h), (b0_h, b1_h), _ = wide_11n()
    ch = [(W.phase_inc(f, W.FS_11A_WIDE), 0, 4096) for f in W.CH_11N]
    r0, r1 = WD.dev_rows(K, n), WD.dev_rows(K, n)
    for c, pl in enumerate(plan):
        for (t, seed), m in zip(pl, mpdus[c]):
            a, b = WD.tx11n(eng, m, 9, seed); r0[c, t:t + len(a)] = a; r1[c, t:t + len(b)] = b
    assert (r0[:, :n].cpu().numpy() == r0_h).all() and (r1[:, :n].cpu().numpy() == r1_h).all()
    y0, d0, stride = _dev_chain(eng, r0, n, ch, TAPS_UP, TAPS_11A)
    y1, d1, _ = _dev_chain(eng, r1, n, ch, TAPS_UP, TAPS_11A)
    assert (y0.cpu().numpy() == y0_h).all() and (y1.cpu().numpy() == y1_h).all()
    assert (d0[:, :n].cpu().numpy() == b0_h).all() and (d1[:, :n].cpu().numpy() == b1_h).all()
    for c, (o, _) in enumerate(WD.equal_11n(b0_h, b1_h, WD.rx11n(eng, d0, d1, stride, n, K))): assert len(o) == 2, (c, o)
