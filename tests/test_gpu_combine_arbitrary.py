"""GPU tests of the arbitrary-rate combiner (sb200_combine_arbitrary, pytest -m gpu): bit for bit against the numpy model of
tests/combine_arbitrary_model.py over lengths around every tile size the call picks, steps, tau0, table lengths, channel counts, gains,
accumulate and full-scale input; one identity row against sb200_channelize_arbitrary on the device; the pointer residency, stream, launch
bookkeeping and argument checks of the C ABI, and the table the two arbitrary-rate calls share; and the 2.4 GHz transmit chain of
test_cpu_combine_arbitrary.py on the device (transmitters -> two combiner calls into one 122.88 Msps buffer -> channel simulator with noise
-> arbitrary-rate channelizer -> stream receivers, all device-resident) against the model and the CPU oracle."""
import ctypes as C
import numpy as np, pytest
import torch
import wideband_inputs as W
import wideband_device as WD
import arbitrary_model as A
import combine_arbitrary_model as CA
import rational_model as R
from sora_b200 import api
from test_gpu_abi_residency import _matrix, _each, _fill
from test_gpu_channelize_arbitrary import _table
from test_cpu_channelize import CCA_WIDE, _full_scale
from test_cpu_channelize_arbitrary import FS, STEP_40, STEP_44, TAPS_40, TAPS_44, _unit
from test_cpu_combine_arbitrary import UP_40, UP_44, UP_TAPS_40, UP_TAPS_44, GAIN_A, GAIN_B, capture_122_88, channelize_122_88
from test_cpu_combine_rational import SIM_LINK_24, SIM_TAPS_24, SIM_SEED_24, frames_24ghz, through_the_air
from test_cpu_combine import _psdus
from wideband_device import GAINS, duc_channels as _channels, duc_rows as _rows, sms as _sms

pytestmark = pytest.mark.gpu
V, U32, U64 = C.c_void_p, C.c_uint32, C.c_uint64
UP_30 = api.arbitrary_step(44e6, 30.72e6)              # 44 -> 30.72 Msps: step 1.43 2^32
STEPS = [1 << 28, (1 << 32) - 1, (1 << 32) + 1, 1 << 34, UP_40, UP_30]

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

def _tm(K, step, ntaps, rot):
    """Outputs per tile that sb200_combine_arbitrary picks: the largest of 1024, 512 whose shared memory fits 57344 bytes, else 256."""
    rs = ((ntaps + 1) // 2) | 1
    for tm in (1024, 512):
        win = ((((tm - 1) * step) >> 32) + 1 + ntaps + 1 + 3 + 3) & ~3
        if ((4096 if rot else 0) + 256 * rs + K * win) * 4 + 16 <= 57344: return tm
    return 256

def _same(eng, rows, ch, tau0, step, taps, n_out, acc=None):
    out = None if acc is None else np.array(acc, np.int16)
    got = eng.combine_arbitrary(rows, ch, step, taps, tau0=tau0, n_out=n_out, accumulate=acc is not None, out=out)
    want = CA.combine_arbitrary(rows, ch, tau0, step, taps, n_out, acc)
    assert got.shape == want.shape and (got == want).all(), (step, tau0, np.argwhere((got != want).any(1))[:5].ravel())

# (K, step, ntaps, rotating channel) -> the tile the call picks: 1024 outputs, 512, and 256 past the budget
TILES = [(3, UP_44, 64, True, 1024), (16, UP_40, 8, False, 1024), (2, 1 << 32, 64, True, 512), (2, 1 << 34, 64, False, 512),
         (16, 1 << 28, 64, True, 512), (16, 1 << 32, 64, True, 256), (1, 1 << 34, 64, True, 256), (16, 1 << 34, 64, True, 256)]

@pytest.mark.parametrize("K,step,ntaps,rot,tm", TILES)
def test_every_tile_size_around_its_edges(eng, K, step, ntaps, rot, tm):
    """n_out of 1 and around one to three tiles of the size the call picks, on rows just long enough for them (zeros past them)."""
    assert _tm(K, step, ntaps, rot) == tm
    ch = [(2 ** 30, 12345, 4096)] + _channels(K - 1, tm + K) if rot else [(0, i << 16, GAINS[i % 8]) for i in range(K)]
    assert any(a or b >> 20 for a, b, _ in ch) == rot
    for n_out in (1, 2, tm - 1, tm, tm + 1, 3 * tm + 2):
        n_in = max(1, (n_out * step >> 32) - 5)
        _same(eng, _rows(K, n_in, n_out + K), ch, 12345, step, _table(ntaps, n_out + ntaps), n_out)

@pytest.mark.parametrize("n_out", [1, 2, 1023, 1024, 1025, 3074, 10001])
@pytest.mark.parametrize("step", STEPS)
def test_lengths_and_steps(eng, n_out, step):
    """Outputs around tile edges at every kind of step: x16, either side of 2^32, /4, 40 -> 122.88 and 44 -> 30.72 Msps."""
    n_in = max(1, (n_out * step >> 32) - 5)
    _same(eng, _rows(3, n_in, n_out + step % 997), _channels(3, n_out), 12345, step, _table(64, n_out), n_out)

def test_tau0(eng):
    """tau0 of 0, fractional, whole and past the rows, and at the 2^63 bound: tau0 + (n_out - 1) step = 2^63 - 1."""
    rows = _rows(2, 5000, 410); t = _table(64, 410)
    for tau0 in (0, 1, 0x7FFFFF, 0x800000, 3 * 2 ** 32 + 0xABCDEF, 4000 << 32, 6000 << 32):
        _same(eng, rows, _channels(2, tau0 % 97), tau0, UP_44, t, 3000)
    for step in (1 << 28, 1 << 34, UP_40):
        n_out = 3 * 1024 + 7; tau0 = 2 ** 63 - 1 - (n_out - 1) * step
        _same(eng, rows, [(0, 0, 4096), (2 ** 30, 5, 65535)], tau0, step, t, n_out)     # every row far behind: zeros from the top of uint64's half

@pytest.mark.parametrize("ntaps", [1, 2, 7, 8, 33, 63, 64])
def test_table_lengths(eng, ntaps):
    rows = _rows(4, 3001, 420 + ntaps)
    for step in STEPS:
        _same(eng, rows, _channels(4, ntaps), 7 << 29, step, _table(ntaps, ntaps + step % 89), A.n_inside(3001, 7 << 29, step) + 50)

@pytest.mark.parametrize("k", [1, 2, 5, 16])
def test_rows_identity_and_rotation(eng, k):
    """1 .. 16 rows mixing the identity channel with rotating ones, all identity, and all rotating; gains 0 .. 65535."""
    rows = _rows(k, 4000, 430 + k)
    _same(eng, rows, _channels(k, 430 + k), 0, UP_44, UP_TAPS_44, None)
    _same(eng, rows, [(0, i << 16, GAINS[i % 8]) for i in range(k)], 0, UP_40, UP_TAPS_40, None)
    _same(eng, rows, [(2 ** 29 * (i + 1), 0xDEADBEEF, GAINS[(i + 2) % 8]) for i in range(k)], 3 << 31, 1 << 30, _table(17, k), 30000)

def test_rails_and_row_sums_at_the_limit(eng):
    """Every row's sum |H| exactly 65535 on rail input, 16 rows at gain 65535 in phase, with and without accumulate onto rails: each
    accumulator reaches its extremes without wrapping and the final sat16 clips."""
    t = _table(64, 440, 65535).astype(np.int64)
    for p in range(256):
        j = np.argmax(np.abs(t[p])); t[p, j] += np.sign(t[p, j]) * (65535 - np.abs(t[p]).sum())
    assert (np.abs(t).sum(1) == 65535).all() and np.abs(t).max() <= 32767
    t = t.astype(np.int16)
    x = np.where(np.random.default_rng(441).random((3000, 2)) < 0.5, -32768, 32767).astype(np.int16)
    x[1000:1300] = np.where(t[0][np.arange(300) % 64] < 0, -32768, 32767)[:, None]
    rows = np.stack([x] * 16); rng = np.random.default_rng(442)
    for step in (1 << 28, 1 << 32, UP_44, 1 << 34):
        for ch in ([(2 ** 30, 0, 65535)] * 16, [(0, 0, 65535)] * 16, [(0, 0, 4096), (2 ** 31, 0, 65535)]):
            n_out = A.n_inside(3000, 0, step)
            _same(eng, rows[:len(ch)], ch, 0, step, t, n_out)
            _same(eng, rows[:len(ch)], ch, 0, step, t, n_out, np.where(rng.random((n_out, 2)) < 0.5, -32768, 32767))
    got = eng.combine_arbitrary(rows, [(2 ** 30, 0, 65535)] * 16, UP_44, t)
    assert (np.abs(got.astype(np.int64)) >= 32767).mean() > 0.5

def test_accumulate(eng):
    """accumulate onto random and rail contents, host and device output."""
    rows = _rows(3, 2000, 450); ch = _channels(3, 450); n = A.n_inside(2000, 0, UP_44) + 17
    rng = np.random.default_rng(451)
    for acc in (rng.integers(-32768, 32768, (n, 2)), np.where(rng.random((n, 2)) < 0.5, -32768, 32767)):
        acc = acc.astype(np.int16)
        _same(eng, rows, ch, 0, UP_44, UP_TAPS_44, n, acc)
        d_in = torch.from_numpy(np.ascontiguousarray(rows)).cuda(); d_out = torch.from_numpy(acc).cuda()
        eng.combine_arbitrary_raw(d_in.data_ptr(), 2000, 2000, ch, 0, UP_44, UP_TAPS_44, d_out.data_ptr(), n, accumulate=True)
        assert (d_out.cpu().numpy() == CA.combine_arbitrary(rows, ch, 0, UP_44, UP_TAPS_44, n, acc)).all()


# ---- long captures --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,step,ntaps", [(3, UP_44, 64), (1, UP_40, 64), (16, 1 << 34, 64), (16, 1 << 28, 33)])
def test_long_captures(eng, K, step, ntaps):
    """At least 4 x SMs tiles plus 777 outputs, on the device; the first, middle and last outputs against combine_arbitrary_window."""
    taps = UP_TAPS_44 if step == UP_44 else UP_TAPS_40 if step == UP_40 else _table(ntaps, 460 + K)
    ch = _channels(K, 460 + K); tm = _tm(K, step, ntaps, True)
    n_out = (4 * _sms() + 3) * tm + 777; n = (n_out * step >> 32) + 100; stride = WD.ceil4(n)
    rows = np.zeros((K, stride, 2), np.int16); rows[:, :n] = _rows(K, n, 470 + K)
    d_in = torch.from_numpy(rows).cuda(); d_out = torch.zeros((n_out, 2), dtype=torch.int16, device="cuda")
    eng.combine_arbitrary_raw(d_in.data_ptr(), stride, n, ch, 0, step, taps, d_out.data_ptr(), n_out)
    for n0, n1 in ((0, 700), (n_out // 2 - 350, n_out // 2 + 350), (n_out - 700, n_out)):
        got = d_out[n0:n1].cpu().numpy(); want = CA.combine_arbitrary_window(rows[:, :n], ch, 0, step, taps, n0, n1)
        assert (got == want).all(), (step, n0, np.argwhere((got != want).any(1))[:5].ravel())


# ---- the other calls on the device ----------------------------------------------------------------------------------------------------
def test_one_identity_row_is_the_channelizer_on_the_device(eng):
    """One row through channel {0, 0, 4096} without accumulate equals sb200_channelize_arbitrary's channel (0, 0), device against device,
    with the same tau0, step, table and n_out; and with the unit-impulse row 0 at step 2^32 it is a pure shift."""
    x = _full_scale(20001, 480); d_in = torch.from_numpy(np.concatenate([x, np.zeros((3, 2), np.int16)])).cuda()
    for tau0, step, t in ((0, UP_44, UP_TAPS_44), (12345, STEP_44, TAPS_44), (3 << 31, 1 << 28, _table(33, 481)), (77, 1 << 34, _table(8, 482)), (5 << 32, 1 << 32, _unit(64))):
        n_out = A.n_inside(20001, tau0, step) + 30
        a = torch.zeros((n_out + 4, 2), dtype=torch.int16, device="cuda"); b = torch.zeros((1, WD.ceil4(n_out), 2), dtype=torch.int16, device="cuda")
        eng.combine_arbitrary_raw(d_in.data_ptr(), 20004, 20001, [(0, 0, 4096)], tau0, step, t, a.data_ptr(), n_out)
        eng.channelize_arbitrary_raw(d_in.data_ptr(), 20001, [(0, 0)], tau0, step, t, b.data_ptr(), b.shape[1], n_out)
        assert (a[:n_out].cpu() == b[0, :n_out].cpu()).all(), (tau0, step)
        if step == 1 << 32: assert (a[:20001 - 5].cpu().numpy() == x[5:]).all() and (a[20001 - 5:n_out].cpu() == 0).all()


# ---- the C ABI ------------------------------------------------------------------------------------------------------------------------
def test_residency(eng):
    """rows and out each host or device, with and without accumulate (a host out is uploaded first); the bytes around out untouched; then
    page-locked rows."""
    K, n, stride = 3, 1001, 1008; n_out = A.n_inside(n, 0, UP_44)
    rows = np.full((K, stride, 2), 0x5A5A, np.int16); rows[:, :n] = _rows(K, n, 490); ch = _channels(K, 490)
    want = CA.combine_arbitrary(rows[:, :n], ch, 0, UP_44, UP_TAPS_44, n_out)
    args = dict(rows=rows, out=_fill(16 + n_out * 4 + 16))
    ref = _matrix(lambda p: eng.combine_arbitrary_raw(p["rows"], stride, n, ch, 0, UP_44, UP_TAPS_44, p["out"] + 16, n_out), args, _each(*args))
    assert (ref["out"][16:16 + n_out * 4].view(np.int16).reshape(-1, 2) == want).all()
    assert (ref["out"][:16] == 0xA5).all() and (ref["out"][16 + n_out * 4:] == 0xA5).all()
    acc = ref["out"].copy(); args = dict(rows=rows, out=acc)
    ref2 = _matrix(lambda p: eng.combine_arbitrary_raw(p["rows"], stride, n, ch, 0, UP_44, UP_TAPS_44, p["out"] + 16, n_out, accumulate=True), args, _each(*args))
    want2 = CA.combine_arbitrary(rows[:, :n], ch, 0, UP_44, UP_TAPS_44, n_out, acc[16:16 + n_out * 4].view(np.int16).reshape(-1, 2))
    assert (ref2["out"][16:16 + n_out * 4].view(np.int16).reshape(-1, 2) == want2).all()
    assert (ref2["out"][:16] == 0xA5).all() and (ref2["out"][16 + n_out * 4:] == 0xA5).all()
    pinned = torch.from_numpy(rows).pin_memory(); out = np.zeros((n_out, 2), np.int16)
    eng.combine_arbitrary_raw(pinned.data_ptr(), stride, n, ch, 0, UP_44, UP_TAPS_44, out.ctypes.data, n_out)
    pinned.zero_()                                                                                  # the call has finished reading it
    assert (out == want).all()

def test_a_callers_stream(eng):
    """Asynchronous on device buffers: calls queued on a caller's stream, then a zeroing queued behind them, then one more call."""
    K, n = 3, 30001; rows = _rows(K, n + 3, 500); ch = _channels(K, 500); n_out = A.n_inside(n, 0, UP_44)
    want = CA.combine_arbitrary(rows[:, :n], ch, 0, UP_44, UP_TAPS_44, n_out)
    d_in = torch.from_numpy(np.ascontiguousarray(rows)).cuda(); s = torch.cuda.Stream(); s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        d_out = torch.zeros((n_out, 2), dtype=torch.int16, device="cuda")
        for _ in range(3): eng.combine_arbitrary_raw(d_in.data_ptr(), n + 3, n, ch, 0, UP_44, UP_TAPS_44, d_out.data_ptr(), n_out, stream=s.cuda_stream)
        d_out.zero_()                                                                               # queued behind the calls on the same stream
        eng.combine_arbitrary_raw(d_in.data_ptr(), n + 3, n, ch, 0, UP_44, UP_TAPS_44, d_out.data_ptr(), n_out, stream=s.cuda_stream)
    s.synchronize()
    assert (d_out.cpu().numpy() == want).all()

def test_both_arbitrary_calls_on_two_streams(eng):
    """sb200_channelize_arbitrary and sb200_combine_arbitrary back to back on one handle, on two streams, with different tables: both stage
    their table into the handle's one buffer, and each result equals its model."""
    x = _full_scale(40001, 510); rows = _rows(2, 14000, 511); chc = _channels(2, 511); chd = [(W.phase_inc(-25e6, FS), 0), (0, 0)]
    n_c = A.n_inside(14000, 0, UP_44); n_d = A.n_inside(40001, 0, STEP_40)
    d_x = torch.from_numpy(np.concatenate([x, np.zeros((3, 2), np.int16)])).cuda(); d_r = torch.from_numpy(rows).cuda()
    yc = torch.zeros((n_c, 2), dtype=torch.int16, device="cuda"); yd = torch.zeros((2, WD.ceil4(n_d), 2), dtype=torch.int16, device="cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream(); torch.cuda.synchronize()
    for _ in range(3):
        eng.channelize_arbitrary_raw(d_x.data_ptr(), 40001, chd, 0, STEP_40, TAPS_40, yd.data_ptr(), yd.shape[1], n_d, stream=s1.cuda_stream)
        eng.combine_arbitrary_raw(d_r.data_ptr(), 14000, 14000, chc, 0, UP_44, UP_TAPS_44, yc.data_ptr(), n_c, stream=s2.cuda_stream)
    s1.synchronize(); s2.synchronize()
    assert (yc.cpu().numpy() == CA.combine_arbitrary(rows, chc, 0, UP_44, UP_TAPS_44, n_c)).all()
    assert (yd[:, :n_d].cpu().numpy() == A.channelize_arbitrary(x, chd, 0, STEP_40, TAPS_40, n_d)).all()

def test_one_launch_and_timing():
    e = api.Engine(0)
    try:
        rows = _rows(3, 50000, 520)
        for acc in (False, True):
            n0 = e.launches; e.combine_arbitrary(rows, _channels(3, 520), UP_44, UP_TAPS_44, accumulate=acc)
            assert e.launches - n0 == 1 and e.last_kernel_ms() > 0
    finally:
        e.close()

def _call(eng, rows, stride, n, ch, nch, tau0, step, taps, ntaps, out, n_out, acc=0):
    return eng._lib.sb200_combine_arbitrary(eng._h, V(rows), U64(stride), U64(n), V(ch), U32(nch), U64(tau0), U64(step), V(taps), U32(ntaps), V(out), U64(n_out), U32(acc), V(0))

def test_invalid_arguments_are_rejected(eng):
    """Every refused argument returns SB200_E_INVALID with a message naming it and launches nothing."""
    x = _rows(17, 1000, 530); out = np.zeros((4000, 2), np.int16)
    ch = (api.DucChannel * 17)(*[api.DucChannel(i << 24, 0, 4096) for i in range(17)])
    hot = (api.DucChannel * 2)(api.DucChannel(0, 0, 4096), api.DucChannel(0, 0, 65536))
    t = np.ascontiguousarray(_table(64, 530)); xp, op, cp, tp = x.ctypes.data, out.ctypes.data, C.addressof(ch), t.ctypes.data
    S = UP_44; n_out = A.n_inside(1000, 0, S)
    assert _call(eng, xp, 1000, 1000, cp, 4, 0, S, tp, 64, op, n_out) == 0
    over = np.zeros((256, 8), np.int16); over[:, 3] = 16384; over[200, :4] = 16384                # row 200: 65536
    at = np.zeros((256, 8), np.int16); at[:, 3] = 16384; at[200, :4] = 16384; at[200, 0] = 16383     # row 200: 65535
    edge = 2 ** 63 - (n_out - 1) * S                                                                # tau0 + (n_out - 1) step = 2^63
    n_events = eng.launches
    bad = {"nchannels 0": ((xp, 1000, 1000, cp, 0, 0, S, tp, 64, op, n_out), "nchannels"), "nchannels 17": ((xp, 1000, 1000, cp, 17, 0, S, tp, 64, op, n_out), "nchannels"),
           "ntaps 0": ((xp, 1000, 1000, cp, 4, 0, S, tp, 0, op, n_out), "ntaps"), "ntaps 65": ((xp, 1000, 1000, cp, 4, 0, S, tp, 65, op, n_out), "ntaps"),
           "step < 2^28": ((xp, 1000, 1000, cp, 4, 0, 2 ** 28 - 1, tp, 64, op, n_out), "step"), "step > 2^34": ((xp, 1000, 1000, cp, 4, 0, 2 ** 34 + 1, tp, 64, op, n_out), "step"),
           "t reaches 2^63": ((xp, 1000, 1000, cp, 4, edge, S, tp, 64, op, n_out), "tau0"), "tau0 >= 2^63": ((xp, 1000, 1000, cp, 4, 2 ** 63, S, tp, 64, op, 1), "tau0"),
           "row sum": ((xp, 1000, 1000, cp, 4, 0, S, over.ctypes.data, 8, op, n_out), "sum of |taps|"),
           "gain 65536": ((xp, 1000, 1000, C.addressof(hot), 2, 0, S, tp, 64, op, n_out), "gain"),
           "accumulate 2": ((xp, 1000, 1000, cp, 4, 0, S, tp, 64, op, n_out, 2), "accumulate"),
           "stride < n_in": ((xp, 996, 1000, cp, 4, 0, S, tp, 64, op, n_out), "row_stride"), "stride % 4": ((xp, 1002, 1000, cp, 4, 0, S, tp, 64, op, n_out), "row_stride"),
           "stride > 2^40": ((xp, (1 << 40) + 4, 1000, cp, 4, 0, S, tp, 64, op, n_out), "row_stride"),
           "n_in > 2^40": ((xp, 1 << 40, (1 << 40) + 1, cp, 4, 0, S, tp, 64, op, n_out), "n_in"),
           "n_out > 2^40": ((xp, 1000, 1000, cp, 4, 0, 1 << 28, tp, 64, op, (1 << 40) + 1), "n_out"),
           "null rows": ((0, 1000, 1000, cp, 4, 0, S, tp, 64, op, n_out), "null"), "null channels": ((xp, 1000, 1000, 0, 4, 0, S, tp, 64, op, n_out), "null"),
           "null taps": ((xp, 1000, 1000, cp, 4, 0, S, 0, 64, op, n_out), "null"), "null out": ((xp, 1000, 1000, cp, 4, 0, S, tp, 64, 0, n_out), "null")}
    for name, (a, word) in bad.items():
        assert _call(eng, *a) == -1, name
        assert word in eng._lib.sb200_last_error(eng._h).decode(), (name, eng._lib.sb200_last_error(eng._h))
    d = torch.zeros(4 * 1000 * 2 + 8, dtype=torch.int16, device="cuda")
    assert _call(eng, d.data_ptr() + 4, 1000, 999, cp, 1, 0, S, tp, 64, op, n_out) == -1, "misaligned device rows"
    assert _call(eng, xp, 1000, 1000, cp, 1, 0, S, tp, 64, d.data_ptr() + 4, n_out) == -1, "misaligned device output"
    out[:] = 7
    assert _call(eng, xp, 1000, 1000, cp, 4, 0, S, tp, 64, op, 0) == 0 and (out == 7).all(), "n_out = 0"
    assert eng.launches == n_events, "a refused call (or n_out = 0) launched"
    assert _call(eng, xp, 1000, 1000, cp, 4, edge - 1, S, tp, 64, op, n_out) == 0                   # 2^63 - 1 is accepted
    assert _call(eng, xp, 1000, 1000, cp, 4, 0, S, at.ctypes.data, 8, op, n_out) == 0                # a row sum of 65535 is accepted
    assert _call(eng, xp, 1000, 0, cp, 4, 0, S, tp, 64, op, n_out) == 0                              # n_in = 0: all-zero rows
    assert (out[:n_out] == 0).all()


# ---- end to end, device-resident: transmitters -> two combiner calls -> arbitrary-rate channelizer -> stream receivers -----------------
def test_24ghz_transmit_at_122_88_on_the_device():
    """k_tx11b frames (COMPLEX8 widened on the device) and k_tx11a frames in device rows -> the 802.11b rows at -25 and +25 MHz and then
    the OFDM row at 0 Hz into one 122.88 Msps device buffer -> sb200_channel_sim (one link, one tap of 16384, noise of sigma 20 LSB) ->
    sb200_channelize_arbitrary to 44 and 40 Msps -> sb200_rx11b_streams and sb200_rx11a_streams.  The capture, before and after the
    channel, equals the model chain on the oracle transmitters' output; the receivers equal the oracle on every field, event position and
    delivered byte; every PSDU delivered with FRAME_OK."""
    rows_h, mpdus, plan = frames_24ghz(); clean_h, _ = capture_122_88(rows_h); y_h = through_the_air(clean_h); back = channelize_122_88(y_h)
    e = api.Engine(0); ea = api.Engine(0, cca_pwr_threshold=CCA_WIDE)
    try:
        n_b = max(len(rows_h[0]), len(rows_h[2])); sb_in = WD.ceil4(n_b); n_a = len(rows_h[1]); sa_in = WD.ceil4(n_a)
        rb = torch.zeros((2, sb_in, 2), dtype=torch.int16, device="cuda"); ra_ = torch.zeros((1, sa_in, 2), dtype=torch.int16, device="cuda")
        for i, c in enumerate((0, 2)):
            for (t, rate, _), m in zip(plan[c], mpdus[c]):
                f = WD.tx11b(e, m, rate); rb[i, t:t + len(f)] = f.to(torch.int16) << 6
        for (t, rate, seed), m in zip(plan[1], mpdus[1]):
            f = WD.tx11a(e, m, rate, seed); ra_[0, t:t + len(f)] = f.to(torch.int16) * 20
        n = len(y_h); tx = torch.zeros((n, 2), dtype=torch.int16, device="cuda"); y = torch.zeros_like(tx)     # n is a multiple of 4
        e.combine_arbitrary_raw(rb.data_ptr(), sb_in, n_b, [(W.phase_inc(R.CH_24[c], FS), 0, GAIN_B) for c in (0, 2)], 0, UP_44, UP_TAPS_44, tx.data_ptr(), n)
        e.combine_arbitrary_raw(ra_.data_ptr(), sa_in, n_a, [(0, 0, GAIN_A)], 0, UP_40, UP_TAPS_40, tx.data_ptr(), n, accumulate=True)
        assert (tx.cpu().numpy() == clean_h).all()
        e.channel_sim_raw(tx.data_ptr(), n, n, 1, n, api.sim_links([SIM_LINK_24]), SIM_TAPS_24, 1, 1, SIM_SEED_24, y.data_ptr(), n, n, 1, n)
        assert (y.cpu().numpy() == y_h).all()
        def dev_rows(chans, step, t):
            n_out = A.n_inside(n, 0, step); out = WD.dev_rows(len(chans), n_out, 64); stride = out.shape[1]
            e.channelize_arbitrary_raw(y.data_ptr(), n, [(W.phase_inc(R.CH_24[c], FS), 0) for c in chans], 0, step, t, out.data_ptr(), stride, n_out)
            return out, stride, n_out
        b_ch, a_ch = [0, 2], [1]
        db_, sb, nb = dev_rows(b_ch, STEP_44, TAPS_44); da_, sa, na = dev_rows(a_ch, STEP_40, TAPS_40)
        for i, c in enumerate(b_ch): assert (db_[i, :nb].cpu().numpy() == back[c]).all(), c
        assert (da_[0, :na].cpu().numpy() == back[1]).all()
        got_b = WD.rx11b(e, db_, sb, nb, len(b_ch)); got_a = WD.rx11a(ea, da_, sa, na, len(a_ch))
    finally:
        e.close(); ea.close()
    for i, (c, (o, _)) in enumerate(zip(b_ch, WD.equal_11b([back[c] for c in b_ch], got_b))):
        ps = _psdus(mpdus[c]); assert len(o) == len(ps), (c, len(o))
        assert (got_b[0][i, :len(o)]["status"] == api.FRAME_OK).all(), c
        for j in range(len(o)):
            L = int(o["length"][j]) - 1; assert bytes(got_b[1][i, j, :L]) == ps[j][:-1], (c, j)
    (o, _), = WD.equal_11a([back[1]], got_a); ps = _psdus(mpdus[1])
    assert len(o) == len(ps), len(o)
    assert (got_a[0][0, :len(o)]["status"] == api.FRAME_OK).all()
    for j in range(len(o)):
        L = int(o["length"][j]); assert bytes(got_a[1][0, j, :L]) == ps[j], j
