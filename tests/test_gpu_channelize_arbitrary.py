"""GPU tests of the arbitrary-rate channelizer (sb200_channelize_arbitrary, pytest -m gpu): bit for bit against the numpy model of
tests/arbitrary_model.py over lengths, steps, tau0, table lengths, channel counts and full-scale input; the identity and sb200_channel_sim's
interpolation on the device; the pointer residency, stream, launch bookkeeping and argument checks of the C ABI; the 122.88 Msps capture of
test_cpu_channelize_arbitrary.py channelized and decoded on the device; and the device transmitters taken up to 122.88 Msps and back."""
import ctypes as C
import numpy as np, pytest
import torch
import wideband_inputs as W
import wideband_device as WD
import arbitrary_model as A
from sora_b200 import api
from test_gpu_abi_residency import _matrix, _each, _fill
from test_cpu_channelize import CCA_WIDE, _full_scale
from test_cpu_channelize_arbitrary import FS, STEP_40, STEP_44, TAPS_40, TAPS_44, rows_24ghz, _unit
from wideband_device import GROUP_CH, ddc_channels as _channels

pytestmark = pytest.mark.gpu
V, U32, U64 = C.c_void_p, C.c_uint32, C.c_uint64
TM = 1024                                              # outputs per tile
STEPS = [1 << 28, (1 << 32) - 1, (1 << 32) + 1, 1 << 34, STEP_44]

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

def _table(ntaps, seed, total=40000):
    """256 random rows of ntaps Q14 taps, every row's sum |H| about `total` (at most 65535)."""
    rng = np.random.default_rng(seed); t = rng.integers(-2000, 2000, (256, ntaps)).astype(np.float64); t[:, (ntaps - 1) // 2] = 9000.0
    return np.trunc(t * total / np.abs(t).sum(1, keepdims=True)).astype(np.int16)

def _same(eng, x, ch, tau0, step, taps, n_out):
    got = eng.channelize_arbitrary(x, ch, step, taps, tau0=tau0, n_out=n_out); want = A.channelize_arbitrary(x, ch, tau0, step, taps, n_out)
    assert got.shape == want.shape and (got == want).all(), (step, tau0, [(i, np.argwhere((got[i] != want[i]).any(1))[:3].ravel()) for i in range(len(ch)) if (got[i] != want[i]).any()])

@pytest.mark.parametrize("n_out", [1, 2, TM - 1, TM, TM + 1, 3 * TM + 2, 10001])
@pytest.mark.parametrize("step", STEPS)
def test_lengths_and_steps(eng, n_out, step):
    """Outputs around tile edges at every kind of step, on a capture just long enough for them (and zeros past it)."""
    n_in = max(1, (n_out * step >> 32) - 5)
    x = _full_scale(n_in, n_out + step % 997)
    _same(eng, x, _channels(3, n_out), 12345, step, _table(64, n_out), n_out)

@pytest.mark.parametrize("ntaps", [1, 2, 7, 8, 33, 64])
def test_table_lengths(eng, ntaps):
    x = _full_scale(9001, 300 + ntaps)
    for step in STEPS:
        _same(eng, x, _channels(4, ntaps), 7 << 29, step, _table(ntaps, ntaps + step % 89), A.n_inside(9001, 7 << 29, step) + 50)

def test_tau0(eng):
    """tau0 of 0, fractional, whole and past the input, and at the 2^63 bound: tau0 + (n_out - 1) step = 2^63 - 1."""
    x = _full_scale(5000, 310); t = _table(64, 310)
    for tau0 in (0, 1, 0x7FFFFF, 0x800000, 3 * 2 ** 32 + 0xABCDEF, 4000 << 32, 6000 << 32):
        _same(eng, x, _channels(2, tau0 % 97), tau0, STEP_44, t, 3000)
    for step in (1 << 28, 1 << 34, STEP_40):
        n_out = 3 * TM + 7; tau0 = 2 ** 63 - 1 - (n_out - 1) * step
        _same(eng, x, [(0, 0), (2 ** 30, 5)], tau0, step, t, n_out)         # every input far behind: zeros, computed from the top of uint64's half

@pytest.mark.parametrize("k", [1, 2, 5, 16])
def test_channels_identity_and_rotation(eng, k):
    """1 .. 16 channels mixing the identity (NCO[0]) with rotating ones, all identity, and all rotating."""
    x = _full_scale(20000, 320 + k)
    _same(eng, x, GROUP_CH[:k], 0, STEP_44, TAPS_44, A.n_inside(20000, 0, STEP_44))
    _same(eng, x, [(0, i << 16) for i in range(k)], 0, STEP_40, TAPS_40, A.n_inside(20000, 0, STEP_40))
    _same(eng, x, [(2 ** 29 * (i + 1), 0xDEADBEEF) for i in range(k)], 3 << 31, 1 << 30, _table(17, k), 30000)

def test_rails_and_row_sums_at_the_limit(eng):
    """Every row's sum |H| exactly 65535 on rail input, and a saturating identity-channel input: each accumulator reaches its extremes."""
    t = _table(64, 330, 65535).astype(np.int64)
    for p in range(256):
        j = np.argmax(np.abs(t[p])); t[p, j] += np.sign(t[p, j]) * (65535 - np.abs(t[p]).sum())
    assert (np.abs(t).sum(1) == 65535).all() and np.abs(t).max() <= 32767
    t = t.astype(np.int16)
    x = np.where(np.random.default_rng(331).random((12000, 2)) < 0.5, -32768, 32767).astype(np.int16)
    x[5000:5300] = np.where(t[0][np.arange(300) % 64] < 0, -32768, 32767)[:, None]
    for step in (1 << 28, 1 << 32, STEP_44, 1 << 34):
        _same(eng, x, [(0, 0), (2 ** 30, 0), (2 ** 31, 0)], 0, step, t, A.n_inside(12000, 0, step))

def _long_case(eng, tiles, k, step, taps, seed):
    n_out = tiles * TM + 777; n = (n_out * step >> 32) + 100; x = _full_scale(n, seed); ch = GROUP_CH[:k]; stride = WD.ceil4(n_out)
    d_in = torch.from_numpy(x).cuda(); d_out = torch.zeros((k, stride, 2), dtype=torch.int16, device="cuda")
    eng.channelize_arbitrary_raw(d_in.data_ptr(), n, ch, 0, step, taps, d_out.data_ptr(), stride, n_out)
    for m0, m1 in ((0, 700), (n_out // 2 - 350, n_out // 2 + 350), (n_out - 700, n_out)):
        got = d_out[:, m0:m1].cpu().numpy(); want = A.channelize_arbitrary_window(x, ch, 0, step, taps, m0, m1)
        assert (got == want).all(), (step, m0, [(i, int((got[i] != want[i]).any(1).sum())) for i in range(k) if (got[i] != want[i]).any()])

@pytest.mark.parametrize("step", [STEP_44, 1 << 34])
def test_long_captures_and_channel_groups(eng, step):
    """4 x SMs tiles and more with 16 channels in every CTA, then a third of that: 16 channels in groups of several per CTA."""
    _long_case(eng, 4 * WD.sms() + 3, 16, step, TAPS_44, 340)
    _long_case(eng, 4 * WD.sms() // 3, 16, step, _table(33, 341), 341)


# ---- two independent kernels: the identity and sb200_channel_sim's interpolation ---------------------------------------------------
def test_identity_on_the_device(eng):
    x = _full_scale(7000, 350)
    for ntaps in (1, 8, 64):
        for d in (0, 3, 6999):
            y = eng.channelize_arbitrary(x, [(0, 0)], 1 << 32, _unit(ntaps), tau0=d << 32, n_out=7001)[0]
            assert (y[:7000 - d] == x[d:]).all() and (y[7000 - d:] == 0).all(), (ntaps, d)

def test_equals_the_channel_simulator(eng):
    """With sim_model's H and 8 taps this call is sb200_channel_sim with T = R = 1, one (16384, 0) tap, no carrier offset and no noise."""
    import sim_model
    x = _full_scale(30000, 360); H = sim_model.H.astype(np.int16); g = np.zeros((1, 1, 1, 2), np.int16); g[..., 0] = 16384
    for tau0, step in ((0, 1 << 32), (3 * 2 ** 32 + 12345, (1 << 32) + (1 << 24)), (2 ** 31, (1 << 32) - (1 << 24)), (77 << 30, api.clock_step(-40))):
        sim = eng.channel_sim(x[None, None], [(tau0, step, 0, 0, 0)], g, 29000)[0, 0]
        assert (eng.channelize_arbitrary(x, [(0, 0)], step, H, tau0=tau0, n_out=29000)[0] == sim).all(), (tau0, step)


# ---- the C ABI ----------------------------------------------------------------------------------------------------------------------
def test_residency_and_stream(eng):
    """iq and out each host, page-locked or device, rows wider than n_out (the bytes between and after them stay untouched), then a
    caller's stream, asynchronous on device buffers."""
    x = _full_scale(3001, 370); ch = _channels(3, 370); n_out = A.n_inside(3001, 0, STEP_44); stride = WD.ceil4(n_out + 9)
    want = A.channelize_arbitrary(x, ch, 0, STEP_44, TAPS_44, n_out)
    args = dict(iq=x, out=_fill(3 * stride * 4 + 16))
    ref = _matrix(lambda p: eng.channelize_arbitrary_raw(p["iq"], 3001, ch, 0, STEP_44, TAPS_44, p["out"], stride, n_out), args, _each(*args))
    rows = ref["out"][:3 * stride * 4].view(np.int16).reshape(3, stride, 2)
    assert (rows[:, :n_out] == want).all()
    assert (ref["out"][:3 * stride * 4].reshape(3, stride * 4)[:, n_out * 4:] == 0xA5).all() and (ref["out"][3 * stride * 4:] == 0xA5).all()
    pinned = torch.from_numpy(x).pin_memory(); out = np.zeros((3, stride, 2), np.int16)
    eng.channelize_arbitrary_raw(pinned.data_ptr(), 3001, ch, 0, STEP_44, TAPS_44, out.ctypes.data, stride, n_out)
    pinned.zero_()                                                                                  # the call has finished reading it
    assert (out[:, :n_out] == want).all()
    s = torch.cuda.Stream(); d_in = torch.from_numpy(x).cuda(); d_out = torch.zeros((3, stride, 2), dtype=torch.int16, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        for _ in range(3): eng.channelize_arbitrary_raw(d_in.data_ptr(), 3001, ch, 0, STEP_44, TAPS_44, d_out.data_ptr(), stride, n_out, stream=s.cuda_stream)
        d_out.zero_()                                                                               # queued behind the calls on the same stream
        eng.channelize_arbitrary_raw(d_in.data_ptr(), 3001, ch, 0, STEP_44, TAPS_44, d_out.data_ptr(), stride, n_out, stream=s.cuda_stream)
    s.synchronize()
    assert (d_out[:, :n_out].cpu().numpy() == want).all()

def test_one_launch_and_timing():
    e = api.Engine(0)
    try:
        x = _full_scale(50000, 380)
        for _ in range(2):
            n0 = e.launches; e.channelize_arbitrary(x, _channels(5, 380), STEP_44, TAPS_44)
            assert e.launches - n0 == 1 and e.last_kernel_ms() >= 0
    finally:
        e.close()

def _call(eng, iq, n, ch, nch, tau0, step, taps, ntaps, out, stride, n_out):
    return eng._lib.sb200_channelize_arbitrary(eng._h, V(iq), U64(n), V(ch), U32(nch), U64(tau0), U64(step), V(taps), U32(ntaps), V(out), U64(stride), U64(n_out), V(0))

def test_invalid_arguments_are_rejected(eng):
    x = _full_scale(1000, 390); out = np.zeros((17, 1000, 2), np.int16)
    ch = (api.DdcChannel * 17)(*[api.DdcChannel(i << 24, 0) for i in range(17)])
    t = np.ascontiguousarray(_table(64, 390)); xp, op, cp, tp = x.ctypes.data, out.ctypes.data, C.addressof(ch), t.ctypes.data
    S = STEP_44; n_out = A.n_inside(1000, 0, S)
    assert _call(eng, xp, 1000, cp, 4, 0, S, tp, 64, op, 360, n_out) == 0
    over = np.zeros((256, 8), np.int16); over[:, 3] = 16384; over[200, :4] = 16384                # row 200: 65536
    at = np.zeros((256, 8), np.int16); at[:, 3] = 16384; at[200, :4] = 16384; at[200, 0] = 16383     # row 200: 65535
    n_events = eng.launches
    edge = 2 ** 63 - (n_out - 1) * S                                                                # tau0 + (n_out - 1) step = 2^63
    bad = {"nchannels 0": (xp, 1000, cp, 0, 0, S, tp, 64, op, 360, n_out), "nchannels 17": (xp, 1000, cp, 17, 0, S, tp, 64, op, 360, n_out),
           "ntaps 0": (xp, 1000, cp, 4, 0, S, tp, 0, op, 360, n_out), "ntaps 65": (xp, 1000, cp, 4, 0, S, tp, 65, op, 360, n_out),
           "step < 2^28": (xp, 1000, cp, 4, 0, 2 ** 28 - 1, tp, 64, op, 360, n_out), "step > 2^34": (xp, 1000, cp, 4, 0, 2 ** 34 + 1, tp, 64, op, 360, n_out),
           "t reaches 2^63": (xp, 1000, cp, 4, edge, S, tp, 64, op, 360, n_out), "tau0 >= 2^63": (xp, 1000, cp, 4, 2 ** 63, S, tp, 64, op, 360, 1),
           "row sum": (xp, 1000, cp, 4, 0, S, over.ctypes.data, 8, op, 360, n_out), "stride < n_out": (xp, 1000, cp, 4, 0, S, tp, 64, op, 356, 358),
           "stride % 4": (xp, 1000, cp, 4, 0, S, tp, 64, op, 362, n_out), "stride > 2^40": (xp, 1000, cp, 4, 0, S, tp, 64, op, 2 ** 40 + 4, n_out),
           "n_in > 2^40": (xp, 2 ** 40 + 1, cp, 4, 0, S, tp, 64, op, 360, n_out), "null iq": (0, 1000, cp, 4, 0, S, tp, 64, op, 360, n_out),
           "null channels": (xp, 1000, 0, 4, 0, S, tp, 64, op, 360, n_out), "null taps": (xp, 1000, cp, 4, 0, S, 0, 64, op, 360, n_out),
           "null out": (xp, 1000, cp, 4, 0, S, tp, 64, 0, 360, n_out)}
    for name, a in bad.items():
        assert _call(eng, *a) == -1, name
    d = torch.zeros(2 * 1000 * 2 + 8, dtype=torch.int16, device="cuda")
    assert _call(eng, d.data_ptr() + 4, 999, cp, 1, 0, S, tp, 64, op, 360, n_out) == -1, "misaligned device input"
    assert _call(eng, xp, 1000, cp, 1, 0, S, tp, 64, d.data_ptr() + 4, 360, n_out) == -1, "misaligned device output"
    assert _call(eng, xp, 1000, cp, 4, 0, S, tp, 64, op, 360, 0) == 0, "n_out = 0"
    assert eng.launches == n_events, "a refused call (or n_out = 0) launched"
    assert _call(eng, xp, 1000, cp, 4, edge - 1, S, tp, 64, op, 360, n_out) == 0                  # 2^63 - 1 is accepted
    assert _call(eng, xp, 1000, cp, 4, 0, S, at.ctypes.data, 8, op, 360, n_out) == 0               # a row sum of 65535 is accepted


# ---- end to end, device-resident ----------------------------------------------------------------------------------------------------
def test_24ghz_at_122_88_on_the_device():
    """The 122.88 Msps capture on the device -> this call (802.11b rows at 44 Msps, the OFDM row at 40 Msps) -> sb200_rx11b_streams and
    sb200_rx11a_streams, against the oracle on the model's rows: every field, event position and delivered byte; every PSDU delivered."""
    iq, rows, ps = rows_24ghz()
    e = api.Engine(0); ea = api.Engine(0, cca_pwr_threshold=CCA_WIDE)
    try:
        d_in = torch.from_numpy(np.ascontiguousarray(iq)).cuda(); n = len(iq)
        b_ch = [c for c, k in enumerate(A.R.KIND_24) if k == "11b"]; a_ch = [c for c, k in enumerate(A.R.KIND_24) if k == "ofdm"]
        def dev_rows(chans, step, t):
            n_out = A.n_inside(n, 0, step); out = WD.dev_rows(len(chans), n_out, 64); stride = out.shape[1]
            e.channelize_arbitrary_raw(d_in.data_ptr(), n, [(W.phase_inc(A.R.CH_24[c], FS), 0) for c in chans], 0, step, t, out.data_ptr(), stride, n_out)
            return out, stride, n_out
        db_, sb, nb = dev_rows(b_ch, STEP_44, TAPS_44); da_, sa, na = dev_rows(a_ch, STEP_40, TAPS_40)
        for i, c in enumerate(b_ch): assert (db_[i, :nb].cpu().numpy() == rows[c]).all(), c
        for i, c in enumerate(a_ch): assert (da_[i, :na].cpu().numpy() == rows[c]).all(), c
        got_b = WD.rx11b(e, db_, sb, nb, len(b_ch)); got_a = WD.rx11a(ea, da_, sa, na, len(a_ch))
    finally:
        e.close(); ea.close()
    for i, (c, (o, _)) in enumerate(zip(b_ch, WD.equal_11b([rows[c] for c in b_ch], got_b))):
        assert len(o) == len(ps[c]), (c, len(o))
        for j in range(len(o)):
            L = int(o["length"][j]) - 1; assert bytes(got_b[1][i, j, :L]) == bytes(ps[c][j][:-1]), (c, j)
    for i, (c, (o, _)) in enumerate(zip(a_ch, WD.equal_11a([rows[c] for c in a_ch], got_a))):
        assert len(o) == len(ps[c]), (c, len(o))
        for j in range(len(o)):
            L = int(o["length"][j]); assert bytes(got_a[1][i, j, :L]) == bytes(ps[c][j]), (c, j)

@pytest.mark.parametrize("kind,rates", [("11a", (6000, 24000, 54000)), ("11b", (1000, 2000, 5500, 11000))])
def test_round_trip_through_122_88(kind, rates):
    """The device transmitter's frame at its own rate (802.11a at 40 Msps, 802.11b at 44 Msps), up to 122.88 Msps with this call (step below
    2^32) and back down with it: the device receiver decodes it to FRAME_OK with the exact bytes at every rate."""
    e = api.Engine(0, cca_pwr_threshold=CCA_WIDE if kind == "11a" else 0); fs_tx = 40e6 if kind == "11a" else 44e6
    up, down = api.arbitrary_step(fs_tx, FS), api.arbitrary_step(FS, fs_tx)
    t_up = api.arbitrary_taps(fs_tx, FS, 64, 9e6 if kind == "11b" else 8.3e6); t_down = TAPS_40 if kind == "11a" else TAPS_44
    try:
        for j, rate in enumerate(rates):
            mpdu = W._psdu(120 + 40 * j, 0x3DA0 + j)
            if kind == "11a": w = WD.tx11a(e, mpdu, rate, 7 + j).to(torch.int16) * 20           # the levels of test_gpu_combine_rational.py
            else: w = WD.tx11b(e, mpdu, rate).to(torch.int16) << 6
            sig = torch.zeros((len(w) + 800, 2), dtype=torch.int16, device="cuda"); sig[400:400 + len(w)] = w
            n_up = A.n_inside(len(sig), 0, up); hi = WD.dev_rows(1, n_up)
            e.channelize_arbitrary_raw(sig.data_ptr(), len(sig), [(0, 0)], 0, up, t_up, hi.data_ptr(), hi.shape[1], n_up)
            n_dn = A.n_inside(n_up, 0, down); lo = WD.dev_rows(1, n_dn, 64)
            e.channelize_arbitrary_raw(hi.data_ptr(), n_up, [(0, 0)], 0, down, t_down, lo.data_ptr(), lo.shape[1], n_dn)
            res, out, _, cnt = (WD.rx11a if kind == "11a" else WD.rx11b)(e, lo, lo.shape[1], n_dn, 1)
            L = len(mpdu) - (kind == "11b")
            assert cnt[0] == 1 and res[0, 0]["status"] == api.FRAME_OK and bytes(out[0, 0, :L]) == bytes(mpdu[:L]), (kind, rate, cnt[0], res[0, :cnt[0]])
    finally:
        e.close()
