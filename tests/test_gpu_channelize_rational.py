"""GPU tests of the rational-rate channelizer (sb200_channelize_rational, pytest -m gpu): bit for bit against the numpy model of
tests/rational_model.py over lengths, every coprime (U, D), channel counts, branch lengths, increments and full-scale input; the pointer
residency, launch bookkeeping and argument checks of the C ABI; and the 2.4 GHz captures of test_cpu_channelize_rational.py channelized
and decoded on the device, all device-resident, against the CPU oracle decoding the numpy-channelized rows."""
import ctypes as C
from math import gcd
import numpy as np, pytest
import torch
import wideband_inputs as W
import wideband_device as WD
import rational_model as R
from sora_b200 import api
from test_gpu_abi_residency import _matrix, _each, _fill
from test_cpu_channelize import CCA_WIDE, _full_scale
from test_cpu_channelize_rational import PLANS, TAPS_160_44, rows_24ghz
from wideband_device import GROUP_CH, DDC_INCS as INCS, ddc_channels as _channels, ddc_taps as _taps, sms as _sms

pytestmark = pytest.mark.gpu
V, U32, U64 = C.c_void_p, C.c_uint32, C.c_uint64
TILE = 4096
COPRIME = [(u, d) for u in range(1, 17) for d in range(u, 65) if gcd(u, d) == 1]

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

def _btaps(U, per_branch, seed, total=40000):
    """U * per_branch - (1 - U % 2) taps (odd), every branch's sum |t| about `total`."""
    n = U * per_branch; n -= 1 - n % 2
    rng = np.random.default_rng(seed); t = rng.integers(-1000, 1000, n).astype(np.float64); t[n // 2] = 5000.0
    for r in range(U):
        s = np.abs(t[r::U]).sum()
        if s: t[r::U] = np.trunc(t[r::U] * total / s)
    return t.astype(np.int16)

def _rational(eng, x, ch, u, d, taps):
    """sb200_channelize_rational itself, also at interp = 1 (where Engine.channelize calls sb200_channelize): host in, host out."""
    x = np.ascontiguousarray(x, np.int16); t = np.ascontiguousarray(taps, np.int16); cha = (api.DdcChannel * len(ch))(*[api.DdcChannel(a, b) for a, b in ch])
    n_out = -(-u * len(x) // d); stride = (n_out + 3) // 4 * 4; out = np.zeros((len(ch), stride, 2), np.int16)
    eng._check(eng._lib.sb200_channelize_rational(eng._h, V(x.ctypes.data), U64(len(x)), V(C.addressof(cha)), U32(len(ch)), U32(u), U32(d), V(t.ctypes.data),
                                                  U32(len(t)), V(out.ctypes.data), U64(stride), V(0)), "sb200_channelize_rational")
    return out[:, :n_out]

def _same(eng, x, ch, u, d, taps):
    got = eng.channelize(x, ch, d, taps, interp=u) if u > 1 else _rational(eng, x, ch, u, d, taps); want = R.channelize_rational(x, ch, u, d, taps)
    assert got.shape == want.shape and (got == want).all(), (u, d, [(i, np.argwhere((got[i] != want[i]).any(1))[:3].ravel()) for i in range(len(ch)) if (got[i] != want[i]).any()])

@pytest.mark.parametrize("n", [1, 2, 39, TILE - 1, TILE, TILE + 1, 3 * TILE + 2, 10001])
def test_lengths(eng, n):
    """n_in of 1, around one tile and lengths where U n_in / D is not whole; random full-scale input with rails."""
    x = _full_scale(n, 110 + n)
    _same(eng, x, _channels(4, n), 11, 40, TAPS_160_44)
    _same(eng, x, [(0, 0), (2 ** 31, 1 << 20)], 5, 22, _btaps(5, 255, n))
    _same(eng, x, _channels(3, n + 1), 3, 64, _btaps(3, 31, n + 1))

def test_every_coprime_ratio_short(eng):
    """Every coprime (U, D) with U <= 16 and D <= 64 on a short capture, two channels."""
    x = _full_scale(1500, 120)
    for i, (u, d) in enumerate(COPRIME):
        _same(eng, x, _channels(2, i), u, d, _btaps(u, [1, 3, 17, 64, 255][i % 5], i))

@pytest.mark.parametrize("u", range(2, 17))
def test_ratios_channels_and_branches(eng, u):
    """U = 2 .. 16 on several tiles with K = 1 .. 16 channels, D spread over u + 1 .. 64, 1 .. 255 taps per branch."""
    for j, d in enumerate(dd for dd in range(u + 1, 65) if gcd(u, dd) == 1 and (dd + u) % 5 == 0):
        x = _full_scale(3 * TILE + 37 * d, 130 + d)
        _same(eng, x, _channels(1 + (u + j) % 16, u + j), u, d, _btaps(u, [1, 2, 9, 127, 255][(u + j) % 5], u * 100 + d))

def test_increments_and_phases(eng):
    """Every increment of INCS (0, quarter and half turns, wrapped negatives, arbitrary) with zero and arbitrary phase0, 16 channels."""
    x = _full_scale(20000, 140)
    _same(eng, x, [(inc, ph) for inc in INCS for ph in (0, 0xDEADBEEF)], 11, 40, TAPS_160_44)

@pytest.mark.parametrize("u,d", [(11, 40), (5, 22), (16, 17), (2, 3)])
def test_every_branch_at_the_limit(eng, u, d):
    """Every branch's sum |t| exactly 65535, on rail input: each accumulator reaches its extremes without wrapping."""
    t = _btaps(u, 63, 150 + u, 65535).astype(np.int64)
    for r in range(u):
        b = t[r::u]; b[np.argmax(np.abs(b))] += np.sign(b[np.argmax(np.abs(b))]) * (65535 - np.abs(b).sum()); t[r::u] = b
    assert all(np.abs(t[r::u]).sum() == 65535 for r in range(u)) and np.abs(t).max() <= 32767
    t = t.astype(np.int16)
    x = np.where(np.random.default_rng(151).random((12000, 2)) < 0.5, -32768, 32767).astype(np.int16)
    x[5000:5200] = np.where(t[(np.arange(200) * u) % len(t)] < 0, 32767, -32768)[:, None]
    _same(eng, x, [(0, 0), (2 ** 30, 0), (2 ** 31, 0)], u, d, t)

@pytest.mark.parametrize("d", range(1, 65))
def test_interp_1_is_the_channelizer(eng, d):
    """interp = 1 is sb200_channelize bit for bit (D <= 16), and the model beyond it."""
    x = _full_scale(9000 + 37 * d, 160 + d); ch = _channels(1 + d % 16, d); t = _taps([1, 31, 127, 255][d % 4], d)
    want = R.channelize_rational(x, ch, 1, d, t)
    assert (_rational(eng, x, ch, 1, d, t) == want).all()
    if d <= 16: assert (eng.channelize(x, ch, d, t) == want).all()


# ---- long captures: several channels per CTA, checked by window ---------------------------------------------------------------------
def _long_case(eng, tiles, k, u, d, taps, seed):
    n = tiles * TILE + 777; x = _full_scale(n, seed); ch = GROUP_CH[:k]
    n_out = -(-u * n // d); stride = (n_out + 3) // 4 * 4
    d_in = torch.from_numpy(x).cuda(); d_out = torch.zeros((k, stride, 2), dtype=torch.int16, device="cuda")
    eng.channelize_raw(d_in.data_ptr(), n, ch, d, taps, d_out.data_ptr(), stride, interp=u)
    mid = (tiles // 2) * TILE * u // d
    for m0, m1 in ((0, 700), (mid - 350, mid + 350), (n_out - 700, n_out)):
        got = d_out[:, m0:m1].cpu().numpy(); want = R.channelize_rational_window(x, ch, u, d, taps, m0, m1)
        assert (got == want).all(), (u, d, m0, [(i, int((got[i] != want[i]).any(1).sum())) for i in range(k) if (got[i] != want[i]).any()])

@pytest.mark.parametrize("u,d", [(11, 40), (5, 22), (11, 50), (2, 3), (16, 63), (7, 8)])
def test_all_channels_in_one_cta(eng, u, d):
    """Captures of 4 x SMs tiles and more, 4 .. 16 channels in every CTA, 253 .. 255 taps per branch (the largest halo)."""
    _long_case(eng, 4 * _sms() + 3, [4, 7, 11, 16][u % 4], u, d, _btaps(u, 255, 170 + u), 170 + d)

@pytest.mark.parametrize("u,d", [(11, 40), (3, 4)])
def test_channel_groups(eng, u, d):
    """A capture of a third of 4 x SMs tiles: 16 channels in groups of several per CTA."""
    _long_case(eng, 4 * _sms() // 3, 16, u, d, _btaps(u, 200, 180 + u), 180 + d)


# ---- the C ABI ----------------------------------------------------------------------------------------------------------------------
def test_residency_and_stream(eng):
    """iq and out each host or device, rows wider than n_out (the bytes between and after them stay untouched), then a caller's stream."""
    x = _full_scale(1001, 190); ch = _channels(3, 190); n_out = -(-11 * 1001 // 40); stride = n_out + 9 + (-(n_out + 9)) % 4
    want = R.channelize_rational(x, ch, 11, 40, TAPS_160_44)
    args = dict(iq=x, out=_fill(3 * stride * 4 + 16))
    ref = _matrix(lambda p: eng.channelize_raw(p["iq"], 1001, ch, 40, TAPS_160_44, p["out"], stride, interp=11), args, _each(*args))
    rows = ref["out"][:3 * stride * 4].view(np.int16).reshape(3, stride, 2)
    assert (rows[:, :n_out] == want).all()
    assert (ref["out"][:3 * stride * 4].reshape(3, stride * 4)[:, n_out * 4:] == 0xA5).all() and (ref["out"][3 * stride * 4:] == 0xA5).all()
    s = torch.cuda.Stream(); d_in = torch.from_numpy(x).cuda(); d_out = torch.zeros((3, stride, 2), dtype=torch.int16, device="cuda")
    torch.cuda.synchronize()
    eng.channelize_raw(d_in.data_ptr(), 1001, ch, 40, TAPS_160_44, d_out.data_ptr(), stride, stream=s.cuda_stream, interp=11)
    s.synchronize()
    assert (d_out[:, :n_out].cpu().numpy() == want).all()

def test_one_launch_and_timing():
    e = api.Engine(0)
    try:
        x = _full_scale(50000, 200)
        for _ in range(2):
            n0 = e.launches; e.channelize(x, _channels(5, 200), 40, TAPS_160_44, interp=11)
            assert e.launches - n0 == 1 and e.last_kernel_ms() >= 0
    finally:
        e.close()

def _call(eng, iq, n, ch, nch, u, d, taps, ntaps, out, stride):
    return eng._lib.sb200_channelize_rational(eng._h, V(iq), U64(n), V(ch), U32(nch), U32(u), U32(d), V(taps), U32(ntaps), V(out), U64(stride), V(0))

def test_invalid_arguments_are_rejected(eng):
    x = _full_scale(1000, 210); out = np.zeros((17, 1000, 2), np.int16)
    ch = (api.DdcChannel * 17)(*[api.DdcChannel(i << 24, 0) for i in range(17)])
    t = np.array(TAPS_160_44); xp, op, cp, tp = x.ctypes.data, out.ctypes.data, C.addressof(ch), t.ctypes.data
    assert _call(eng, xp, 1000, cp, 4, 11, 40, tp, 1287, op, 276) == 0                           # n_out = ceil(11000 / 40) = 275
    over = np.zeros(67, np.int16); over[0::11] = 9363                                          # branch 0: 7 x 9363 = 65541, the others 0
    at = np.zeros(67, np.int16); at[0::11] = 9362; at[33] += 1                                   # branch 0: 65535
    long_ = np.zeros(11 * 255 + 2, np.int16); long_[11 * 127] = 16384                          # odd, 256 taps in branch 0
    n_events = eng.launches
    bad = {"nchannels 0": (xp, 1000, cp, 0, 11, 40, tp, 1287, op, 276), "nchannels 17": (xp, 1000, cp, 17, 11, 40, tp, 1287, op, 276),
           "interp 0": (xp, 1000, cp, 4, 0, 40, tp, 1287, op, 276), "interp 17": (xp, 1000, cp, 4, 17, 40, tp, 1287, op, 276),
           "decim < interp": (xp, 1000, cp, 4, 11, 10, tp, 1287, op, 1100), "decim 65": (xp, 1000, cp, 4, 11, 65, tp, 1287, op, 276),
           "not coprime": (xp, 1000, cp, 4, 10, 40, tp, 1287, op, 276), "interp = decim": (xp, 1000, cp, 4, 11, 11, tp, 1287, op, 1000),
           "ntaps even": (xp, 1000, cp, 4, 11, 40, tp, 1286, op, 276), "branch of 256": (xp, 1000, cp, 4, 11, 40, long_.ctypes.data, len(long_), op, 276),
           "branch sum": (xp, 1000, cp, 4, 11, 40, over.ctypes.data, len(over), op, 276), "stride < n_out": (xp, 1000, cp, 4, 11, 40, tp, 1287, op, 272),
           "stride % 4": (xp, 1000, cp, 4, 11, 40, tp, 1287, op, 277), "null iq": (0, 1000, cp, 4, 11, 40, tp, 1287, op, 276),
           "null channels": (xp, 1000, 0, 4, 11, 40, tp, 1287, op, 276), "null taps": (xp, 1000, cp, 4, 11, 40, 0, 1287, op, 276),
           "null out": (xp, 1000, cp, 4, 11, 40, tp, 1287, 0, 276), "n_in > 2^40": (xp, 2 ** 40 + 1, cp, 4, 11, 40, tp, 1287, op, 2 ** 40),
           "stride > 2^40": (xp, 1000, cp, 4, 11, 40, tp, 1287, op, 2 ** 40 + 4)}
    for name, a in bad.items():
        assert _call(eng, *a) == -1, name
    d = torch.zeros(2 * 1000 * 2 + 8, dtype=torch.int16, device="cuda")
    assert _call(eng, d.data_ptr() + 4, 999, cp, 1, 11, 40, tp, 1287, op, 276) == -1, "misaligned device input"
    assert _call(eng, xp, 1000, cp, 1, 11, 40, tp, 1287, d.data_ptr() + 4, 276) == -1, "misaligned device output"
    assert eng.launches == n_events, "a refused call launched"
    assert abs(at[0::11].astype(np.int64)).sum() == 65535
    assert _call(eng, xp, 1000, cp, 4, 11, 40, at.ctypes.data, len(at), op, 276) == 0          # a branch sum of 65535 is accepted


# ---- end to end, device-resident ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fs", [160e6, 176e6])
def test_24ghz_on_the_device(fs):
    """capture_24ghz on the device -> device channelizer (802.11b rows at 44 Msps, the OFDM row at 40 Msps) -> sb200_rx11b_streams and
    sb200_rx11a_streams, against the oracle on the model's rows: every field, event position and delivered byte; every PSDU delivered."""
    iq, rows, ps = rows_24ghz(fs); (ub, db), tb, (ua, da), ta = PLANS[fs]
    e = api.Engine(0); ea = api.Engine(0, cca_pwr_threshold=CCA_WIDE)           # the OFDM receiver with the wideband carrier-sense threshold
    try:
        d_in = torch.from_numpy(np.ascontiguousarray(iq)).cuda(); n = len(iq)
        b_ch = [c for c, k in enumerate(R.KIND_24) if k == "11b"]; a_ch = [c for c, k in enumerate(R.KIND_24) if k == "ofdm"]
        def dev_rows(chans, u, d, t):
            n_out = -(-u * n // d); out = WD.dev_rows(len(chans), n_out, 64); stride = out.shape[1]
            e.channelize_raw(d_in.data_ptr(), n, [(W.phase_inc(R.CH_24[c], fs), 0) for c in chans], d, t, out.data_ptr(), stride, interp=u)
            return out, stride, n_out
        db_, sb, nb = dev_rows(b_ch, ub, db, tb); da_, sa, na = dev_rows(a_ch, ua, da, ta)
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
