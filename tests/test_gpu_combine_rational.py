"""GPU tests of the rational-rate combiner (sb200_combine_rational, pytest -m gpu): bit for bit against the numpy model of
tests/combine_rational_model.py over lengths around the tile, output counts, every coprime (U, D), channel counts, branch lengths, gains,
increments, accumulate and full-scale input; decim = 1 against sb200_combine on the device; the pointer residency, stream, launch bookkeeping
and argument checks of the C ABI; and the 2.4 GHz transmit chain of test_cpu_combine_rational.py on the device (transmitters -> two combiner
calls into one buffer -> channel simulator with noise -> rational channelizers -> stream receivers, all device-resident) against the model
and the CPU oracle."""
import ctypes as C
from math import gcd
import numpy as np, pytest
import torch
import wideband_inputs as W
import wideband_device as WD
import combine_rational_model as CR
import rational_model as R
from sora_b200 import api
from test_gpu_abi_residency import _matrix, _each, _fill
from test_cpu_channelize import CCA_WIDE
from test_cpu_channelize_rational import PLANS
from test_cpu_combine_rational import TX_PLANS, GAIN_A, GAIN_B, TAPS_44_160, TAPS_40_176, SIM_LINK_24, SIM_TAPS_24, SIM_SEED_24, frames_24ghz, capture_of, through_the_air
from test_cpu_combine import _psdus
from wideband_device import GAINS, DUC_INCS as INCS, duc_channels as _channels, duc_rows as _rows, duc_taps as _taps, sms as _sms

pytestmark = pytest.mark.gpu
V, U32, U64 = C.c_void_p, C.c_uint32, C.c_uint64

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

def _tq(K, U, D, ntaps):
    """Outputs per phase of a tile that sb200_combine_rational picks: the largest of 1024 .. 64 whose shared memory fits 57344 bytes, else 32."""
    halo = ((ntaps // 2 + U - 1) // U + 3) // 4 * 4
    for tq in (1024, 512, 256, 128, 64):
        if (K * (D * tq + 2 * halo) + U * tq + 4096) * 4 + 16 <= 57344: return tq
    return 32

def _btaps(U, per_branch, seed, total=50000):
    """U per_branch taps, one fewer when that is even (so at most per_branch per branch): test_gpu_combine's random Q15 taps."""
    n = U * per_branch; n -= 1 - n % 2
    return _taps(max(n, 1), U, seed, total)

def _same(eng, rows, ch, u, d, taps, n_out=None, acc=None):
    n = -(-u * rows.shape[1] // d) if n_out is None else n_out
    out = None if acc is None else np.array(acc, np.int16)
    got = eng.combine(rows, ch, u, taps, decim=d, n_out=n, accumulate=acc is not None, out=out)
    want = CR.combine_rational(rows, ch, u, d, taps, n, acc)
    assert got.shape == want.shape and (got == want).all(), (u, d, np.argwhere((got != want).any(1))[:5].ravel())

COPRIME = [(u, d) for d in range(1, 17) for u in range(d, 65) if gcd(u, d) == 1]

@pytest.mark.parametrize("U,D,K,ntaps", [(40, 11, 3, 1761), (22, 5, 1, 1321), (4, 1, 16, 127), (17, 16, 16, 255), (64, 1, 2, 4095)])
def test_lengths(eng, U, D, K, ntaps):
    """n_in of 1 .. 5 and around the tile the call picks (U n_in / D mostly not whole), and several tiles + 777."""
    tq = _tq(K, U, D, ntaps); taps = _btaps(U, -(-ntaps // U), U) if ntaps < 4095 else _btaps(U, 64, U)
    for n in (1, 2, 3, 5, D * tq - 1, D * tq, D * tq + 1, 3 * D * tq + 777):                    # a tile reads D tq inputs per row
        _same(eng, _rows(K, max(n, 1), n), _channels(K, n), U, D, taps)

@pytest.mark.parametrize("U,D", [(40, 11), (22, 5), (7, 3)])
def test_n_out(eng, U, D):
    """n_out shorter than, equal to and longer than ceil(U n_in / D), and 0 (nothing launched)."""
    rows = _rows(2, 1001, 3); ch = _channels(2, 3); taps = _btaps(U, 31, 3); n = -(-U * 1001 // D)
    for m in (1, 4, n - 555, n - 1, n, n + 1, n + 3 * U, n + 5000):
        _same(eng, rows, ch, U, D, taps, m)
    x = np.zeros((2, 1004, 2), np.int16); x[:, :1001] = rows; out = np.full((4, 2), 7, np.int16)
    l0 = eng.launches; eng.combine_raw(api._ptr(x), 1004, 1001, ch, U, taps, api._ptr(out), decim=D, n_out=0)
    assert eng.launches == l0 and (out == 7).all()

def test_every_coprime_ratio_short(eng):
    """Every coprime (U, D) with 1 <= D <= 16 and D <= U <= 64, on 97 input samples of 3 channels."""
    for u, d in COPRIME:
        _same(eng, _rows(3, 97, u + 64 * d), _channels(3, u), u, d, _btaps(u, 1 + (u * d) % 23, u + d))

@pytest.mark.parametrize("U,D", [(40, 11), (22, 5), (4, 1), (64, 1), (17, 16), (16, 15)])
def test_dense_ratios_over_several_tiles(eng, U, D):
    K = 5; taps = _btaps(U, 41, U + D); tq = _tq(K, U, D, len(taps))
    _same(eng, _rows(K, 5 * D * tq + 333, U), _channels(K, U + 1), U, D, taps)

@pytest.mark.parametrize("K", [1, 2, 5, 8, 16])
def test_channels_and_branch_lengths(eng, K):
    """K = 1 .. 16 channels, 1 to 255 taps per branch, and ntaps = 4095."""
    for U, D, per in ((40, 11, 1), (22, 5, 255), (16, 3, 256 - 1), (64, 15, 64), (5, 2, 100)):
        taps = _btaps(U, per, K) if U * per <= 4095 else _btaps(U, 4095 // U, K)
        _same(eng, _rows(K, 600, K + U), _channels(K, K + U), U, D, taps)

def test_rails_at_every_limit(eng):
    """Every branch of the taps sums to exactly 65535 on rail input, and 16 channels at gain 65535 in phase: the accumulator reaches its
    extremes without wrapping and the final sat16 clips."""
    U, D = 40, 11; t = np.zeros(40 * 9 + 1, np.int64)
    for r in range(U):
        idx = np.arange(r, len(t), U); t[idx] = 65535 // len(idx); t[idx[0]] += 65535 - t[idx].sum()
    t = t.astype(np.int16); assert all(np.abs(t[r::U].astype(np.int64)).sum() == 65535 for r in range(U))
    x = np.where(np.random.default_rng(41).random((800, 2)) < 0.5, -32768, 32767).astype(np.int16); x[300:340] = -32768
    rows = np.stack([x] * 16); ch = [(2 ** 30, 0, 65535)] * 16
    got = eng.combine(rows, ch, U, t, decim=D)
    assert (got == CR.combine_rational(rows, ch, U, D, t)).all() and (np.abs(got.astype(np.int64)) >= 32767).mean() > 0.5

def test_gains_and_increments(eng):
    """Every increment of INCS (quarter and half turns, wrapped negative ones) with zero and arbitrary phase0, 16 channels, gains 0 .. 65535."""
    ch = [(inc, ph, GAINS[i % 8]) for i, (inc, ph) in enumerate((inc, ph) for inc in INCS for ph in (0, 0xDEADBEEF))]
    _same(eng, _rows(16, 1500, 30), ch, 22, 5, TAPS_40_176)

def test_accumulate(eng):
    """accumulate onto random and rail contents, host and device output."""
    rows = _rows(3, 2000, 31); ch = _channels(3, 31); U, D = 40, 11; n = -(-U * 2000 // D) + 17
    rng = np.random.default_rng(5)
    for acc in (rng.integers(-32768, 32768, (n, 2)), np.where(rng.random((n, 2)) < 0.5, -32768, 32767)):
        _same(eng, rows, ch, U, D, TAPS_44_160, n, acc.astype(np.int16))
        d_in = torch.from_numpy(np.ascontiguousarray(rows)).cuda(); d_out = torch.from_numpy(acc.astype(np.int16)).cuda()
        eng.combine_raw(d_in.data_ptr(), 2000, 2000, ch, U, TAPS_44_160, d_out.data_ptr(), decim=D, n_out=n, accumulate=True)
        assert (d_out.cpu().numpy() == CR.combine_rational(rows, ch, U, D, TAPS_44_160, n, acc.astype(np.int16))).all()

def test_shared_memory_corners(eng):
    """The tiles at the shared-memory corners: K = 16 at D = 16 (the smallest tile) and U = 64 with long branches."""
    _same(eng, _rows(16, 3000, 80), _channels(16, 80), 17, 16, _btaps(17, 240, 80))
    _same(eng, _rows(16, 900, 81), _channels(16, 81), 63, 16, _btaps(63, 65, 81))
    _same(eng, _rows(4, 700, 82), _channels(4, 82), 64, 1, _btaps(64, 63, 82))


# ---- long captures --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,U,D,ntaps", [(3, 40, 11, 1761), (1, 22, 5, 1321), (16, 17, 16, 255), (2, 64, 1, 4095)])
def test_long_captures(eng, K, U, D, ntaps):
    """At least 4 x SMs tiles plus 777 samples, on the device; the first, middle and last outputs against combine_rational_window."""
    taps = TAPS_44_160 if ntaps == 1761 else TAPS_40_176 if ntaps == 1321 else _btaps(U, -(-ntaps // U), 90 + U)
    n = (4 * _sms() + 3) * _tq(K, U, D, len(taps)) * D + 777; stride = (n + 3) // 4 * 4; n_out = -(-U * n // D)
    rows = np.zeros((K, stride, 2), np.int16); rows[:, :n] = _rows(K, n, 70 + U); ch = _channels(K, 70 + U)
    d_in = torch.from_numpy(rows).cuda(); d_out = torch.zeros((n_out, 2), dtype=torch.int16, device="cuda")
    eng.combine_raw(d_in.data_ptr(), stride, n, ch, U, taps, d_out.data_ptr(), decim=D, n_out=n_out)
    for n0, n1 in ((0, 700), (n_out // 2 - 350, n_out // 2 + 350), (n_out - 700, n_out)):
        got = d_out[n0:n1].cpu().numpy(); want = CR.combine_rational_window(rows[:, :n], ch, U, D, taps, n0, n1)
        assert (got == want).all(), (n0, np.argwhere((got != want).any(1))[:5].ravel())


# ---- the C ABI ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("u", range(1, 17))
def test_decim_1_is_the_combiner(eng, u):
    """sb200_combine_rational with D = 1 and n_out = U n_in equals sb200_combine, device against device."""
    K = 17 - u; n = 3001; ntaps = [1, 3, 17, 31, 63, 101, 127, 255][u % 8]
    rows = torch.from_numpy(_rows(K, n + 3, u)).cuda(); ch = _channels(K, u); taps = _taps(ntaps, u, u)
    a = torch.zeros((u * n, 2), dtype=torch.int16, device="cuda"); b = torch.zeros_like(a)
    eng.combine_raw(rows.data_ptr(), n + 3, n, ch, u, taps, a.data_ptr())
    eng.combine_raw(rows.data_ptr(), n + 3, n, ch, u, taps, b.data_ptr(), decim=1, n_out=u * n)
    assert (a.cpu() == b.cpu()).all()

def test_residency(eng):
    """rows and out each host or device, with and without accumulate (a host out is uploaded first); the bytes after out untouched."""
    K, n, stride, U, D = 3, 1001, 1008, 40, 11; n_out = -(-U * n // D)
    rows = np.full((K, stride, 2), 0x5A5A, np.int16); rows[:, :n] = _rows(K, n, 50); ch = _channels(K, 50)
    args = dict(rows=rows, out=_fill(n_out * 4 + 16))
    ref = _matrix(lambda p: eng.combine_raw(p["rows"], stride, n, ch, U, TAPS_44_160, p["out"], decim=D, n_out=n_out), args, _each(*args))
    assert (ref["out"][:n_out * 4].view(np.int16).reshape(-1, 2) == CR.combine_rational(rows[:, :n], ch, U, D, TAPS_44_160)).all()
    assert (ref["out"][n_out * 4:] == 0xA5).all()
    acc = ref["out"].copy(); args = dict(rows=rows, out=acc)
    ref2 = _matrix(lambda p: eng.combine_raw(p["rows"], stride, n, ch, U, TAPS_44_160, p["out"], decim=D, n_out=n_out, accumulate=True), args, _each(*args))
    want = CR.combine_rational(rows[:, :n], ch, U, D, TAPS_44_160, n_out, acc[:n_out * 4].view(np.int16).reshape(-1, 2))
    assert (ref2["out"][:n_out * 4].view(np.int16).reshape(-1, 2) == want).all() and (ref2["out"][n_out * 4:] == 0xA5).all()

def test_a_callers_stream(eng):
    K, n, U, D = 3, 30001, 40, 11; rows = _rows(K, n + 3, 51); ch = _channels(K, 51); n_out = -(-U * n // D)
    d_in = torch.from_numpy(np.ascontiguousarray(rows)).cuda(); s = torch.cuda.Stream(); s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        d_out = torch.zeros((n_out, 2), dtype=torch.int16, device="cuda")
        eng.combine_raw(d_in.data_ptr(), n + 3, n, ch, U, TAPS_44_160, d_out.data_ptr(), s.cuda_stream, decim=D)
        got = d_out.cpu().numpy()
    assert (got == CR.combine_rational(rows[:, :n], ch, U, D, TAPS_44_160)).all()

def test_one_launch_and_timing():
    e = api.Engine(0)
    try:
        rows = _rows(3, 50000, 60)
        for acc in (False, True):
            n0 = e.launches; e.combine(rows, _channels(3, 60), 40, TAPS_44_160, decim=11, accumulate=acc)
            assert e.launches - n0 == 1 and e.last_kernel_ms() > 0
    finally:
        e.close()

def _call(eng, rows, stride, n, ch, nch, u, d, taps, ntaps, out, n_out, acc=0):
    return eng._lib.sb200_combine_rational(eng._h, V(rows), U64(stride), U64(n), V(ch), U32(nch), U32(u), U32(d), V(taps), U32(ntaps), V(out), U64(n_out), U32(acc), V(0))

def test_invalid_arguments_are_rejected(eng):
    x = _rows(17, 1000, 70); out = np.zeros((4 * 1000, 2), np.int16)
    ch = (api.DucChannel * 17)(*[api.DucChannel(i << 24, 0, 4096) for i in range(17)])
    hot = (api.DucChannel * 2)(api.DucChannel(0, 0, 4096), api.DucChannel(0, 0, 65536))
    t = np.array(TAPS_44_160); xp, op, cp, tp = x.ctypes.data, out.ctypes.data, C.addressof(ch), t.ctypes.data; nt = len(t)
    assert _call(eng, xp, 1000, 1000, cp, 4, 40, 11, tp, nt, op, 3637) == 0
    over = np.zeros(41 * 40 + 1, np.int16); over[0:40 * 7:40] = 9363                  # branch 0: 7 x 9363 = 65541
    at = np.zeros(41 * 40 + 1, np.int16); at[0:40 * 7:40] = 9362; at[40 * 7] = 1                    # branch 0: 65535
    assert abs(at[0::40].astype(np.int64)).sum() == 65535 and abs(over[0::40].astype(np.int64)).sum() == 65541
    b16 = np.zeros(41, np.int16); b16[0::4] = 5958; b16[0] += 65536 - 5958 * 11                         # branch 0 of U = 4: exactly 65536
    assert abs(b16[0::4].astype(np.int64)).sum() == 65536
    long_ = np.zeros(40 * 255 + 1, np.int16); long_[40 * 127] = 16384                                  # 4095 < ntaps
    wide = np.zeros(4 * 255 + 3, np.int16); wide[510] = 16384                                           # odd, ceil(ntaps / 4) = 256
    n_events = eng.launches
    bad = {"nchannels 0": (xp, 1000, 1000, cp, 0, 40, 11, tp, nt, op, 3637), "nchannels 17": (xp, 1000, 1000, cp, 17, 40, 11, tp, nt, op, 3637),
           "decim 0": (xp, 1000, 1000, cp, 4, 40, 0, tp, nt, op, 3637), "decim 17": (xp, 1000, 1000, cp, 4, 40, 17, tp, nt, op, 3637),
           "interp < decim": (xp, 1000, 1000, cp, 4, 10, 11, tp, nt, op, 3637), "interp 65": (xp, 1000, 1000, cp, 4, 65, 11, tp, nt, op, 3637),
           "not coprime": (xp, 1000, 1000, cp, 4, 44, 11, tp, nt, op, 3637), "interp = decim = 2": (xp, 1000, 1000, cp, 4, 2, 2, tp, nt, op, 3637),
           "ntaps even": (xp, 1000, 1000, cp, 4, 40, 11, tp, nt - 1, op, 3637), "ntaps > 4095": (xp, 1000, 1000, cp, 4, 40, 11, long_.ctypes.data, len(long_), op, 3637),
           "branch of 256": (xp, 1000, 1000, cp, 4, 4, 1, wide.ctypes.data, len(wide), op, 3637),
           "branch sum": (xp, 1000, 1000, cp, 4, 40, 11, over.ctypes.data, len(over), op, 3637),
           "branch sum 65536": (xp, 1000, 1000, cp, 4, 4, 1, b16.ctypes.data, len(b16), op, 3637),
           "gain 65536": (xp, 1000, 1000, C.addressof(hot), 2, 40, 11, tp, nt, op, 3637),
           "stride < n_in": (xp, 996, 1000, cp, 4, 40, 11, tp, nt, op, 3637), "stride % 4": (xp, 1002, 1000, cp, 4, 40, 11, tp, nt, op, 3637),
           "stride > 2^40": (xp, (1 << 40) + 4, 1000, cp, 4, 40, 11, tp, nt, op, 3637),
           "n_in > 2^40": (xp, 1 << 40, (1 << 40) + 1, cp, 4, 40, 11, tp, nt, op, 3637), "n_out > 2^40": (xp, 1000, 1000, cp, 4, 40, 11, tp, nt, op, (1 << 40) + 1),
           "accumulate 2": (xp, 1000, 1000, cp, 4, 40, 11, tp, nt, op, 3637, 2),
           "null rows": (0, 1000, 1000, cp, 4, 40, 11, tp, nt, op, 3637), "null channels": (xp, 1000, 1000, 0, 4, 40, 11, tp, nt, op, 3637),
           "null taps": (xp, 1000, 1000, cp, 4, 40, 11, 0, nt, op, 3637), "null out": (xp, 1000, 1000, cp, 4, 40, 11, tp, nt, 0, 3637)}
    for name, a in bad.items():
        assert _call(eng, *a) == -1, name
    d = torch.zeros(4 * 1000 * 2 + 8, dtype=torch.int16, device="cuda")
    assert _call(eng, d.data_ptr() + 4, 1000, 999, cp, 1, 40, 11, tp, nt, op, 3637) == -1, "misaligned device rows"
    assert _call(eng, xp, 1000, 1000, cp, 1, 40, 11, tp, nt, d.data_ptr() + 4, 3637) == -1, "misaligned device output"
    assert eng.launches == n_events, "a refused call launched"
    assert _call(eng, xp, 1000, 1000, cp, 4, 40, 11, at.ctypes.data, len(at), op, 3637) == 0          # a branch sum of 65535 is accepted
    b16[0] -= 1
    assert _call(eng, xp, 1000, 1000, cp, 4, 4, 1, b16.ctypes.data, len(b16), op, 3637) == 0
    one = np.array([32767], np.int16)
    assert _call(eng, xp, 1000, 1000, cp, 4, 1, 1, one.ctypes.data, 1, op, 1000) == 0                   # U = D = 1
    assert _call(eng, xp, 1000, 0, cp, 4, 40, 11, tp, nt, op, 3637) == 0                               # n_in = 0: all-zero rows
    assert (out[:3637] == 0).all()


# ---- end to end, device-resident: transmitters -> two combiner calls -> rational channelizers -> stream receivers ---------------------
@pytest.mark.parametrize("fs", [160e6, 176e6])
def test_24ghz_transmit_on_the_device(fs):
    """k_tx11b frames (COMPLEX8 widened on the device) and k_tx11a frames in device rows -> the 802.11b rows and then the OFDM row into one
    device buffer -> sb200_channel_sim (one link, one tap of 16384, no clock or carrier offset, noise of sigma 20 LSB) -> the rational
    channelizers -> sb200_rx11b_streams and sb200_rx11a_streams.  The capture, before and after the channel, equals the model chain on the
    oracle transmitters' output; the receivers equal the oracle on every field, event position and delivered byte; every PSDU delivered."""
    rows_h, mpdus, plan = frames_24ghz(); clean_h, _ = capture_of(fs, rows_h); y_h = through_the_air(clean_h)
    (ub, db), tb, (ua, da), ta = TX_PLANS[fs]; (rub, rdb), rtb, (rua, rda), rta = PLANS[fs]
    e = api.Engine(0); ea = api.Engine(0, cca_pwr_threshold=CCA_WIDE)
    try:
        n_b = max(len(rows_h[0]), len(rows_h[2])); sb_in = (n_b + 3) // 4 * 4; n_a = len(rows_h[1]); sa_in = (n_a + 3) // 4 * 4
        rb = torch.zeros((2, sb_in, 2), dtype=torch.int16, device="cuda"); ra_ = torch.zeros((1, sa_in, 2), dtype=torch.int16, device="cuda")
        for i, c in enumerate((0, 2)):
            for (t, rate, _), m in zip(plan[c], mpdus[c]):
                f = WD.tx11b(e, m, rate); rb[i, t:t + len(f)] = f.to(torch.int16) << 6
        for (t, rate, seed), m in zip(plan[1], mpdus[1]):
            f = WD.tx11a(e, m, rate, seed); ra_[0, t:t + len(f)] = f.to(torch.int16) * 20
        assert (rb[0, :len(rows_h[0])].cpu().numpy() == rows_h[0]).all() and (rb[1, :len(rows_h[2])].cpu().numpy() == rows_h[2]).all()
        assert (ra_[0, :n_a].cpu().numpy() == rows_h[1]).all()
        n = len(y_h); tx = torch.zeros((n, 2), dtype=torch.int16, device="cuda"); y = torch.zeros_like(tx)     # n is a multiple of 4
        e.combine_raw(rb.data_ptr(), sb_in, n_b, [(W.phase_inc(R.CH_24[c], fs), 0, GAIN_B) for c in (0, 2)], ub, tb, tx.data_ptr(), decim=db, n_out=n)
        e.combine_raw(ra_.data_ptr(), sa_in, n_a, [(0, 0, GAIN_A)], ua, ta, tx.data_ptr(), decim=da, n_out=n, accumulate=True)
        assert (tx.cpu().numpy() == clean_h).all()
        e.channel_sim_raw(tx.data_ptr(), n, n, 1, n, api.sim_links([SIM_LINK_24]), SIM_TAPS_24, 1, 1, SIM_SEED_24, y.data_ptr(), n, n, 1, n)
        assert (y.cpu().numpy() == y_h).all()
        def dev_rows(chans, u, d, t):
            n_out = -(-u * n // d); out = WD.dev_rows(len(chans), n_out, 64); stride = out.shape[1]
            e.channelize_raw(y.data_ptr(), n, [(W.phase_inc(R.CH_24[c], fs), 0) for c in chans], d, t, out.data_ptr(), stride, interp=u)
            return out, stride, n_out
        b_ch, a_ch = [0, 2], [1]
        db_, sb, nb = dev_rows(b_ch, rub, rdb, rtb); da_, sa, na = dev_rows(a_ch, rua, rda, rta)
        back = {c: R.channelize_rational(y_h, [(W.phase_inc(R.CH_24[c], fs), 0)], *((rub, rdb, rtb) if c != 1 else (rua, rda, rta)))[0] for c in range(3)}
        for i, c in enumerate(b_ch): assert (db_[i, :nb].cpu().numpy() == back[c]).all(), c
        assert (da_[0, :na].cpu().numpy() == back[1]).all()
        got_b = WD.rx11b(e, db_, sb, nb, len(b_ch)); got_a = WD.rx11a(ea, da_, sa, na, len(a_ch))
    finally:
        e.close(); ea.close()
    for i, (c, (o, _)) in enumerate(zip(b_ch, WD.equal_11b([back[c] for c in b_ch], got_b))):
        ps = _psdus(mpdus[c]); assert len(o) == len(ps), (c, len(o))
        for j in range(len(o)):
            L = int(o["length"][j]) - 1; assert bytes(got_b[1][i, j, :L]) == ps[j][:-1], (c, j)
    (o, _), = WD.equal_11a([back[1]], got_a); ps = _psdus(mpdus[1])
    assert len(o) == len(ps), len(o)
    for j in range(len(o)):
        L = int(o["length"][j]); assert bytes(got_a[1][0, j, :L]) == ps[j], j
