"""GPU tests of the filter-bank combiner (sb200_combine_bank, pytest -m gpu): bit for bit against the numpy model of
tests/combine_bank_model.py over lengths, grids, interpolations, stackings, tap counts, full-scale and rail rows, n_out and accumulate;
the pointer residency, streams, launch bookkeeping and argument checks of the C ABI; the device's sb200_combine within the header's bound;
and the transmit chains of test_cpu_combine_bank.py run on the device, all device-resident, against the model chain and the CPU oracle."""
import ctypes as C
import numpy as np, pytest
import torch
import oracle_py
import wideband_inputs as W
import wideband_device as WD
import bank_model as B
import combine_bank_model as CB
import combine_rational_model as CR
import rational_model as R
from sora_b200 import api
from test_gpu_abi_residency import _matrix, _each, _fill
from test_cpu_channelize import CCA_WIDE
from test_cpu_combine import _psdus
from test_cpu_combine_bank import GRID, TAPS_TX, combine_taps, OFDM_ROWS, F_11B, GAIN_11B, FRAMES_11B, max_taps, frames_octet, frames_11b_row, mixed_capture
from test_cpu_channelize_rational import TAPS_160_44
from test_cpu_combine_rational import TAPS_44_160

pytestmark = pytest.mark.gpu
V, U32, U64 = C.c_void_p, C.c_uint32, C.c_uint64

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

def _rows(M, n, seed, amp=32768):
    return np.random.default_rng(seed).integers(-amp, amp, (M, n, 2)).astype(np.int16)

def _taps(n, seed):
    return np.random.default_rng(seed).integers(-32768, 32768, n).astype(np.int16)

def _tile(M, U):
    return U * 1024 // M                                   # outputs per CTA of k_combine_bank<M>

def _same(eng, x, U, odd, taps, n_out=None, acc=None):
    M, n_in = x.shape[:2]; n = U * n_in if n_out is None else n_out
    out = None if acc is None else acc.copy()
    got = eng.combine_bank(x, U, taps, odd=odd, n_out=n_out, accumulate=acc is not None, out=out)
    want = CB.window(x, M, U, odd, taps, 0, n, acc)
    assert got.shape == want.shape and (got == want).all(), (M, U, odd, len(taps), np.argwhere((got != want).any(1))[:5].ravel())

@pytest.mark.parametrize("n", [1, 60, 255, 256, 257, 1000, 3001])
def test_lengths(eng, n):
    """n_in of 1, below ntaps, and around the tile (256 inputs at M = 4, 128 at M = 8)."""
    _same(eng, _rows(8, n, n), 4, 1, _taps(255, n))
    _same(eng, _rows(4, n, n + 1), 2, 0, _taps(511, n + 1))

@pytest.mark.parametrize("M,U", GRID)
def test_grid(eng, M, U):
    """Every M = 2 .. 64 and every U | M, both stackings, full-scale rows and taps."""
    n = 3 * 1024 // M + 37
    for odd in (0, 1):
        nt = [1, 3, 2 * U + 1, max_taps(M, U)][(M + U + odd) % 4]
        _same(eng, _rows(M, n, M * 64 + U + odd), U, odd, _taps(nt, M + U + odd))

@pytest.mark.parametrize("ntaps", [1, 3, 5, 31, 63, 65, 127, 255, 257, 511, 1021, 1023])
def test_ntaps(eng, ntaps):
    """Tap counts 1 .. 1023 up to the 2048 U / M edge (the largest halo of each grid)."""
    for M, U in ((2, 1), (4, 2), (8, 4), (16, 16), (64, 64), (64, 32)):
        if ntaps <= max_taps(M, U):
            _same(eng, _rows(M, 4 * 1024 // M + 99, ntaps + M), U, ntaps % 2, _taps(ntaps, ntaps + U))

def test_rails_at_m64(eng):
    """Full-scale and rail rows at M = 64, where W is at its extremes, with +-32767 taps whose branch sums exceed 65535 (no tap-sum limit):
    the int64 filter and the saturation at the end."""
    rng = np.random.default_rng(64)
    rails = np.where(rng.random((64, 300, 2)) < 0.5, -32768, 32767).astype(np.int16)
    same = np.full((64, 300, 2), -32768, np.int16)                         # every row alike: W_0 at its largest
    for U in (1, 8, 64):
        nt = max_taps(64, U); t = np.where(rng.random(nt) < 0.5, -32767, 32767).astype(np.int16)
        assert max(int(np.abs(t[r::U].astype(np.int64)).sum()) for r in range(U)) > 65535
        for x in (rails, same, _rows(64, 300, U)):
            for odd in (0, 1):
                _same(eng, x, U, odd, t)

@pytest.mark.parametrize("M,U", [(8, 4), (2, 1), (64, 16)])
def test_n_out(eng, M, U):
    """n_out 0 (nothing launched), shorter than, equal to and longer than U n_in (the filter's tail, then zeros)."""
    x = _rows(M, 700, M + U); taps = _taps(max_taps(M, U), U)
    n0 = eng.launches; out = np.full((0, 2), 0, np.int16)
    eng.combine_bank(x, U, taps, n_out=0, out=out); assert eng.launches == n0
    for n in (1, U * 700 - 13, U * 700, U * 700 + 1000):
        _same(eng, x, U, 1, taps, n_out=n)

def test_accumulate(eng):
    """accumulate onto random and rail contents, host and device out."""
    x = _rows(16, 900, 31); taps = _taps(255, 31); U = 4; n = U * 900 + 17
    rng = np.random.default_rng(5)
    for acc in (rng.integers(-32768, 32768, (n, 2)), np.where(rng.random((n, 2)) < 0.5, -32768, 32767)):
        acc = acc.astype(np.int16)
        _same(eng, x, U, 1, taps, n, acc)
        d_in = torch.from_numpy(np.ascontiguousarray(x)).cuda(); d_out = torch.from_numpy(acc.copy()).cuda()
        eng.combine_bank_raw(d_in.data_ptr(), 900, 900, 16, U, taps, d_out.data_ptr(), n, odd=True, accumulate=True)
        assert (d_out.cpu().numpy() == CB.window(x, 16, U, 1, taps, 0, n, acc)).all()

@pytest.mark.parametrize("M,U,ntaps", [(8, 4, 255), (64, 64, 1023), (2, 1, 63), (64, 1, 31)])
def test_long_capture(eng, M, U, ntaps):
    """4 x SMs tiles plus 777 outputs, device-resident; the first, middle and last outputs against the model's windows."""
    n_out = 4 * WD.sms() * _tile(M, U) + 777; n = -(-n_out // U); stride = (n + 3) // 4 * 4
    x = np.zeros((M, stride, 2), np.int16); x[:, :n] = _rows(M, n, M + ntaps); taps = _taps(ntaps, M)
    d_in = torch.from_numpy(x).cuda(); d_out = torch.zeros((n_out, 2), dtype=torch.int16, device="cuda")
    for odd in (0, 1):
        eng.combine_bank_raw(d_in.data_ptr(), stride, n, M, U, taps, d_out.data_ptr(), n_out, odd=odd)
        mid = n_out // 2
        for n0, n1 in ((0, 300), (mid - 150, mid + 150), (n_out - 300, n_out)):
            got = d_out[n0:n1].cpu().numpy(); want = CB.window(x[:, :n], M, U, odd, taps, n0, n1)
            assert (got == want).all(), (M, U, odd, n0)


# ---- the C ABI ----------------------------------------------------------------------------------------------------------------------
def test_residency(eng):
    """rows and out each host or device, with and without accumulate (a host out is uploaded first); the bytes after out untouched."""
    M, n, stride, U = 8, 1001, 1008, 4; n_out = U * n + 5; taps = _taps(255, 50)
    rows = np.full((M, stride, 2), 0x5A5A, np.int16); rows[:, :n] = _rows(M, n, 50)
    args = dict(rows=rows, out=_fill(n_out * 4 + 16))
    ref = _matrix(lambda p: eng.combine_bank_raw(p["rows"], stride, n, M, U, taps, p["out"], n_out, odd=True), args, _each(*args))
    assert (ref["out"][:n_out * 4].view(np.int16).reshape(-1, 2) == CB.window(rows[:, :n], M, U, 1, taps, 0, n_out)).all()
    assert (ref["out"][n_out * 4:] == 0xA5).all()
    acc = ref["out"].copy(); args = dict(rows=rows, out=acc)
    ref2 = _matrix(lambda p: eng.combine_bank_raw(p["rows"], stride, n, M, U, taps, p["out"], n_out, odd=True, accumulate=True), args, _each(*args))
    want = CB.window(rows[:, :n], M, U, 1, taps, 0, n_out, acc[:n_out * 4].view(np.int16).reshape(-1, 2))
    assert (ref2["out"][:n_out * 4].view(np.int16).reshape(-1, 2) == want).all() and (ref2["out"][n_out * 4:] == 0xA5).all()

def test_caller_stream_one_launch_and_timing():
    e = api.Engine(0)
    try:
        M, U, n = 16, 4, 20000; x = _rows(M, n, 60); taps = _taps(255, 60)
        d_in = torch.from_numpy(x).cuda(); s = torch.cuda.Stream(); s.wait_stream(torch.cuda.current_stream())
        for acc in (False, True):
            with torch.cuda.stream(s):
                d_out = torch.zeros((U * n, 2), dtype=torch.int16, device="cuda")
                n0 = e.launches
                e.combine_bank_raw(d_in.data_ptr(), n, n, M, U, taps, d_out.data_ptr(), U * n, odd=acc, accumulate=acc, stream=s.cuda_stream)
                assert e.launches - n0 == 1
                got = d_out.cpu().numpy()
            assert e.last_kernel_ms() > 0 and (got == CB.combine_bank(x, U, int(acc), taps)).all()
    finally:
        e.close()

def _call(eng, rows, stride, n, M, U, odd, taps, ntaps, out, n_out, acc=0):
    return eng._lib.sb200_combine_bank(eng._h, V(rows), U64(stride), U64(n), U32(M), U32(U), U32(odd), V(taps), U32(ntaps), V(out), U64(n_out), U32(acc), V(0))

def test_invalid_arguments_are_rejected(eng):
    x = _rows(64, 1000, 70); out = np.full((4 * 1000, 2), 0x1234, np.int16); before = out.copy()
    t = _taps(255, 70); xp, op, tp = x.ctypes.data, out.ctypes.data, t.ctypes.data
    t257 = _taps(257, 71); t1025 = _taps(1025, 72); t33 = _taps(33, 73)
    n_events = eng.launches
    bad = {"M 0": (xp, 1000, 1000, 0, 1, 0, tp, 255, op, 4000), "M 1": (xp, 1000, 1000, 1, 1, 0, tp, 255, op, 4000),
           "M 6": (xp, 1000, 1000, 6, 2, 0, tp, 255, op, 4000), "M 128": (xp, 1000, 1000, 128, 4, 0, tp, 255, op, 4000),
           "U 0": (xp, 1000, 1000, 8, 0, 0, tp, 255, op, 4000), "U 3": (xp, 1000, 1000, 8, 3, 0, tp, 255, op, 4000),
           "U 16 > M": (xp, 1000, 1000, 8, 16, 0, tp, 255, op, 4000), "odd 2": (xp, 1000, 1000, 8, 4, 2, tp, 255, op, 4000),
           "ntaps even": (xp, 1000, 1000, 8, 4, 0, tp, 254, op, 4000), "ntaps 0": (xp, 1000, 1000, 8, 4, 0, tp, 0, op, 4000),
           "ntaps 1025": (xp, 1000, 1000, 2, 2, 0, t1025.ctypes.data, 1025, op, 4000),
           "ntaps > 2048 U / M": (xp, 1000, 1000, 8, 1, 0, t257.ctypes.data, 257, op, 4000),
           "ntaps > 2048 U / M at 64": (xp, 1000, 1000, 64, 1, 0, t33.ctypes.data, 33, op, 4000),
           "accumulate 2": (xp, 1000, 1000, 8, 4, 0, tp, 255, op, 4000, 2),
           "stride < n_in": (xp, 996, 1000, 8, 4, 0, tp, 255, op, 4000), "stride % 4": (xp, 1002, 1000, 8, 4, 0, tp, 255, op, 4000),
           "stride > 2^40": (xp, (1 << 40) + 4, 1000, 8, 4, 0, tp, 255, op, 4000),
           "n_in > 2^40": (xp, 1 << 40, (1 << 40) + 1, 8, 4, 0, tp, 255, op, 4000), "n_out > 2^40": (xp, 1000, 1000, 8, 4, 0, tp, 255, op, (1 << 40) + 1),
           "null rows": (0, 1000, 1000, 8, 4, 0, tp, 255, op, 4000), "null taps": (xp, 1000, 1000, 8, 4, 0, 0, 255, op, 4000),
           "null out": (xp, 1000, 1000, 8, 4, 0, tp, 255, 0, 4000)}
    for name, a in bad.items():
        assert _call(eng, *a) == -1, name
    d = torch.zeros(8 * 1000 * 2 + 8, dtype=torch.int16, device="cuda")
    assert _call(eng, d.data_ptr() + 4, 1000, 999, 8, 4, 0, tp, 255, op, 4000) == -1, "misaligned device rows"
    dout = torch.full((4000 * 2 + 8,), 0x1234, dtype=torch.int16, device="cuda")
    assert _call(eng, xp, 1000, 1000, 8, 4, 0, tp, 255, dout.data_ptr() + 4, 3999) == -1, "misaligned device output"
    assert eng.launches == n_events, "a refused call launched"
    assert (out == before).all() and (dout.cpu().numpy() == 0x1234).all(), "a refused call wrote out"
    assert _call(eng, xp, 1000, 1000, 8, 1, 0, tp, 255, op, 4000) == 0                     # ntaps = 255 <= 2048 / 8 is accepted
    assert _call(eng, xp, 1000, 1000, 64, 1, 0, t33.ctypes.data, 31, op, 4000) == 0        # 31 <= 32 at M = 64, U = 1
    assert _call(eng, xp, 1000, 0, 8, 4, 0, tp, 255, op, 4000) == 0                        # n_in = 0: all-zero rows
    assert (out == 0).all()

@pytest.mark.parametrize("M", [2, 4, 8, 16])
def test_against_the_device_combiner(eng, M):
    """The bank against the device's sb200_combine at channels {(2k + o) 2^31 / M, 0, 4096}, within the header's bound where nothing
    saturates."""
    for U in sorted({1, M // 2, M}):
        x = _rows(M, 5000, M * 10 + U, 6000 // M); x[M - 1] = 0
        taps = combine_taps(M, U)
        for odd in (0, 1):
            bank = eng.combine_bank(x, U, taps, odd=odd).astype(np.int64)
            comb = eng.combine(x, CB.channels(M, odd), U, taps).astype(np.int64)
            assert np.abs(comb).max() < 32767 and np.abs(bank).max() < 32767
            assert np.abs(bank - comb).max() <= CB.combine_bound(x, taps, U), (M, U, odd)


# ---- end to end, device-resident ----------------------------------------------------------------------------------------------------
def _equal_to_the_oracle_11a(rows, got, want):
    """The receiver equal to the oracle on the model chain's rows, and every PSDU of want[c] delivered on row c."""
    res, out, _, cnt = got
    for c, (o, _) in enumerate(WD.equal_11a(rows, got)):
        assert sum(o["status"] == oracle_py.E_FRAME_OK) == len(want[c]), (c, cnt[c], o)
        for i in range(len(o)):
            L = int(o["length"][i]); assert bytes(out[c, i, :L]) == want[c][i], (c, i)

def _dev_rows_11a(e, rows_h, plan, mpdus):
    """k_tx11a frames (x 20) in device rows at the oracle rows' positions; checked against them -> (device [8, stride, 2], stride)."""
    n = rows_h.shape[1]; d = WD.dev_rows(8, n); stride = d.shape[1]
    for c, (t, rate, seed) in plan.items():
        f = WD.tx11a(e, mpdus[c][0], rate, seed); d[c, t:t + len(f)] = f.to(torch.int16) * 20
    assert (d[:, :n].cpu().numpy() == rows_h).all()
    return d, stride

def test_octet_round_trip_on_the_device():
    """k_tx11a frames in device rows -> sb200_combine_bank (M = 8, U = 4, odd) -> sb200_channelize_bank (D = 4) -> sb200_rx11a_streams,
    every stage against its model; the receiver equal to the oracle on the model chain, every PSDU on its own channel."""
    rows_h, mpdus, plan = frames_octet(); n = rows_h.shape[1]
    y_h = CB.combine_bank(rows_h, 4, 1, TAPS_TX); back_h = B.bank(y_h, 8, 4, 1, B.TAPS_BANK)
    e = api.Engine(0, cca_pwr_threshold=CCA_WIDE)
    try:
        d, stride = _dev_rows_11a(e, rows_h, plan, mpdus)
        y = torch.zeros((4 * n, 2), dtype=torch.int16, device="cuda")
        e.combine_bank_raw(d.data_ptr(), stride, n, 8, 4, TAPS_TX, y.data_ptr(), 4 * n, odd=True)
        assert (y.cpu().numpy() == y_h).all()
        rows = WD.dev_rows(8, n, 64); rs = rows.shape[1]
        e.channelize_bank_raw(y.data_ptr(), 4 * n, 8, 4, B.TAPS_BANK, rows.data_ptr(), rs, odd=True)
        assert (rows[:, :n].cpu().numpy() == back_h).all()
        got = WD.rx11a(e, rows, rs, n, 8)
    finally:
        e.close()
    _equal_to_the_oracle_11a(back_h, got, [_psdus(mpdus[c]) for c in range(8)])

def test_mixed_capture_on_the_device():
    """OFDM rows on four bank channels by sb200_combine_bank, then an 802.11b row over two empty channels added by
    sb200_combine_rational(accumulate = 1); sb200_channelize_bank into sb200_rx11a_streams and sb200_channelize_rational into
    sb200_rx11b_streams.  Every stage equals its model; the receivers equal the oracle, every PSDU delivered."""
    y_h, first_h, rows_h, mpdus, rb_h, mb = mixed_capture(); n_out = len(y_h); n = rows_h.shape[1]
    back_h = B.bank(y_h, 8, 4, 1, B.TAPS_BANK)
    row_b_h = R.channelize_rational(y_h, [(W.phase_inc(F_11B, 160e6), 0)], 11, 40, TAPS_160_44)[0]
    _, _, plan = frames_octet(OFDM_ROWS)
    e = api.Engine(0, cca_pwr_threshold=CCA_WIDE)
    try:
        d, stride = _dev_rows_11a(e, rows_h, plan, mpdus)
        y = torch.zeros((n_out, 2), dtype=torch.int16, device="cuda")
        e.combine_bank_raw(d.data_ptr(), stride, n, 8, 4, TAPS_TX, y.data_ptr(), n_out, odd=True)
        assert (y.cpu().numpy() == first_h).all()
        nb = len(rb_h); rb = WD.dev_rows(1, nb); sb = rb.shape[1]; t = 500
        for (rate, _), m in zip(FRAMES_11B, mb):
            f = WD.tx11b(e, m, rate); rb[0, t:t + len(f)] = f.to(torch.int16) << 6; t += len(f) + 900
        assert (rb[0, :nb].cpu().numpy() == rb_h).all()
        e.combine_raw(rb.data_ptr(), sb, nb, [(W.phase_inc(F_11B, 160e6), 0, GAIN_11B)], 40, TAPS_44_160, y.data_ptr(), decim=11, n_out=n_out, accumulate=True)
        assert (y.cpu().numpy() == y_h).all()
        no = n_out // 4; rows = WD.dev_rows(8, no, 64); rs = rows.shape[1]
        e.channelize_bank_raw(y.data_ptr(), n_out, 8, 4, B.TAPS_BANK, rows.data_ptr(), rs, odd=True)
        assert (rows[:, :no].cpu().numpy() == back_h).all()
        ofdm = torch.stack([rows[c] for c in OFDM_ROWS]).contiguous()
        got_a = WD.rx11a(e, ofdm, rs, no, len(OFDM_ROWS))
        nbo = len(row_b_h); row_b = WD.dev_rows(1, nbo); sbo = row_b.shape[1]
        e.channelize_raw(y.data_ptr(), n_out, [(W.phase_inc(F_11B, 160e6), 0)], 40, TAPS_160_44, row_b.data_ptr(), sbo, interp=11)
        assert (row_b[0, :nbo].cpu().numpy() == row_b_h).all()
        got_b = WD.rx11b(e, row_b, sbo, nbo, 1)
    finally:
        e.close()
    _equal_to_the_oracle_11a(back_h[list(OFDM_ROWS)], got_a, [_psdus(mpdus[c]) for c in OFDM_ROWS])
    ps = _psdus(mb); (o, _), = WD.equal_11b([row_b_h], got_b)
    assert len(o) == len(ps), len(o)
    for j in range(len(o)):
        L = int(o["length"][j]) - 1; assert bytes(got_b[1][0, j, :L]) == ps[j][:-1], j
