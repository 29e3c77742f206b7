"""The wideband combiner's model (tests/combine_model.py, the arithmetic of sb200_combine in include/sora_b200.h) and what it is for,
without a GPU: its properties, then frames of the oracle's 802.11a / b / n transmitters placed in channel rows, combined into one wideband
capture and channelized again in numpy, and decoded by the CPU oracle's continuous-capture receivers, every channel on its own.  Which
cases decode is fixed here; test_gpu_combine.py runs the same chains on the device."""
import numpy as np
import oracle_py
import wideband_inputs as W
import combine_model as CM
from sora_b200 import synth
from test_cpu_channelize import TAPS_11A, TAPS_11B, _decoded, _full_scale, decode_11a

def test_an_impulse_returns_the_taps():
    """x = -32768 at m0 on channel (0, 0, 4096), U = 3: y[U m0 + c - j] = (-32768 t[j] + 2^14) >> 15 = -t[j] exactly, zero elsewhere."""
    taps = np.random.default_rng(3).integers(-6000, 6000, 41).astype(np.int16); c = 20; m0 = 40; U = 3; at = U * m0 + c - np.arange(41)
    x = np.zeros((1, 100, 2), np.int16); x[0, m0, 0] = -32768
    y = CM.combine(x, [(0, 0, 4096)], U, taps)
    assert len(y) == 300 and (y[at, 0] == -taps).all() and (np.delete(y[:, 0], at) == 0).all() and (y[:, 1] == 0).all()

def test_a_constant_comes_out_as_a_tone_at_fc():
    """A constant row through channel f_c: output n = U i + r sees branch r of the taps only, so its amplitude is A (branch sum / 32768)
    (gain / 4096), at the phase phase0 sets."""
    fs, f, U, A = 160e6, -25e6, 4, 9000
    taps = W.lowpass(63, 0.1, gain=U); inc = W.phase_inc(f, fs)
    for gain, ph in ((4096, 0), (2048, 0x40000000), (6000, 0x9E3779B9)):
        x = np.zeros((1, 3000, 2), np.int16); x[0, :, 0] = A
        y = CM.combine(x, [(inc, ph, gain)], U, taps)[200:-200].astype(np.float64)
        n = np.arange(200, 200 + len(y))
        base = (y[:, 0] + 1j * y[:, 1]) * np.exp(-2j * np.pi * (inc / 2 ** 32 * n + ph / 2 ** 32))      # back to 0 Hz
        for r in range(U):
            bsum = taps[(len(taps) // 2 - r) % U::U].astype(np.int64).sum()             # branch r: taps j = c - r (mod U)
            want = A * bsum / 32768 * gain / 4096
            assert np.abs(base[(r - 200) % U::U] - want).max() < 0.01 * A, (gain, r)

def test_quarter_turn_increments_are_exact():
    """phase_inc = 2^30 multiplies by +j each sample, 2^31 by -1: exact, the sign mirrored against the channelizer's."""
    x = _full_scale(4000, 4).astype(np.int64)
    neg = lambda a: np.clip(-a, -32768, 32767)
    want = np.empty_like(x)
    want[0::4] = x[0::4]
    want[1::4] = np.stack([neg(x[1::4, 1]), x[1::4, 0]], 1)                         # times +j
    want[2::4] = np.stack([neg(x[2::4, 0]), neg(x[2::4, 1])], 1)
    want[3::4] = np.stack([x[3::4, 1], neg(x[3::4, 0])], 1)                         # times -j
    assert (CM.rotate_up(x, 2 ** 30, 0) == want).all()
    assert (CM.rotate_up(x[2:], 2 ** 30, 2 ** 31) == want[2:]).all()                # a half-turn start: two samples later
    assert (CM.rotate_up(x, 2 ** 31, 0)[1::2] == neg(x[1::2])).all() and (CM.rotate_up(x, 2 ** 31, 0)[0::2] == x[0::2]).all()
    # through the combiner, identity filter and unity gain: the same turns
    y = CM.combine(x[None].astype(np.int16), [(2 ** 30, 0, 4096)], 1, np.array([32767], np.int16))
    assert (y == CM.rotate_up(CM.interpolate(x, 1, np.array([32767], np.int16)), 2 ** 30, 0)).all()

def test_the_channelizer_undoes_the_shift():
    """A channel sent with (phase_inc, phase0) and received with the same pair: the NCO terms cancel to within the table's rounding."""
    x = _full_scale(3000, 7) // 4
    for inc, ph in ((W.phase_inc(-20e6, 160e6), 0), (0x9E3779B9, 0x12345678), (2 ** 30, 5 << 20)):
        back = W.rotate(CM.rotate_up(x, inc, ph), inc, ph)
        assert np.abs(back - x).max() <= 8, (inc, ph)

def test_a_phase_offset_is_a_later_start():
    """A row delayed by m input samples comes out U m output samples later with phase0 advanced by U m phase_inc."""
    x = _full_scale(2000, 5) // 2; taps = W.lowpass(31, 0.1, gain=4)
    for inc, ph, m, U in ((W.phase_inc(-20e6, 160e6), 0x12345678, 77, 4), (0x9E3779B9, 0, 256, 3), (2 ** 30, 5, 3, 5)):
        xd = np.concatenate([np.zeros((m, 2), np.int16), x])
        y1 = CM.combine(x[None], [(inc, (ph + U * m * inc) % 2 ** 32, 4096)], U, taps)
        y2 = CM.combine(xd[None], [(inc, ph, 4096)], U, taps)
        assert (y2[U * m:] == y1).all(), (inc, m, U)

def test_gains_and_sums():
    """Gain 0 silences a channel, 4096 is unity; without saturation the sum of K one-channel outputs is the joint output."""
    rng = np.random.default_rng(8); taps = W.lowpass(63, 0.12, gain=4)
    rows = rng.integers(-3000, 3000, (3, 1500, 2)).astype(np.int16)
    ch = [(W.phase_inc(-40e6, 160e6), 0, 4096), (W.phase_inc(10e6, 160e6), 0xABCDEF01, 3000), (2 ** 31, 0, 7000)]
    assert (CM.combine(rows[:1], [(ch[0][0], 0, 0)], 4, taps) == 0).all()
    assert (CM.combine(rows[:1], ch[:1], 4, taps) == CM.rotate_up(CM.interpolate(rows[0], 4, taps), ch[0][0], 0)).all()
    joint = CM.combine(rows, ch, 4, taps); singles = [CM.combine(rows[k:k + 1], ch[k:k + 1], 4, taps).astype(np.int64) for k in range(3)]
    assert np.abs(joint).max() < 32767 and (joint == sum(singles)).all()
    gz = [(a, b, 0) if k == 1 else (a, b, g) for k, (a, b, g) in enumerate(ch)]
    assert (CM.combine(rows, gz, 4, taps) == singles[0] + singles[2]).all()

def test_a_window_of_outputs_needs_only_its_inputs():
    """combine_window (what the device tests of long captures compare with) equals the whole model on every window, edges included."""
    rows = np.stack([_full_scale(701, 6 + k) for k in range(3)]); taps = W.lowpass(255, 0.05, gain=1)
    ch = [(0, 0, 4096), (2 ** 29, 0, 65535), (0x9E3779B9, 0xDEADBEEF, 1234)]
    for u in (1, 4, 15):
        full = CM.combine(rows, ch, u, taps); n = len(full)
        for n0, n1 in ((0, 7), (0, n), (n // 2 - 5, n // 2 + 90), (n - 3, n), (3, 5)):
            assert (CM.combine_window(rows, ch, u, taps, n0, n1) == full[n0:n1]).all(), (u, n0, n1)


# ---- transmit -> combine -> channelize -> receive, through the CPU oracle ---------------------------------------------------------
TAPS_UP = W.lowpass(127, 0.1, gain=4)                  # 40 (44) -> 160 (176) Msps: each of the four branches near unity, sum |t| < 65535
U = 4

def rows_of(chans, n=None):
    """chans: per channel a list of (start, frame int [len, 2]) -> int16 [K, n, 2], the frames at their starts of zeroed rows."""
    n = n or max(s + len(f) for fr in chans for s, f in fr) + 400
    rows = np.zeros((len(chans), n, 2), np.int16)
    for k, fr in enumerate(chans):
        for s, f in fr: rows[k, s:s + len(f)] = f
    return rows

def _mpdu(n, seed):
    return np.random.RandomState(seed).randint(0, 256, n).astype(np.uint8)

def _psdus(mpdus):
    return [bytes(synth.psdu_with_fcs(m)) for m in mpdus]

RATES_11A = ((6000, 24000, 54000), (12000, 36000, 6000), (54000, 6000, 24000), (24000, 48000, 12000))
GAIN_11A = (4096, 4096, 40960, 4096)                   # channel 2 (+20 MHz) 20 dB above the others, through its gain

def frames_11a():
    """Four channels, three MPDUs each at different rates and staggered starts, COMPLEX8 scaled by 20 (the receiver loses a 54 Mbps frame
    at 16) -> (rows, [[mpdu, ...] per channel], [[(start, rate, scrambler seed), ...] per channel])."""
    chans, mpdus, plan = [], [], []
    for ci, rates in enumerate(RATES_11A):
        t, fr, ms, pl = 300 + 450 * ci, [], [], []
        for j, rate in enumerate(rates):
            m = _mpdu(116 + 60 * j + 20 * ci, 0x3E1A0000 + 16 * ci + j); seed = 1 + 7 * ci + j
            f = oracle_py.tx11a_modulate(m, rate, seed).astype(np.int16) * 20
            fr.append((t, f)); ms.append(m); pl.append((t, rate, seed)); t += len(f) + 750
        chans.append(fr); mpdus.append(ms); plan.append(pl)
    return rows_of(chans), mpdus, plan

def wide_11a(taps=TAPS_UP):
    """The 802.11a rows combined at 160 Msps (model), and channelized back to 40 Msps rows (model)."""
    rows, mpdus, _ = frames_11a()
    ch = [(W.phase_inc(f, W.FS_11A_WIDE), 0, g) for f, g in zip(W.CH_11A, GAIN_11A)]
    y = CM.combine(rows, ch, U, taps)
    return y, W.channelize(y, [(a, b) for a, b, _ in ch], 4, TAPS_11A), mpdus

def test_round_trip_11a():
    """Four 802.11a channels at -60 / -20 / +20 / +60 MHz of 160 Msps, the one at +20 MHz 20 dB up through its gain: every channel returns
    exactly its own PSDUs with a good FCS, nothing of its neighbours; no stage saturates."""
    y, back, mpdus = wide_11a()
    assert np.abs(y.astype(np.int64)).max() < 32767 and np.abs(back.astype(np.int64)).max() < 32767
    for c, (r, o) in enumerate(decode_11a(back)):
        assert _decoded(r, o, lambda L: L) == _psdus(mpdus[c]), c
        assert (r["status"] == oracle_py.E_FRAME_OK).all(), (c, r["status"])

def test_round_trip_11a_needs_the_filter():
    """The negative control: a single tap (zero-stuffing only) leaves the images of every channel 40 MHz away, on its neighbours.  The
    strong channel's images bury the weak channels, which decode none of their own frames; the strong one loses one of its three."""
    _, back, mpdus = wide_11a(np.array([32767], np.int16))
    own = [sum(d in _psdus(mpdus[c]) for d in _decoded(r, o, lambda L: L)) for c, (r, o) in enumerate(decode_11a(back))]
    assert own == [0, 0, 2, 0], own

RATES_11B = ((2000, 11000), (5500, 1000), (11000, 2000))

def frames_11b():
    """Three channels, two MPDUs each at 44 Msps, COMPLEX8 widened by << 6 (the receiver finds nothing at << 3) -> (rows, mpdus,
    [[(start, rate), ...] per channel])."""
    chans, mpdus, plan = [], [], []
    for ci, rates in enumerate(RATES_11B):
        t, fr, ms, pl = 400 + 600 * ci, [], [], []
        for j, rate in enumerate(rates):
            m = _mpdu(56 + 40 * j + 10 * ci, 0x3E1B0000 + 16 * ci + j)
            f = oracle_py.tx11b_modulate(m, rate).astype(np.int16) << 6
            fr.append((t, f)); ms.append(m); pl.append((t, rate)); t += len(f) + 1000
        chans.append(fr); mpdus.append(ms); plan.append(pl)
    return rows_of(chans), mpdus, plan

def wide_11b():
    rows, mpdus, _ = frames_11b()
    ch = [(W.phase_inc(f, W.FS_11B_WIDE), 0, 4096) for f in W.CH_11B]
    y = CM.combine(rows, ch, U, TAPS_UP_11B)
    return y, W.channelize(y, [(a, b) for a, b, _ in ch], 4, TAPS_11B), mpdus

TAPS_UP_11B = W.lowpass(127, 0.068, gain=4)

def test_round_trip_11b():
    """Three 802.11b channels at -25 / 0 / +25 MHz of 176 Msps (the PSDU is delivered without its last FCS byte)."""
    y, back, mpdus = wide_11b()
    assert np.abs(y.astype(np.int64)).max() < 32767
    for c in range(3):
        r, o = oracle_py.rx11b_run(back[c], max_frames=16, out_stride=4096)
        assert _decoded(r, o, lambda L: L - 1) == [p[:-1] for p in _psdus(mpdus[c])], c

def frames_11n(mcs=9):
    """Two channels, two MPDUs each, the int16 streams as they are -> (rows of stream 0, rows of stream 1, mpdus, [[(start, seed), ...]])."""
    c0, c1, mpdus, plan = [], [], [], []
    for ci in range(2):
        t, f0, f1, ms, pl = 350 + 550 * ci, [], [], [], []
        for j in range(2):
            m = _mpdu(96 + 50 * j + 30 * ci, 0x3E1C0000 + 16 * ci + j); seed = 3 + 5 * ci + j
            a, b = oracle_py.tx11n_modulate(m, mcs, seed)
            f0.append((t, a)); f1.append((t, b)); ms.append(m); pl.append((t, seed)); t += len(a) + 750
        c0.append(f0); c1.append(f1); mpdus.append(ms); plan.append(pl)
    n = max(s + len(f) for fr in c0 for s, f in fr) + 400
    return rows_of(c0, n), rows_of(c1, n), mpdus, plan

def wide_11n():
    r0, r1, mpdus, _ = frames_11n()
    ch = [(W.phase_inc(f, W.FS_11A_WIDE), 0, 4096) for f in W.CH_11N]
    y0, y1 = CM.combine(r0, ch, U, TAPS_UP), CM.combine(r1, ch, U, TAPS_UP)                 # stream s to antenna s
    dd = [(a, b) for a, b, _ in ch]
    return (y0, y1), (W.channelize(y0, dd, 4, TAPS_11A), W.channelize(y1, dd, 4, TAPS_11A)), mpdus

def test_round_trip_11n():
    """Two 802.11n 2x2 channels at -20 / +20 MHz, one combine per antenna."""
    (y0, y1), (b0, b1), mpdus = wide_11n()
    assert max(np.abs(y0.astype(np.int64)).max(), np.abs(y1.astype(np.int64)).max()) < 32767
    for c in range(2):
        r, o = oracle_py.rx11n_run(b0[c], b1[c], max_frames=16, out_stride=2048)
        assert _decoded(r, o, lambda L: L) == _psdus(mpdus[c]), c
