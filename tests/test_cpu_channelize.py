"""The wideband channelizer's model (tests/wideband_inputs.py, the arithmetic of sb200_channelize in include/sora_b200.h) and what it is
for, without a GPU: its properties, then 802.11a / b / n captures holding several channels, channelized in numpy and decoded by the CPU
oracle's continuous-capture receivers, every channel on its own.  Which cases decode is fixed here; test_gpu_channelize.py runs the same
captures through the device."""
import ctypes as C
import numpy as np, pytest
import oracle_py
import wideband_inputs as W
from test_gpu_fir import fir_model, HALF_BAND_31

CCA_WIDE = 100 * 100                                   # 802.11a carrier-sense threshold for the wideband captures (see test_wideband_11a)

def _full_scale(n, seed):
    rng = np.random.default_rng(seed)
    x = rng.integers(-32768, 32768, (n, 2)).astype(np.int16)
    x[rng.random((n, 2)) < 0.05] = -32768; x[rng.random((n, 2)) < 0.05] = 32767        # the rails
    return x

def test_identity_channel_with_d2_is_the_fir_decimator():
    x = _full_scale(9001, 1)
    assert (W.channelize(x, [(0, 0)], 2, HALF_BAND_31)[0] == fir_model(x, HALF_BAND_31)).all()
    taps = np.random.default_rng(2).integers(-3000, 3000, 63).astype(np.int16); taps[31] = 20000
    assert (W.channelize(x, [(0, 0)], 2, taps)[0] == fir_model(x, taps)).all()

def test_an_impulse_returns_the_taps():
    """x = -32768 at n0 through the identity channel, D = 1: y[n0 + c - k] = (-32768 t[k] + 2^14) >> 15 = -t[k] exactly, zero elsewhere;
    with D = 3 every third of them."""
    taps = np.random.default_rng(3).integers(-20000, 20000, 41).astype(np.int16); c = 20; n0 = 100; at = n0 + c - np.arange(41)
    x = np.zeros((300, 2), np.int16); x[n0, 0] = -32768
    y = W.channelize(x, [(0, 0)], 1, taps)[0]
    assert (y[at, 0] == -taps).all() and (np.delete(y[:, 0], at) == 0).all() and (y[:, 1] == 0).all()
    y3 = W.channelize(x, [(0, 0)], 3, taps)[0]
    assert (y3[at[at % 3 == 0] // 3, 0] == -taps[at % 3 == 0]).all()

def test_a_tone_at_fc_comes_out_at_0hz():
    fs, f = 160e6, 25e6; n = 8000; A = 12000
    t = np.arange(n); z = A * np.exp(2j * np.pi * f / fs * t + 0.7j)
    x = np.stack([np.round(z.real), np.round(z.imag)], 1).astype(np.int16)
    taps = W.lowpass(63, 0.05)
    y = W.channelize(x, [(W.phase_inc(f, fs), 0)], 4, taps)[0][40:-40].astype(np.float64)
    v = y[:, 0] + 1j * y[:, 1]
    assert abs(abs(v.mean()) - A * taps.sum() / 32768) < 0.01 * A and abs(np.angle(v.mean()) - 0.7) < 0.02
    assert np.abs(v - v.mean()).max() < 0.01 * A                                    # a constant: the phase error of a 12-bit NCO index only

def test_quarter_turn_increments_are_exact():
    x = _full_scale(4000, 4).astype(np.int64)
    neg = lambda a: np.clip(-a, -32768, 32767)
    want = np.empty_like(x)
    want[0::4] = x[0::4]
    want[1::4] = np.stack([x[1::4, 1], neg(x[1::4, 0])], 1)                         # times -j
    want[2::4] = np.stack([neg(x[2::4, 0]), neg(x[2::4, 1])], 1)
    want[3::4] = np.stack([neg(x[3::4, 1]), x[3::4, 0]], 1)                         # times +j
    assert (W.rotate(x, 2 ** 30, 0) == want).all()
    assert (W.rotate(x[2:], 2 ** 30, 2 ** 31) == want[2:]).all()                   # a half-turn start: two samples later
    assert (W.rotate(x, 2 ** 31, 0)[1::2] == neg(x[1::2])).all() and (W.rotate(x, 2 ** 31, 0)[0::2] == x[0::2]).all()

def test_a_phase_offset_is_a_later_start():
    x = _full_scale(5000, 5)
    for inc, ph, n0 in ((W.phase_inc(-20e6, 160e6), 0x12345678, 777), (0x9E3779B9, 0, 4096), (2 ** 30, 5, 3)):
        assert (W.rotate(x[n0:], inc, (ph + n0 * inc) % 2 ** 32) == W.rotate(x, inc, ph)[n0:]).all()
    y = W.channelize(x, [(0x9E3779B9, 0)], 4, W.lowpass(31, 0.1))[0]
    z = W.channelize(x[400:], [(0x9E3779B9, 400 * 0x9E3779B9 % 2 ** 32)], 4, W.lowpass(31, 0.1))[0]
    assert (y[100 + 8: -8] == z[8: len(y) - 100 - 8]).all()                       # away from the edges where the two captures differ

def test_a_window_of_outputs_needs_only_its_inputs():
    """channelize_window (what the device tests of long captures compare with) equals the whole model on every window, edges included."""
    x = _full_scale(3001, 6); taps = W.lowpass(255, 0.05); ch = [(0, 0), (2 ** 29, 0), (0x9E3779B9, 0xDEADBEEF)]
    for d in (1, 4, 15):
        full = W.channelize(x, ch, d, taps); n_out = full.shape[1]
        for m0, m1 in ((0, 7), (0, n_out), (n_out // 2 - 5, n_out // 2 + 90), (n_out - 3, n_out)):
            assert (W.channelize_window(x, ch, d, taps, m0, m1) == full[:, m0:m1]).all(), (d, m0, m1)


# ---- end to end through the CPU oracle --------------------------------------------------------------------------------------------------
TAPS_11A = W.lowpass(127, 0.1)                         # 160 Msps: passes 8.3 MHz, 60 dB down from about 20 MHz
TAPS_11B = W.lowpass(127, 0.068)                       # 176 Msps: passes the 11 MHz main lobe

def _decoded(res, out, nbytes):
    return [bytes(out[i, :nbytes(int(res["length"][i]))]) for i in range(len(res)) if res["status"][i] == oracle_py.E_FRAME_OK]

def channels_11a(taps=TAPS_11A):
    iq, fcs, ps = W.capture_11a()
    return W.channelize(iq, [(W.phase_inc(f, W.FS_11A_WIDE), 0) for f in fcs], 4, taps), ps

def decode_11a(rows):
    """The oracle's RxThread on every row, with the carrier-sense threshold the wideband captures need."""
    oracle_py.lib().sbo_set_cca_threshold(C.c_uint32(CCA_WIDE))
    try:
        return [oracle_py.rx11a_run(r, max_frames=16, out_stride=4096) for r in rows]
    finally:
        oracle_py.lib().sbo_set_cca_threshold(C.c_uint32(0))

def test_wideband_11a():
    """Four 802.11a channels at -60 / -20 / +20 / +60 MHz of a 160 Msps capture, the one at +20 MHz 20 dB above the others, D = 4 to
    40 Msps: every channel returns exactly its own PSDUs with a good FCS, nothing of its neighbours.  The weak channels sit 20 dB below
    the strong one in an int16 capture, below the default carrier-sense threshold (10^6, a full-scale single channel): it is lowered to
    10^4, as for any capture whose channels share the converter's range."""
    rows, ps = channels_11a()
    for c, (r, o) in enumerate(decode_11a(rows)):
        assert _decoded(r, o, lambda L: L) == [bytes(p) for p in ps[c]], c
        assert (r["status"] == oracle_py.E_FRAME_OK).all(), (c, r["status"])

def test_wideband_11a_needs_the_filter():
    """The negative control: a single tap (decimation only) folds the channels 40 MHz apart onto each other; none of the weak channels
    decodes a frame of its own, the strong one only one of its three."""
    rows, ps = channels_11a(np.array([32767], np.int16))
    own = [sum(d in [bytes(p) for p in ps[c]] for d in _decoded(r, o, lambda L: L)) for c, (r, o) in enumerate(decode_11a(rows))]
    assert own == [0, 0, 1, 0], own

def channels_11b():
    iq, fcs, ps = W.capture_11b()
    return W.channelize(iq, [(W.phase_inc(f, W.FS_11B_WIDE), 0) for f in fcs], 4, TAPS_11B), ps

def test_wideband_11b():
    """Three 802.11b channels at -25 / 0 / +25 MHz of a 176 Msps capture, D = 4 to 44 Msps (the PSDU is delivered without its last FCS byte)."""
    rows, ps = channels_11b()
    for c in range(3):
        r, o = oracle_py.rx11b_run(rows[c], max_frames=16, out_stride=4096)
        assert _decoded(r, o, lambda L: L - 1) == [bytes(p[:-1]) for p in ps[c]], c

def channels_11n():
    (a0, a1), fcs, ps = W.capture_11n()
    ch = [(W.phase_inc(f, W.FS_11A_WIDE), 0) for f in fcs]
    return W.channelize(a0, ch, 4, TAPS_11A), W.channelize(a1, ch, 4, TAPS_11A), ps

def test_wideband_11n():
    """Two 802.11n 2x2 channels at -20 / +20 MHz, both antennas at 160 Msps, D = 4 to 40 Msps."""
    r0, r1, ps = channels_11n()
    for c in range(2):
        r, o = oracle_py.rx11n_run(r0[c], r1[c], max_frames=16, out_stride=2048)
        assert _decoded(r, o, lambda L: L) == [bytes(p) for p in ps[c]], c
