"""The rational-rate channelizer's model (tests/rational_model.py, the arithmetic of sb200_channelize_rational in include/sora_b200.h)
and what it is for, without a GPU: its properties, then one 2.4 GHz capture holding 802.11b on channels 1 and 11 and OFDM on channel 6,
at 160 and at 176 Msps, channelized in numpy to 44 Msps for the 802.11b receiver and 40 Msps for the OFDM receiver and decoded by the
CPU oracle, every channel on its own.  test_gpu_channelize_rational.py runs the same captures through the device."""
import numpy as np, pytest
import oracle_py
import wideband_inputs as W
import rational_model as R
from test_cpu_channelize import TAPS_11A, TAPS_11B, _decoded, _full_scale, decode_11a

def test_interp_1_is_the_channelizer():
    x = _full_scale(3001, 11); taps = W.lowpass(255, 0.05); ch = [(0, 0), (2 ** 29, 0), (0x9E3779B9, 0xDEADBEEF)]
    for d in range(1, 17):
        assert (R.channelize_rational(x, ch, 1, d, taps) == W.channelize(x, ch, d, taps)).all(), d

def test_an_impulse_returns_the_branch_taps():
    """x = -32768 at n0 through the identity channel: y[m] = -taps[U n0 - D m + c] wherever that index is a tap, zero elsewhere."""
    for U, D in ((11, 40), (5, 22), (3, 4), (16, 63)):
        taps = np.random.default_rng(U).integers(-3000, 3000, 10 * U + 1).astype(np.int16); c = len(taps) // 2; n0 = 57
        x = np.zeros((200, 2), np.int16); x[n0, 0] = -32768
        y = R.channelize_rational(x, [(0, 0)], U, D, taps)[0]
        k = U * n0 - D * np.arange(len(y)) + c; at = (k >= 0) & (k < len(taps))
        assert (y[at, 0] == -taps[k[at]]).all() and (y[~at] == 0).all() and (y[:, 1] == 0).all(), (U, D)

def test_a_tone_lands_at_its_offset():
    """A tone at f_c comes out at 0 Hz with the filter's branch gain, one at f_c + delta at delta of the output rate."""
    fs, f, U, D = 160e6, 25e6, 11, 40; n = 20000; A = 8000; taps = W.lowpass(1287, 12e6 / 1.76e9, gain=11); fo = fs * U / D
    for delta in (0.0, 3e6):
        z = A * np.exp(2j * np.pi * (f + delta) / fs * np.arange(n) + 0.7j)
        x = np.stack([np.round(z.real), np.round(z.imag)], 1).astype(np.int16)
        y = R.channelize_rational(x, [(W.phase_inc(f, fs), 0)], U, D, taps)[0][100:-100].astype(np.float64)
        v = (y[:, 0] + 1j * y[:, 1]) * np.exp(-2j * np.pi * delta / fo * np.arange(100, 100 + len(y)))
        assert abs(abs(v.mean()) - A) < 0.02 * A and np.abs(v - v.mean()).max() < 0.02 * A, delta

def test_a_window_of_outputs_needs_only_its_inputs():
    x = _full_scale(3001, 12); ch = [(0, 0), (2 ** 29, 0), (0x9E3779B9, 0xDEADBEEF)]
    for U, D, taps in ((1, 15, W.lowpass(255, 0.05)), (11, 40, W.lowpass(1287, 12e6 / 1.76e9, gain=11)), (5, 22, W.lowpass(505, 0.02, gain=5))):
        full = R.channelize_rational(x, ch, U, D, taps); n_out = full.shape[1]
        for m0, m1 in ((0, 7), (0, n_out), (n_out // 2 - 5, n_out // 2 + 90), (n_out - 3, n_out)):
            assert (R.channelize_rational_window(x, ch, U, D, taps, m0, m1) == full[:, m0:m1]).all(), (U, D, m0, m1)


# ---- end to end through the CPU oracle --------------------------------------------------------------------------------------------------
# fs -> ((U, D) to 44 Msps, its taps, (U, D) to 40 Msps, its taps).  160 -> 44: 117 taps per branch at 1.76 GHz, 0 dB to 8.3 MHz,
# -26 dB at 14 MHz, -86 dB at 20 MHz.  176 -> 40: 255 taps per branch at 880 MHz, 0 dB to 8.3 MHz, -88 dB at 14 MHz (where the 802.11b
# main lobes 25 MHz away begin).
TAPS_160_44 = W.lowpass(1287, 12e6 / 1.76e9, gain=11)
TAPS_176_40 = W.lowpass(1275, 11.3e6 / 880e6, gain=5)
PLANS = {160e6: ((11, 40), TAPS_160_44, (1, 4), TAPS_11A), 176e6: ((1, 4), TAPS_11B, (5, 22), TAPS_176_40)}

def rows_24ghz(fs):
    """capture_24ghz(fs) channelized by the model: -> (capture, {channel: row}, psdus); 802.11b rows at 44 Msps, the OFDM row at 40 Msps."""
    iq, fcs, kinds, ps = R.capture_24ghz(fs); (ub, db), tb, (ua, da), ta = PLANS[fs]
    rows = {}
    for c, (f, kind) in enumerate(zip(fcs, kinds)):
        u, d, t = (ub, db, tb) if kind == "11b" else (ua, da, ta)
        rows[c] = R.channelize_rational(iq, [(W.phase_inc(f, fs), 0)], u, d, t)[0]
    return iq, rows, ps

def decode_24ghz(rows):
    """Every row through the oracle receiver of its kind -> {channel: (results, bytes, delivered PSDUs)}."""
    out = {}
    for c, kind in enumerate(R.KIND_24):
        if kind == "11b":
            r, o = oracle_py.rx11b_run(rows[c], max_frames=16, out_stride=4096); out[c] = (r, o, _decoded(r, o, lambda L: L - 1))
        else:
            (r, o), = decode_11a([rows[c]]); out[c] = (r, o, _decoded(r, o, lambda L: L))
    return out

def test_tap_plans_fit_the_limits():
    for (ub, _), tb, (ua, _), ta in PLANS.values():
        for u, t in ((ub, tb), (ua, ta)):
            assert len(t) % 2 == 1 and -(-len(t) // u) <= 255
            assert max(int(np.abs(t[r::u].astype(np.int64)).sum()) for r in range(u)) <= 65535

@pytest.mark.parametrize("fs", [160e6, 176e6])
def test_mixed_24ghz_capture(fs):
    """802.11b on channels 1 and 11 and OFDM on channel 6 of one capture: every channel returns exactly its own PSDUs (802.11b without the
    last FCS byte), every one with a good FCS, and nothing of its neighbours."""
    _, rows, ps = rows_24ghz(fs)
    for c, (r, o, got) in decode_24ghz(rows).items():
        own = [bytes(p[:-1]) if R.KIND_24[c] == "11b" else bytes(p) for p in ps[c]]
        assert got == own, (fs, c, len(got), len(own))
        assert (r["status"] == oracle_py.E_FRAME_OK).all(), (fs, c, r["status"])
