"""The arbitrary-rate combiner's model (tests/combine_arbitrary_model.py, the arithmetic of sb200_combine_arbitrary in include/sora_b200.h)
and what it is for, without a GPU: its properties, then the oracle transmitters' 802.11b frames (44 Msps) and OFDM frames (40 Msps)
combined into one 122.88 Msps capture with two calls into one buffer, passed through the channel simulator's model with noise, channelized
again by the arbitrary-rate channelizer's model and decoded by the CPU oracle, every channel on its own.  test_gpu_combine_arbitrary.py
runs the same chain on the device."""
import numpy as np, pytest
import oracle_py
import wideband_inputs as W
import arbitrary_model as A
import combine_arbitrary_model as CA
import rational_model as R
from sora_b200 import api
from test_cpu_channelize import _full_scale
from test_cpu_channelize_arbitrary import FS, STEP_40, STEP_44, TAPS_40, TAPS_44, _unit
from test_cpu_channelize_rational import decode_24ghz
from test_cpu_combine import _psdus
from test_cpu_combine_rational import frames_24ghz, through_the_air

# rows at 44 and 40 Msps up to 122.88 Msps: the tables' default stop band puts the cut at the rows' Nyquist rate, which removes the images
UP_44, UP_40 = api.arbitrary_step(44e6, FS), api.arbitrary_step(40e6, FS)
UP_TAPS_44 = api.arbitrary_taps(44e6, FS, 64, 9e6)
UP_TAPS_40 = api.arbitrary_taps(40e6, FS, 64, 8.3e6)
CH3 = [(0, 0, 4096), (2 ** 29, 0, 65535), (0x9E3779B9, 0xDEADBEEF, 1234)]

@pytest.mark.parametrize("tau0,step,ntaps", [(0, UP_44, 64), (12345, UP_40, 64), (7 << 29, 1 << 28, 33), (3 << 31, 1 << 34, 8), (0, (1 << 32) + 1, 1)])
def test_one_identity_row_is_the_channelizer(tau0, step, ntaps):
    """One row through channel {0, 0, 4096} without accumulate is sb200_channelize_arbitrary's channel (0, 0): NCO[0] = (2^14, 0) and the
    Q12 gain of 4096 are exact identities."""
    x = _full_scale(3001, ntaps); H = np.random.default_rng(ntaps).integers(-255, 256, (256, ntaps)).astype(np.int16)
    n_out = A.n_inside(3001, tau0, step) + 40
    assert (CA.combine_arbitrary(x[None], [(0, 0, 4096)], tau0, step, H, n_out) == A.channelize_arbitrary(x, [(0, 0)], tau0, step, H, n_out)[0]).all()

@pytest.mark.parametrize("ntaps", [1, 2, 7, 8, 33, 64])
def test_unit_impulse_row_is_a_shift(ntaps):
    """step = 2^32, tau0 = d 2^32 and the unit-impulse row 0: y[n] = x[n + d] bit for bit, zero past the row."""
    x = _full_scale(3000, 40 + ntaps)
    for d in (0, 5, 2999):
        y = CA.combine_arbitrary(x[None], [(0, 0, 4096)], d << 32, 1 << 32, _unit(ntaps), 3001)
        assert (y[:3000 - d] == x[d:]).all() and (y[3000 - d:] == 0).all(), (ntaps, d)

def test_an_impulse_returns_the_rows():
    """x = -32768 at i0 through channel {0, 0, 4096}: y[n] = (-32768 H[p_n][i0 - i_n + c] + 2^13) >> 14 where that index is a tap, else 0."""
    for ntaps, step in ((64, UP_44), (33, 1 << 28), (8, 1 << 34), (7, (1 << 32) - 1)):
        H = np.random.default_rng(ntaps).integers(-2000, 2000, (256, ntaps)).astype(np.int16); c = (ntaps - 1) // 2; i0 = 300
        x = np.zeros((1, 700, 2), np.int16); x[0, i0, 0] = -32768
        n_out = A.n_inside(700, 12345, step); y = CA.combine_arbitrary(x, [(0, 0, 4096)], 12345, step, H, n_out)
        i, p = A._times(12345, step, 0, n_out); k = i0 - i + c; at = (k >= 0) & (k < ntaps)
        assert at.sum() > 0 and (y[at, 0] == ((-32768 * H[p[at], k[at]].astype(np.int64) + (1 << 13)) >> 14)).all(), ntaps
        assert (y[~at] == 0).all() and (y[:, 1] == 0).all(), ntaps

@pytest.mark.parametrize("fr,f", [(44e6, -25e6), (40e6, 0.0), (44e6, 25e6)])
def test_a_constant_becomes_a_tone_and_a_tone_moves_by_fc(fr, f):
    """A constant row comes out at f_c with every row of H at its unity DC gain; a tone at delta of the row rate comes out at f_c + delta
    of the capture rate with the table's float response at delta."""
    Amp, n = 8000, 6000; step = api.arbitrary_step(fr, FS); H = api.arbitrary_taps(fr, FS, 64, 9e6); inc = W.phase_inc(f, FS)
    x = np.zeros((1, n, 2), np.int16); x[0, :, 0] = Amp
    m = np.arange(300, A.n_inside(n, 0, step) - 300)
    y = CA.combine_arbitrary_window(x, [(inc, 0, 4096)], 0, step, H, int(m[0]), int(m[-1]) + 1).astype(np.float64)
    base = (y[:, 0] + 1j * y[:, 1]) * np.exp(-2j * np.pi * inc / 2 ** 32 * m)
    assert np.abs(base - Amp).max() < 0.01 * Amp                                         # the NCO's phase steps and roundings only
    for delta in (3e6, 7e6):
        z = Amp * np.exp(2j * np.pi * delta / fr * np.arange(n) + 0.4j); x = np.stack([np.round(z.real), np.round(z.imag)], 1)[None].astype(np.int16)
        y = CA.combine_arbitrary_window(x, [(inc, 0, 4096)], 0, step, H, int(m[0]), int(m[-1]) + 1).astype(np.float64)
        v = (y[:, 0] + 1j * y[:, 1]) * np.exp(-2j * np.pi * (f + delta) / FS * m)
        gain = np.abs((H / 16384.0) @ np.exp(2j * np.pi * delta / fr * np.arange(64)))    # every row at its own fractional delay
        assert abs(abs(v.mean()) - Amp * gain.mean()) < 0.01 * Amp and np.abs(np.abs(v) - Amp * gain.mean()).max() < 0.03 * Amp, (delta, gain.min(), gain.max())

def test_a_window_of_outputs_needs_only_its_inputs():
    rows = np.stack([_full_scale(2001, 50 + k) for k in range(3)])
    for tau0, step, H in ((0, UP_44, UP_TAPS_44), (5 << 31, 1 << 28, _unit(33)), (12345, 1 << 34, api.arbitrary_taps(4, 1, 7, 0.1))):
        n_out = A.n_inside(2001, tau0, step) + 20; full = CA.combine_arbitrary(rows, CH3, tau0, step, H, n_out)
        old = A.SLICE
        try:
            A.SLICE = 37                                                 # slices inside the windows, too
            for n0, n1 in ((0, 7), (0, n_out), (n_out // 2 - 5, n_out // 2 + 90), (n_out - 3, n_out), (3, 5)):
                assert (CA.combine_arbitrary_window(rows, CH3, tau0, step, H, n0, n1) == full[n0:n1]).all(), (step, n0, n1)
        finally:
            A.SLICE = old

def test_n_out_cuts_or_extends():
    """n_out defaults to the outputs whose time lies inside the rows; shorter is a prefix; longer adds the filter's tail and then zeros."""
    rows = (_full_scale(300, 9) // 4)[None]; ch = [(W.phase_inc(10e6, FS), 7, 4096)]
    full = CA.combine_arbitrary(rows, ch, 0, UP_44, UP_TAPS_44); n = len(full)
    assert n == A.n_inside(300, 0, UP_44) == -(-(300 << 32) // UP_44)
    assert (CA.combine_arbitrary(rows, ch, 0, UP_44, UP_TAPS_44, n - 100) == full[:n - 100]).all()
    long = CA.combine_arbitrary(rows, ch, 0, UP_44, UP_TAPS_44, n + 400)
    assert (long[:n] == full).all() and np.abs(long[n:n + 50].astype(np.int64)).max() > 0 and (long[n + 300:] == 0).all()

def test_accumulate_is_one_saturation():
    """accumulate: y = sat16(a + sum) exactly, on random and rail contents; two calls equal one joint call wherever no partial sum
    leaves int16."""
    rng = np.random.default_rng(12)
    rows = rng.integers(-6000, 6000, (3, 500, 2)).astype(np.int16)
    ch = [(W.phase_inc(-25e6, FS), 0, 4096), (W.phase_inc(25e6, FS), 0x12345678, 9000), (0, 0, 3000)]
    n_out = A.n_inside(500, 0, UP_44)
    plain = CA.combine_arbitrary(rows, ch, 0, UP_44, UP_TAPS_44, n_out).astype(np.int64)
    assert np.abs(plain).max() < 32767                                                 # the sum is not clipped, so sat16(a + sum) is exact here
    for a in (rng.integers(-32768, 32768, (n_out, 2)), np.where(rng.random((n_out, 2)) < 0.5, -32768, 32767)):
        a = a.astype(np.int16)
        got = CA.combine_arbitrary(rows, ch, 0, UP_44, UP_TAPS_44, n_out, acc=a)
        assert (got == np.clip(a.astype(np.int64) + plain, -32768, 32767)).all()
    first = CA.combine_arbitrary(rows[:1], ch[:1], 0, UP_44, UP_TAPS_44, n_out)
    two = CA.combine_arbitrary(rows[1:], ch[1:], 0, UP_44, UP_TAPS_44, n_out, acc=first)
    assert (two == plain).all()

def test_the_arbitrary_channelizer_undoes_it():
    """A tone sent with (phase_inc, phase0) and step s comes back from the arbitrary-rate channelizer with the same pair and step
    ~ 2^64 / s at its amplitude within 2 %."""
    Amp = 6000
    for fr, f, up, t_up, down, t_down in ((44e6, -25e6, UP_44, UP_TAPS_44, STEP_44, TAPS_44), (40e6, 0.0, UP_40, UP_TAPS_40, STEP_40, TAPS_40)):
        z = Amp * np.exp(2j * np.pi * 1.5e6 / fr * np.arange(3000) + 1.1j)
        x = np.stack([np.round(z.real), np.round(z.imag)], 1).astype(np.int16)
        inc = W.phase_inc(f, FS); ph = 0x0ABCDEF0
        y = CA.combine_arbitrary(x[None], [(inc, ph, 4096)], 0, up, t_up)
        back = A.channelize_arbitrary(y, [(inc, ph)], 0, down, t_down, A.n_inside(len(y), 0, down))[0][300:-300].astype(np.float64)
        m = np.arange(300, 300 + len(back)); v = (back[:, 0] + 1j * back[:, 1]) * np.exp(-2j * np.pi * 1.5e6 / fr * m)
        assert abs(abs(v.mean()) - Amp) < 0.02 * Amp and np.abs(v - v.mean()).max() < 0.02 * Amp, fr


# ---- transmit -> combine (two calls into one buffer) -> channelize -> receive, through the CPU oracle ------------------------------------
# The gains of test_cpu_combine_rational.py's chain: both the rational branches and these tables have unity DC gain, so the capture has the
# same levels.  Each 802.11b row at half scale and the OFDM row at twice its scale, 12 dB above each 802.11b row: the 36 Mbps frame needs
# that margin over what the 64-tap receive table lets through of the 802.11b neighbours 25 MHz away, and the sum still does not clip.
GAIN_B, GAIN_A = 2048, 8192

def capture_122_88(rows):
    """Two calls into one buffer: the 802.11b rows (44 Msps) at -25 and +25 MHz, then the OFDM row (40 Msps) at 0 Hz added onto them
    -> (int16 [n_out, 2], the first call's output)."""
    n_b = max(len(rows[0]), len(rows[2])); rb = np.zeros((2, n_b, 2), np.int16); rb[0, :len(rows[0])] = rows[0]; rb[1, :len(rows[2])] = rows[2]
    n_out = max(A.n_inside(n_b, 0, UP_44), A.n_inside(len(rows[1]), 0, UP_40)) + 400
    n_out += (-n_out) % 4
    chb = [(W.phase_inc(R.CH_24[c], FS), 0, GAIN_B) for c in (0, 2)]
    first = CA.combine_arbitrary(rb, chb, 0, UP_44, UP_TAPS_44, n_out)
    y = CA.combine_arbitrary(rows[1][None], [(0, 0, GAIN_A)], 0, UP_40, UP_TAPS_40, n_out, acc=first)
    return y, first

def channelize_122_88(y):
    """The capture back down by the arbitrary-rate channelizer's model: {channel: row}, 802.11b at 44 Msps, OFDM at 40 Msps."""
    return {c: A.channelize_arbitrary(y, [(W.phase_inc(f, FS), 0)], 0, *((STEP_44, TAPS_44) if kind == "11b" else (STEP_40, TAPS_40)),
                                      A.n_inside(len(y), 0, STEP_44 if kind == "11b" else STEP_40))[0]
            for c, (f, kind) in enumerate(zip(R.CH_24, R.KIND_24))}

def test_mixed_24ghz_transmit_at_122_88():
    """802.11b on channels 1 and 11 and OFDM on channel 6 sent into one 122.88 Msps capture, through the channel simulator's noise: every
    channel returns exactly its own PSDUs (802.11b without the last FCS byte), every one with a good FCS, and nothing of its neighbours;
    the capture does not clip."""
    rows, mpdus, _ = frames_24ghz()
    clean, _ = capture_122_88(rows)
    assert np.abs(clean.astype(np.int64)).max() < 32767
    y = through_the_air(clean)
    assert 18 < np.std((y.astype(np.int64) - clean)) < 22                               # the noise is there, at sigma = 20
    for c, (r, o, got) in decode_24ghz(channelize_122_88(y)).items():
        own = [p[:-1] if R.KIND_24[c] == "11b" else p for p in _psdus(mpdus[c])]
        assert got == own, (c, len(got), len(own))
        assert (r["status"] == oracle_py.E_FRAME_OK).all(), (c, r["status"])
