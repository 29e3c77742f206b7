"""The arbitrary-rate channelizer's model (tests/arbitrary_model.py, the arithmetic of sb200_channelize_arbitrary in include/sora_b200.h),
its table helper api.arbitrary_taps, and what it is for, without a GPU: its properties, then a 2.4 GHz capture at 122.88 Msps holding
802.11b on channels 1 and 11 and OFDM on channel 6, channelized in numpy to 44 Msps for the 802.11b receiver and 40 Msps for the OFDM
receiver and decoded by the CPU oracle.  test_gpu_channelize_arbitrary.py runs the same capture through the device."""
import numpy as np, pytest
import oracle_py
import wideband_inputs as W
import arbitrary_model as A
import sim_model
from sora_b200 import api
from test_cpu_channelize import _decoded, _full_scale, decode_11a

def _unit(ntaps):
    """Row 0 the unit impulse at k = c, the other rows arbitrary within the limits (64 taps of |t| < 1000)."""
    t = np.random.default_rng(ntaps).integers(-999, 1000, (256, ntaps)).astype(np.int16)
    t[0] = 0; t[0, (ntaps - 1) // 2] = 16384
    return t

@pytest.mark.parametrize("ntaps", [1, 2, 7, 8, 33, 64])
def test_identity(ntaps):
    """step = 2^32, tau0 = d 2^32, the identity channel and the unit-impulse row 0: y[m] = x[m + d] bit for bit, zero past the input."""
    x = _full_scale(3000, ntaps)
    for d in (0, 5, 2999):
        y = A.channelize_arbitrary(x, [(0, 0)], d << 32, 1 << 32, _unit(ntaps), 3001)[0]
        assert (y[:3000 - d] == x[d:]).all() and (y[3000 - d:] == 0).all(), (ntaps, d)

def test_simulator_stage_1():
    """ntaps = 8 with sb200_channel_sim's H is that call's interpolation stage across its step range."""
    x = _full_scale(5000, 3); H = sim_model.H.astype(np.int16)
    for tau0, step in ((0, 1 << 32), (3 * 2 ** 32 + 12345, (1 << 32) + (1 << 24)), (2 ** 31, (1 << 32) - (1 << 24)), (77 << 30, api.clock_step(-40))):
        n_out = 4900
        want = sim_model.interpolate(x, tau0, step, np.arange(n_out))
        assert (A.channelize_arbitrary(x, [(0, 0)], tau0, step, H, n_out)[0] == want).all(), (tau0, step)

def test_an_impulse_returns_the_rows():
    """x = -32768 at n0 through the identity channel: y[m] = (-32768 H[p_m][n0 - i_m + c] + 2^13) >> 14 where that index is a tap, else 0."""
    for ntaps, step in ((64, api.arbitrary_step(122.88e6, 44e6)), (33, 1 << 28), (8, 1 << 34), (7, (1 << 32) - 1)):
        H = np.random.default_rng(ntaps).integers(-2000, 2000, (256, ntaps)).astype(np.int16); c = (ntaps - 1) // 2; n0 = 300
        x = np.zeros((700, 2), np.int16); x[n0, 0] = -32768
        n_out = A.n_inside(700, 12345, step); y = A.channelize_arbitrary(x, [(0, 0)], 12345, step, H, n_out)[0]
        i, p = A._times(12345, step, 0, n_out); k = n0 - i + c; at = (k >= 0) & (k < ntaps)
        assert (y[at, 0] == ((-32768 * H[p[at], k[at]].astype(np.int64) + (1 << 13)) >> 14)).all() and (y[~at] == 0).all() and (y[:, 1] == 0).all(), ntaps

@pytest.mark.parametrize("fs_in,fs_out", [(122.88e6, 44e6), (122.88e6, 40e6), (30.72e6, 40e6), (61.44e6, 44e6)])
def test_a_tone_lands_at_its_offset(fs_in, fs_out):
    """A tone at f_c + delta comes out at delta of the output rate with the table's float response at delta."""
    n, f, Aamp = 20000, 10e6, 8000.0; step = api.arbitrary_step(fs_in, fs_out)
    H = api.arbitrary_taps(fs_in, fs_out, 64, 9e6)
    for delta in (0.0, 3e6, 7e6):
        z = Aamp * np.exp(2j * np.pi * (f + delta) / fs_in * np.arange(n) + 0.7j)
        x = np.stack([np.round(z.real), np.round(z.imag)], 1).astype(np.int16)
        m = np.arange(100, A.n_inside(n, 0, step) - 100)
        y = A.channelize_arbitrary_window(x, [(W.phase_inc(f, fs_in), 0)], 0, step, H, int(m[0]), int(m[-1]) + 1)[0].astype(np.float64)
        v = (y[:, 0] + 1j * y[:, 1]) * np.exp(-2j * np.pi * delta / fs_out * m)
        # the float response of the rows at delta, each row at its own fractional delay
        gain = np.abs((H / 16384.0) @ np.exp(2j * np.pi * delta / fs_in * np.arange(64)))
        assert abs(abs(v.mean()) - Aamp * gain.mean()) < 0.01 * Aamp and np.abs(np.abs(v) - Aamp * gain.mean()).max() < 0.03 * Aamp, (delta, gain.min(), gain.max())

def test_a_window_of_outputs_needs_only_its_inputs():
    x = _full_scale(6001, 12); ch = [(0, 0), (2 ** 29, 0), (0x9E3779B9, 0xDEADBEEF)]
    for tau0, step, H in ((0, api.arbitrary_step(122.88e6, 44e6), api.arbitrary_taps(122.88e6, 44e6, 64, 9e6)), (5 << 31, 1 << 28, _unit(33)),
                          (12345, 1 << 34, api.arbitrary_taps(4, 1, 7, 0.1))):
        n_out = A.n_inside(6001, tau0, step) + 20; full = A.channelize_arbitrary(x, ch, tau0, step, H, n_out)
        old = A.SLICE
        try:
            A.SLICE = 37                                                 # slices inside the windows, too
            for m0, m1 in ((0, 7), (0, n_out), (n_out // 2 - 5, n_out // 2 + 90), (n_out - 3, n_out)):
                assert (A.channelize_arbitrary_window(x, ch, tau0, step, H, m0, m1) == full[:, m0:m1]).all(), (step, m0, m1)
        finally:
            A.SLICE = old


# ---- the table helper -------------------------------------------------------------------------------------------------------------
def _response(H, fs_in, f):
    """|float response| of every row at the frequencies f (Hz): [256, len(f)]."""
    return np.abs((H / 16384.0) @ np.exp(-2j * np.pi * np.outer(np.arange(H.shape[1]), np.asarray(f) / fs_in)))

def _prototype(H, fs_in, f):
    """|float response| at f (Hz) of the filter the rows sample: tap k of row p is its value at d = k - c - p / 256 input samples, one
    sample of a prototype at 256 fs_in.  Its stop band holds both what a decimation folds into the passband and the images of an
    interpolation."""
    c = (H.shape[1] - 1) // 2; d = (256 * (np.arange(H.shape[1])[None, :] - c) - np.arange(256)[:, None]).ravel()
    return np.abs(np.exp(-2j * np.pi * np.outer(f, d) / (256 * fs_in)) @ (H.ravel() / (256 * 16384.0)))

# (fs_in, fs_out, passband Hz, stop band Hz): the plans of the 122.88 Msps capture below, and the rates of the 30.72 MHz family
PLANS = [(122.88e6, 44e6, 9e6, 17e6), (122.88e6, 40e6, 8.3e6, 17e6), (61.44e6, 44e6, 9e6, 17e6), (30.72e6, 40e6, 8.3e6, None), (30.72e6, 44e6, 9e6, None)]

@pytest.mark.parametrize("fs_in,fs_out,fp,fs", PLANS)
def test_arbitrary_taps_meet_the_limits(fs_in, fs_out, fp, fs):
    """Every row has a DC gain of exactly 16384 and sum |H| <= 65535 and ripples by less than 0.1 dB over the passband; the prototype is
    60 dB down over the stop band, to four times the input rate."""
    H = api.arbitrary_taps(fs_in, fs_out, 64, fp, fs).astype(np.int64)
    fs = min(fs_in, fs_out) - fp if fs is None else fs
    assert H.shape == (256, 64) and (H.sum(1) == 16384).all() and (np.abs(H).sum(1) <= 65535).all()
    rp = 20 * np.log10(_response(H, fs_in, np.linspace(-fp, fp, 101)))
    assert np.abs(rp).max() < 0.1, np.abs(rp).max()
    rs = 20 * np.log10(_prototype(H, fs_in, np.linspace(fs, 4 * fs_in, 3000)))
    assert rs.max() < -60, rs.max()

def test_arbitrary_taps_rows_are_fractional_delays():
    """Row p advances by p / 256 of an input sample (the output of row p stands at i + p / 256 and reads inputs i - c + k): a tone's
    phase through it at a low frequency matches, and row 0 of an odd table is symmetric."""
    H = api.arbitrary_taps(122.88e6, 44e6, 63, 9e6).astype(np.float64); w = 2 * np.pi * 8e6 / 122.88e6
    delay = np.angle((H / 16384.0) @ np.exp(1j * w * (np.arange(63) - 31))) / w                  # in input samples, at 8 MHz
    assert np.abs(delay - np.arange(256) / 256).max() < 1 / 512
    assert (H[0] == H[0][::-1]).all()


# ---- end to end through the CPU oracle --------------------------------------------------------------------------------------------------
FS = 122.88e6
GRID = 768                                             # 6.25 us: 250 samples at 40 Msps, 275 at 44 Msps
STEP_44, STEP_40 = api.arbitrary_step(FS, 44e6), api.arbitrary_step(FS, 40e6)
TAPS_44 = api.arbitrary_taps(FS, 44e6, 64, 9e6, 17e6)  # 802.11b main lobe to 11 MHz
TAPS_40 = api.arbitrary_taps(FS, 40e6, 64, 8.3e6, 17e6)  # OFDM to 8.3 MHz; the 802.11b neighbours' main lobes begin at 14 MHz

def rows_24ghz():
    """capture_24ghz_grid(122.88 Msps) channelized by the model: -> (capture, {channel: row}, psdus); 802.11b rows at 44 Msps, the OFDM
    row at 40 Msps."""
    iq, fcs, kinds, ps = A.capture_24ghz_grid(FS, GRID)
    rows = {}
    for c, (f, kind) in enumerate(zip(fcs, kinds)):
        step, t = (STEP_44, TAPS_44) if kind == "11b" else (STEP_40, TAPS_40)
        rows[c] = A.channelize_arbitrary(iq, [(W.phase_inc(f, FS), 0)], 0, step, t, A.n_inside(len(iq), 0, step))[0]
    return iq, rows, ps

def test_24ghz_capture_at_122_88():
    """802.11b on channels 1 and 11 and OFDM on channel 6 of one 122.88 Msps capture, one 64-tap table per rate: every channel returns
    exactly its own PSDUs (802.11b without the last FCS byte), every one with a good FCS, and nothing of its neighbours."""
    _, rows, ps = rows_24ghz()
    for c, kind in enumerate(A.R.KIND_24):
        if kind == "11b":
            r, o = oracle_py.rx11b_run(rows[c], max_frames=16, out_stride=4096); got = _decoded(r, o, lambda L: L - 1)
        else:
            (r, o), = decode_11a([rows[c]]); got = _decoded(r, o, lambda L: L)
        own = [bytes(p[:-1]) if kind == "11b" else bytes(p) for p in ps[c]]
        assert got == own, (c, len(got), len(own))
        assert (r["status"] == oracle_py.E_FRAME_OK).all(), (c, r["status"])
