"""The radio channel simulator's model (tests/sim_model.py, the arithmetic of sb200_channel_sim in include/sora_b200.h) and what it is for,
without a GPU: Philox4x32-10 against the Random123 known answers, the interpolation table, the statistics of the fixed-point Gaussian noise,
exact properties of the four stages, the accuracy of the resampler against channel_inputs.resample, and round trips of the oracle
transmitters' frames through multipath, clock and carrier offsets and noise into the oracle receivers.  frame_11a / frame_11b /
frame_11n build the links that test_gpu_channel_sim.py runs on the device."""
import numpy as np, pytest
import oracle_py
import channel_inputs as CI
import sim_model as SM
from wideband_inputs import NCO
from sora_b200 import api, synth

S32 = 1 << 32


# ---- Philox, tables, noise ----------------------------------------------------------------------------------------------------------
def test_philox_known_answers():
    """Random123's kat_vectors for philox4x32_10."""
    kat = [((0, 0, 0, 0, 0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 6, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344, 0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for args, want in kat:
        assert tuple(int(v) for v in SM.philox4x32_10(*args)) == want

def test_interpolation_table():
    """Row 0 is the unit impulse at k = 3 (a whole-sample delay is exact); H[256 - p][k] = H[p][7 - k]; every row sums to about 2^14."""
    assert (SM.H[0] == [0, 0, 0, 16384, 0, 0, 0, 0]).all()
    for p in range(1, 256):
        assert (SM.H[256 - p] == SM.H[p][::-1]).all(), p
    assert np.abs(SM.H.sum(1) - 16384).max() < 200 and np.abs(SM.H).sum(1).max() < 2 ** 31 // 32768

def test_noise_statistics():
    """2^22 outputs of each of three (row, link) streams at sigma = 100 LSB (noise_q8 = 25600); n = 2^23 components per stream.
    Tolerances, from the sampling error of n draws: the mean's standard error is 100 / sqrt(n) = 0.035, so |mean| < 0.25 is 7 of them;
    the variance's relative standard error is sqrt(2 / n) = 5e-4, and the output's rounding adds 1/12, so 1 % covers the table's
    quantisation too; P(|G| > 3 sigma) = 2.70e-3 has a relative standard error of 0.7 %, bounded at 5 %; P(|G| > 4 sigma) = 6.3e-5 one
    of 4.4 %, bounded at 25 % (the fixed-point tail sits a few % high, as a prototype over 2^23 draws found: 6.6e-5); correlations between
    re and im, at lag 1 and across rows and links have a standard error of 1 / sqrt(2^22) = 4.9e-4, bounded at 3e-3."""
    n, sig = 1 << 22, 25600
    m = np.arange(n, dtype=np.uint64) + np.uint64(2 ** 33 - 1000)           # across the counter's word boundary
    seed = 0x0123456789ABCDEF
    streams = [SM.noise(m, r, l, seed, sig).astype(np.float64) for r, l in ((0, 0), (1, 0), (0, 1))]
    g = streams[0]; s = sig / 256.0
    comp = g.reshape(-1)
    assert abs(comp.mean()) < 0.25 and np.abs(g.mean(0)).max() < 0.35
    var = comp.var() - 1 / 12
    assert abs(var / s ** 2 - 1) < 0.01, var / s ** 2
    p3, p4 = (np.abs(comp) > 3 * s).mean(), (np.abs(comp) > 4 * s).mean()
    assert abs(p3 / 2.6998e-3 - 1) < 0.05 and abs(p4 / 6.334e-5 - 1) < 0.25, (p3, p4)
    corr = lambda a, b: np.corrcoef(a, b)[0, 1]
    assert abs(corr(g[:, 0], g[:, 1])) < 3e-3
    assert max(abs(corr(g[:-1, k], g[1:, k])) for k in (0, 1)) < 3e-3
    for o in streams[1:]:
        assert max(abs(corr(g[:, k], o[:, k])) for k in (0, 1)) < 3e-3
    assert np.abs(g).max() <= 6.7 * s


# ---- exact properties -----------------------------------------------------------------------------------------------------------------
def _full(nl, T, n, seed):
    return np.random.default_rng(seed).integers(-32768, 32768, (nl, T, n, 2)).astype(np.int16)

def _unit(R, T, L=1, j=0):
    t = np.zeros((R, T, L, 2), np.int16)
    for r in range(min(R, T)): t[r, r, j, 0] = 16384
    return t

def test_a_neutral_link_is_the_identity():
    for T, L in ((1, 1), (2, 5), (4, 64)):
        x = _full(2, T, 3000, T)
        assert (SM.sim(x, [(0, S32, 0, 0, 0)] * 2, _unit(T, T, L), 3000) == x).all()

def test_whole_sample_delays_are_shifts():
    """tau0 = D 2^32 reads D samples later; a single tap at delay j gives the samples j earlier (zeros before the start)."""
    x = _full(1, 1, 2000, 3)
    for D in (1, 7, 100):
        y = SM.sim(x, [(D * S32, S32, 0, 0, 0)], _unit(1, 1), 2000)
        assert (y[0, 0, :2000 - D] == x[0, 0, D:]).all() and (y[0, 0, 2000 - D:] == 0).all()
    for j in (1, 17, 63):
        y = SM.sim(x, [(0, S32, 0, 0, 0)], _unit(1, 1, 64, j), 2000)
        assert (y[0, 0, j:] == x[0, 0, :2000 - j]).all() and (y[0, 0, :j] == 0).all()

def test_an_impulse_reads_out_every_row_of_h():
    """x = 16384 at i0, step 2^32, tau0 = p 2^24: s(m) = H[p][i0 - m + 3] for m in (i0 - 5, i0 + 3], zero elsewhere."""
    i0, n = 40, 64
    x = np.zeros((256, 1, n, 2), np.int16); x[:, 0, i0, 0] = 16384
    y = SM.sim(x, [(p << 24, S32, 0, 0, 0) for p in range(256)], _unit(1, 1), n)
    for p in range(256):
        want = np.zeros(n, np.int64); want[i0 + 3 - np.arange(8)] = SM.H[p]
        assert (y[p, 0, :, 0] == want).all() and (y[p, 0, :, 1] == 0).all(), p

def test_a_constant_becomes_the_nco_tone():
    A, inc, ph = 12000, 0x9E3779B9, 0x12345678
    x = np.zeros((1, 1, 4000, 2), np.int16); x[..., 0] = A
    y = SM.sim(x, [(0, S32, inc, ph, 0)], _unit(1, 1), 4000)[0, 0].astype(np.int64)
    th = (ph + np.arange(4000, dtype=np.uint64) * np.uint64(inc)) & np.uint64(0xFFFFFFFF)
    cs = NCO[(th >> np.uint64(20)).astype(np.int64)]
    assert (y[:, 0] == (A * cs[:, 0] + (1 << 13)) >> 14).all() and (y[:, 1] == (A * cs[:, 1] + (1 << 13)) >> 14).all()

def test_a_window_is_the_slice():
    x = _full(3, 2, 5000, 9); taps = np.random.default_rng(9).integers(-2000, 2000, (3, 2, 2, 11, 2)).astype(np.int16)
    links = [(3 * S32 + 12345, api.clock_step(37), 0x9E3779B9, 5, 700), ((1 << 31), api.clock_step(-40), 0, 0, 0), (0, S32 + (1 << 24), 3 << 30, 0, 25600)]
    full = SM.sim(x, links, taps, 4500, 2 ** 40 + 3)
    for m0, m1 in ((0, 10), (777, 1500), (4499, 4500), (4000, 4500)):
        assert (SM.sim_window(x, links, taps, 2 ** 40 + 3, m0, m1) == full[:, :, m0:m1]).all(), (m0, m1)


# ---- resampling accuracy ------------------------------------------------------------------------------------------------------------
def _frame_iq(rate, nbytes, seed, scale):
    m = np.random.RandomState(seed).randint(0, 256, nbytes).astype(np.uint8)
    return oracle_py.tx11a_modulate(m, rate, 1 + seed % 100).astype(np.int16) * scale, m

@pytest.mark.parametrize("ppm", [40, -40])
def test_resampling_accuracy(ppm):
    """802.11a at 40 Msps through the model's clock (step = clock_step(ppm)) against channel_inputs.resample (a 48-tap float resampler,
    below -80 dB of error): the error is 40 dB or more below the signal.  Measured: 45.4 dB at +40 ppm and at -40 ppm."""
    f, _ = _frame_iq(54000, 1000, 5, 128)
    x = np.zeros((1, 1, len(f) + 800, 2), np.int16); x[0, 0, 400:400 + len(f)] = f
    n_out = int(x.shape[2] * (1 + ppm * 1e-6)) - 8
    y = SM.sim(x, [(0, api.clock_step(ppm), 0, 0, 0)], _unit(1, 1), n_out)[0, 0].astype(np.float64)
    ref = CI.resample(x[0, 0, :, 0] + 1j * x[0, 0, :, 1], 1 + ppm * 1e-6)[:n_out]
    a, b = 600, n_out - 600
    err = (y[a:b, 0] + 1j * y[a:b, 1]) - ref[a:b]
    snr = 10 * np.log10((np.abs(ref[a:b]) ** 2).mean() / (np.abs(err) ** 2).mean())
    assert snr >= 40, snr


# ---- round trips through the oracle -------------------------------------------------------------------------------------------------
def fit_taps(delays, gains, L):
    """sim_taps of the profile, scaled down where a row's tap sum would pass 65535 (to 65000) -> (taps, channel power gain)."""
    g = [np.asarray(v, np.complex128) for v in gains]
    h = np.zeros(g[0].shape + (L,), np.complex128)
    for d, v in zip(delays, g): h[..., d] += v
    worst = (np.abs(h.real) + np.abs(h.imag)).reshape(-1 if g[0].ndim == 0 else g[0].shape[0], L if g[0].ndim == 0 else -1).sum(-1).max() * 16384
    s = min(1.0, 65000 / worst)
    return api.sim_taps(delays, [v * s for v in g], L), s * s

def _sigma_q8(iq, chan_gain, snr_db, rows=1):
    """noise_q8 for snr_db below the mean received power per row: the frame's mean power (over its rows) times the channel's power gain."""
    p = (iq.astype(np.float64) ** 2).sum(-1).mean() * chan_gain * rows
    return int(round(256 * np.sqrt(p / 10 ** (snr_db / 10) / 2)))

def _pad(frames, lead=400, trail=400):
    """T frames of one link -> int16 [1, T, si, 2], si a multiple of 4."""
    n = len(frames[0]); si = (lead + n + trail + 3) // 4 * 4
    x = np.zeros((1, len(frames), si, 2), np.int16)
    for t, f in enumerate(frames): x[0, t, lead:lead + n] = f
    return x

# Oscillator offsets, each with its matching carrier offset: the receivers' carrier-offset ranges set them.  802.11a at 5.2 GHz runs at
# +-25 ppm (130 kHz): a clean frame decodes at +-150 kHz and fails its SIGNAL field at +-208 kHz (40 ppm).  At 2.4 GHz the 802.11n
# receiver decodes +-20 ppm (48 kHz) and fails at +-40 ppm; the 802.11b receiver at 11 Mbps decodes +10 .. +40 ppm minus the ends and
# fails the FCS at -10 ppm and below, so it runs at +20 ppm.  The sampling clock alone is tested to +-40 ppm (test_resampling_accuracy).
PROFILE_11A = {6000: ("exp50ns", 25), 12000: ("exp150ns", -25), 24000: ("exp150ns", 25), 54000: ("exp50ns", -25)}

def link_for(ppm, fc, fs, sig):
    return (S32 // 3, api.clock_step(ppm), api.phase_inc(-ppm * 1e-6 * fc, fs), 0x1000000, sig)

def frame_11a(rate, snr, nl=1, L=32):
    """One 300-byte 802.11a frame (oracle transmitter, x 200: the receiver's carrier sense finds nothing of a clean frame at x 64, nor of
    one through exp150ns's taps (power gain 0.59) at x 128) through the profile of PROFILE_11A[rate] at 40 Msps, its ppm and the matching
    carrier offset at 5.2 GHz, noise snr dB below the received power -> (x [nl, 1, si, 2], psdu with FCS, links, taps [1, 1, L, 2], n_out, seed)."""
    name, ppm = PROFILE_11A[rate]
    f, m = _frame_iq(rate, 296, rate // 1000, 200)
    d, g = CI.exp_profile({"exp50ns": 50, "exp150ns": 150}[name], CI.FS_11A, 1 if name == "exp50ns" else 2)
    taps, pg = fit_taps(d, g, L)
    x = np.repeat(_pad([f]), nl, 0)
    n_out = int(x.shape[2] * (1 + ppm * 1e-6)) - 8; n_out -= n_out % 4
    links = [link_for(ppm, CI.FC_11A, CI.FS_11A, _sigma_q8(f, pg, snr))] * nl
    return x, synth.psdu_with_fcs(m), links, taps, n_out, 0x5EED0000 + rate

def decode_11a(y, n_out):
    nl = len(y); yy = np.ascontiguousarray(y[:, 0, :n_out])
    return oracle_py.rx11a_batch(yy.reshape(-1, 2), np.arange(nl, dtype=np.uint64) * n_out, np.full(nl, n_out, np.uint32), out_stride=4096)

def frame_11b(snr, nl=1, rate=11000, L=16):
    """One 100-byte 802.11b frame (oracle transmitter, << 6) at 44 Msps through exp50ns, +20 ppm and the matching offset at 2.4 GHz."""
    m = np.random.RandomState(rate).randint(0, 256, 96).astype(np.uint8)
    f = oracle_py.tx11b_modulate(m, rate).astype(np.int16) << 6
    taps, pg = fit_taps(*CI.exp_profile(50, CI.FS_11B, 7), L)
    x = np.repeat(_pad([f]), nl, 0)
    n_out = int(x.shape[2] * (1 + 20e-6)) - 8; n_out -= n_out % 4
    return x, synth.psdu_with_fcs(m), [link_for(20, CI.FC_11B, CI.FS_11B, _sigma_q8(f, pg, snr))] * nl, taps, n_out, 0x5EED11B0 + rate

def decode_11b(y, n_out):
    nl = len(y); yy = np.ascontiguousarray(y[:, 0, :n_out])
    return oracle_py.rx11b_batch(yy.reshape(-1, 2), np.arange(nl, dtype=np.uint64) * n_out, np.full(nl, n_out, np.uint32), out_stride=4096)

def frame_11n(mcs, snr, nl=1, L=16):
    """One 200-byte 802.11n 2x2 frame (oracle transmitter, both streams) through mimo_profile, -20 ppm and the matching offset at 2.4 GHz."""
    m = np.random.RandomState(mcs).randint(0, 256, 196).astype(np.uint8)
    a, b = oracle_py.tx11n_modulate(m, mcs, 0x5A)
    taps, pg = fit_taps(*CI.mimo_profile(mcs), L)
    x = np.repeat(_pad([a, b]), nl, 0)
    n_out = int(x.shape[2] * (1 - 20e-6)) - 8; n_out -= n_out % 4
    sig = _sigma_q8(np.concatenate([a, b]), pg, snr, rows=2)
    return x, synth.psdu_with_fcs(m), [link_for(-20, CI.FC_11B, CI.FS_11A, sig)] * nl, taps, n_out, 0x5EED11A0 + mcs

def decode_11n(y, n_out):
    nl = len(y); y0 = np.ascontiguousarray(y[:, 0, :n_out]); y1 = np.ascontiguousarray(y[:, 1, :n_out])
    return oracle_py.rx11n_batch(y0.reshape(-1, 2), y1.reshape(-1, 2), np.arange(nl, dtype=np.uint64) * n_out, np.full(nl, n_out, np.uint32), out_stride=1536)

def _got(res, out, psdu, drop=0):
    L = len(psdu) - drop
    return [bool(r["status"] == oracle_py.E_FRAME_OK and (o[:L] == psdu[:L]).all()) for r, o in zip(res, out)]

@pytest.mark.parametrize("rate", sorted(PROFILE_11A))
def test_round_trip_11a(rate):
    """Two links (different noise) of one frame at each rate: every PSDU at 30 dB SNR, none at -5 dB."""
    for snr, want in ((30, True), (-5, False)):
        x, psdu, links, taps, n_out, seed = frame_11a(rate, snr, nl=2)
        res, out = decode_11a(SM.sim(x, links, taps, n_out, seed), n_out)
        assert _got(res, out, psdu) == [want] * 2, (snr, res["status"])

@pytest.mark.parametrize("rate", [2000, 11000])
def test_round_trip_11b(rate):
    """The 802.11b receiver delivers the PSDU without its last FCS byte."""
    for snr, want in ((30, True), (-5, False)):
        x, psdu, links, taps, n_out, seed = frame_11b(snr, nl=2, rate=rate)
        res, out = decode_11b(SM.sim(x, links, taps, n_out, seed), n_out)
        assert _got(res, out, psdu, drop=1) == [want] * 2, (snr, res["status"])

@pytest.mark.parametrize("mcs", [8, 10])
def test_round_trip_11n(mcs):
    for snr, want in ((30, True), (-5, False)):
        x, psdu, links, taps, n_out, seed = frame_11n(mcs, snr, nl=2)
        res, out = decode_11n(SM.sim(x, links, taps, n_out, seed), n_out)
        assert _got(res, out, psdu) == [want] * 2, (snr, res["status"])


# ---- the Python helpers ---------------------------------------------------------------------------------------------------------------
def test_clock_step_and_sim_taps():
    assert api.clock_step(0) == S32 and api.clock_step(40) == round(S32 / 1.00004) and api.clock_step(-40) > S32
    t = api.sim_taps([0, 3], [0.5, -0.25j], 8)
    assert t.shape == (1, 1, 8, 2) and t[0, 0, 0].tolist() == [8192, 0] and t[0, 0, 3].tolist() == [0, -4096] and not t[0, 0, [1, 2, 4, 5, 6, 7]].any()
    d, g = CI.mimo_profile(1)
    m = api.sim_taps(d, [0.25 * v for v in g], 16)
    assert m.shape == (2, 2, 16, 2) and m[1, 0, 2, 0] == round(0.25 * g[1][1, 0].real * 16384)
    with pytest.raises(ValueError): api.sim_taps([16], [1.0], 16)
    with pytest.raises(ValueError): api.sim_taps([0, 1, 2, 3], [1.0, 1.0, 1.0, 1.0 + 0.01j], 8)
