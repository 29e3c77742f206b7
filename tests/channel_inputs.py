"""Receive-chain captures through frequency-selective channels and a sampling-clock offset (test input only).

Every other test capture goes through a flat channel: synth.to_iq16 adds noise, a carrier offset and a gain, and make_frames_11n applies
one 2x2 matrix to every subcarrier.  So the per-bin parts of the receivers (the 802.11a channel inverse, equaliser and pilot tracker, the
802.11n per-bin 2x2 inverse) only ever see channel coefficients of about one size, and no capture drifts against the receiver's sample
clock.  The captures here are rendered from the float modulators of synth (modulate, modulate_11b, modulate_11n) through a tapped delay
line at the capture rate and, for some, a band-limited resampler that models a sampling-clock offset; only then are they quantised to
int16 with a gain and seeded noise.

cases_11a(rate), cases_11n(mcs) and cases_11b(rate) return a list of (name, capture) for one chain: int16 [n, 2] (802.11n: a pair, one
per antenna), n a multiple of 28.  cases_11a(rate, fs_mhz=44) renders the same cases at 44 Msps.  stream_11a(), stream_11n() and
stream_11b() chain cases of several rates into one continuous capture.

Run as a script (python channel_inputs.py [oracle.so]) it passes every case through the CPU oracle's entry points, naming each case on
stdout before it runs and printing its batch status after: test_cpu_channels.py runs it against an oracle built with a trapping signed-
overflow check.
"""
import functools, os, sys
if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from sora_b200 import synth

FC_11A, FC_11B = 5.2e9, 2.4e9                          # carrier frequencies of the matched carrier offsets
SUBCARRIER_HZ = 312.5e3


# ---- channel models -----------------------------------------------------------------------------------------------------------------
def multipath(x, delays, gains):
    """Tapped delay line at the capture rate, complex float64: y[n] = sum_k g_k x[n - d_k], delays d_k in whole samples (>= 0).
    x [..., n] -> y [..., n + max(d)].  802.11n: x [2, n] holds the transmit chains and every g_k is a 2x2 matrix,
    y[a, n] = sum_k sum_b g_k[a, b] x[b, n - d_k]: a frequency-selective MIMO channel."""
    x = np.asarray(x, np.complex128)
    d = [int(v) for v in delays]
    assert len(d) == len(gains) and min(d) >= 0
    n = x.shape[-1]
    y = np.zeros(x.shape[:-1] + (n + max(d),), np.complex128)
    for dk, g in zip(d, gains):
        g = np.asarray(g, np.complex128)
        y[..., dk:dk + n] += g @ x if g.ndim == 2 else g * x
    return y

@functools.lru_cache(maxsize=None)
def _sinc_table(half, phases, beta):
    """Kaiser-windowed sinc of 2*half taps at phases + 1 fractional delays p / phases: row p weights x[i0 - half + 1 .. i0 + half] for
    the instant i0 + p / phases.  Rows 0 and `phases` are exact deltas (sinc vanishes on the other samples)."""
    k = np.arange(-half + 1, half + 1)
    u = k[None, :] - (np.arange(phases + 1) / phases)[:, None]
    w = np.sinc(u) * np.i0(beta * np.sqrt(np.clip(1 - (u / half) ** 2, 0, 1))) / np.i0(beta)
    w[0] = k == 0; w[phases] = k == 1
    return w

def resample(x, ratio, half=24, phases=1024, beta=8.0, chunk=16384):
    """Band-limited resampling in float64 along the last axis: y[m] = x(m / ratio), x interpolated with a Kaiser-windowed sinc of 2*half
    taps (zero outside x) whose fractional delay is interpolated linearly between `phases` tabulated ones: below -80 dB of error on
    signals within +-0.3 of the sample rate.  ratio > 1 gives more samples of the same stretch of signal; ratio 1 returns x unchanged, bit for bit."""
    x = np.asarray(x, np.complex128)
    n = x.shape[-1]
    m = int(np.floor((n - 1) * ratio + 1e-9)) + 1
    xp = np.concatenate([np.zeros(x.shape[:-1] + (half,)), x, np.zeros(x.shape[:-1] + (half + 1,))], -1)
    W = _sinc_table(half, phases, beta)
    k = np.arange(-half + 1, half + 1)
    y = np.zeros(x.shape[:-1] + (m,), np.complex128)
    for m0 in range(0, m, chunk):
        t = np.arange(m0, min(m, m0 + chunk)) / ratio
        i0 = np.floor(t).astype(np.int64); f = (t - i0) * phases
        p = np.floor(f).astype(np.int64); a = (f - p)[:, None]
        w = (1 - a) * W[p] + a * W[p + 1]
        y[..., m0:m0 + len(t)] = np.einsum("...tk,tk->...t", xp[..., (i0 + half)[:, None] + k[None, :]], w)
    return y

def sco(x, ppm, fs, fc=None):
    """x as captured by a receiver whose oscillator runs ppm parts per million fast against the transmitter's.  Its sample clock takes
    (1 + ppm 1e-6) times as many samples of the same signal; with fc (Hz) its mixer is as far off, which leaves a carrier offset of
    -ppm 1e-6 fc in the baseband (both offsets from one oscillator)."""
    y = resample(x, 1.0 + ppm * 1e-6)
    if fc is not None and ppm:
        y = y * np.exp(-2j * np.pi * ppm * 1e-6 * fc * np.arange(y.shape[-1]) / fs)
    return y

def quantise(y, gain=1.0, snr_db=None, seed=0, lead=400, trail=228):
    """Complex waveform in the modulators' int8 units [..., n] -> int16 [..., lead + n + trail', 2]: x 256 gain, complex AWGN snr_db below
    the mean power of y (all rows together, so a faded antenna gets the other one's noise), rounded, clipped to the int16 rails.  trail
    grows to make the length a multiple of 28."""
    y = np.asarray(y, np.complex128)
    trail += (-(lead + y.shape[-1] + trail)) % 28
    z = np.zeros(y.shape[:-1] + (lead + y.shape[-1] + trail,), np.complex128)
    z[..., lead:lead + y.shape[-1]] = y * (256.0 * gain)
    if snr_db is not None:
        p = (np.abs(z[..., lead:lead + y.shape[-1]]) ** 2).mean()
        sigma = np.sqrt(p / 10 ** (snr_db / 10) / 2)
        rng = np.random.default_rng(seed)
        z = z + rng.normal(0, sigma, z.shape) + 1j * rng.normal(0, sigma, z.shape)
    return np.clip(np.round(np.stack([z.real, z.imag], -1)), -32768, 32767).astype(np.int16)


# ---- channel profiles ---------------------------------------------------------------------------------------------------------------
def exp_profile(rms_ns, fs, seed, max_taps=32):
    """(delays, gains): an exponential power-delay profile with rms spread rms_ns, one tap per sample at fs, fewer than max_taps taps,
    every tap complex Gaussian (one Rayleigh draw per tap), total power 1."""
    s = rms_ns * 1e-9 * fs                                          # rms spread in samples; geometric profile r^k: rms = sqrt(r) / (1 - r)
    q = (np.sqrt(1 + 4 * s * s) - 1) / (2 * s)
    d = np.arange(min(max_taps - 1, int(np.ceil(6 * s)) + 1))
    rng = np.random.default_rng(seed)
    g = q ** d * (rng.normal(size=len(d)) + 1j * rng.normal(size=len(d))) / np.sqrt(2)
    return list(d), list(g / np.sqrt((np.abs(g) ** 2).sum()))

def two_ray_null(k, d, fs, depth_db=None):
    """(delays, gains) of two rays d samples apart whose sum cancels on 20 MHz subcarrier k: exactly (depth_db None) or to depth_db below
    the direct ray's power.  Total power 1."""
    a = 1.0 if depth_db is None else 1.0 - 10 ** (-depth_db / 20)
    g = np.array([1.0, a * np.exp(1j * (np.pi + 2 * np.pi * k * SUBCARRIER_HZ * d / fs))])
    return [0, d], list(g / np.sqrt((np.abs(g) ** 2).sum()))

def _turn(profile, phi):
    """The channel `profile` with every tap turned by phi radians."""
    d, g = profile
    return d, [x * np.exp(1j * phi) for x in g]

def _norm(delays, gains):
    g = np.asarray(gains, np.complex128)
    return list(delays), list(g / np.sqrt((np.abs(g) ** 2).sum()))


# ---- 802.11a ------------------------------------------------------------------------------------------------------------------------
FS_11A = 40e6

def _psdu(n, seed):
    r = np.random.RandomState(seed & 0xFFFFFFFF)
    return synth.psdu_with_fcs(r.randint(0, 256, n - 4).astype(np.uint8))

def _spec_11a(rate):
    """(name, psdu bytes, (delays, gains) at 40 Msps, ppm, carrier for a matched offset or None, snr_db) per case."""
    long_len = {6000: 2500, 12000: 2000, 24000: 1500, 54000: 1500}[rate]     # 2500 B: the longest PSDU the receiver accepts
    S = [
        ("exp50ns", 300, exp_profile(50, FS_11A, 1), 0, None, 30),          # rms spread 2 samples
        ("exp150ns", 300, exp_profile(150, FS_11A, 2), 0, None, 30),        # rms spread 6 samples, last tap 31: inside the 32-sample GI
        ("echo1.0us", 300, _norm([0, 40], [1, 0.35j]), 0, None, 30),        # beyond the 0.8 us guard interval: inter-symbol interference
        ("echo1.2us", 300, _norm([0, 48], [1, -0.5]), 0, None, 30),
        ("preecho", 300, _norm([0, 6], [0.6, 1.0]), 0, None, 30),           # the later path is the stronger one
        ("null_data+10", 300, two_ray_null(10, 3, FS_11A), 0, None, 30),      # exact nulls: on a data bin, on the pilots, next to DC
        ("null_pilot+7", 300, two_ray_null(7, 3, FS_11A), 0, None, 30),
        ("null_pilot-21", 300, two_ray_null(-21, 3, FS_11A), 0, None, 30),
        ("null_dc-1", 300, two_ray_null(-1, 2, FS_11A), 0, None, 30),
        ("nearnull40dB", 300, two_ray_null(-15, 3, FS_11A, 40), 0, None, 45),   # |Y|^2 >> 8 small: large channel-inverse coefficients
        ("notch21dB_trunc16", 300, _turn(two_ray_null(-15, 3, FS_11A, 21), np.pi / 4), 0, None, None),   # no noise: on bin -15 |Y|^2 >> 8 == 1
                                                                                # and |Re Y| = 21, so 1600 Re Y wraps in the int16 truncation
        ("sco+40ppm", long_len, ([0], [1]), 40, None, 35),                  # sample drift over the frame: 2500 B at 6 Mbps, 40 ppm: 5.4 samples
        ("sco-40ppm", long_len, ([0], [1]), -40, None, 35),
        ("sco+100ppm", long_len, ([0], [1]), 100, None, 35),
        ("sco-100ppm", long_len, ([0], [1]), -100, None, 35),
        ("sco+25ppm_cfo", long_len, ([0], [1]), 25, FC_11A, 35),            # one oscillator: 25 ppm at 5.2 GHz is -130 kHz
        ("exp150ns_sco-20ppm_cfo_snr22", long_len, exp_profile(150, FS_11A, 8), -20, FC_11A, 22),
    ]
    return S

@functools.lru_cache(maxsize=None)
def cases_11a(rate_kbps, fs_mhz=40):
    """802.11a at 40 Msps (or the same signals at 44 Msps): one frame per case at rate_kbps."""
    out = []
    for i, (name, L, (d, g), ppm, fc, snr) in enumerate(_spec_11a(rate_kbps)):
        td = synth.modulate(_psdu(L, 0xC4A00000 + 16 * rate_kbps + i)[None, :], rate_kbps)[0]
        y = multipath(td, d, g)
        ratio = (1.0 + ppm * 1e-6) * fs_mhz / 40.0
        y = resample(y, ratio)
        if fc is not None:
            y = y * np.exp(-2j * np.pi * ppm * 1e-6 * fc * np.arange(y.shape[-1]) / (fs_mhz * 1e6))
        out.append((name, quantise(y, 0.5, snr, seed=0xC4A0 + rate_kbps + i, lead=400 * fs_mhz // 40)))
    return out


# ---- 802.11n ------------------------------------------------------------------------------------------------------------------------
def _rand2x2(rng):
    return (rng.normal(size=(2, 2)) + 1j * rng.normal(size=(2, 2))) / np.sqrt(2)

def mimo_profile(seed, delays=(0, 2, 5, 9), decay=0.6):
    """(delays, 2x2 gains): an independent complex Gaussian matrix per tap, tap power decay ** k."""
    rng = np.random.default_rng(seed)
    return list(delays), [_rand2x2(rng) * decay ** (k / 2) for k in range(len(delays))]

def mimo_near_singular(seed, k, d=3, eps=0.03):
    """(delays, 2x2 gains) of two taps whose sum on 20 MHz subcarrier k is a rank-one matrix plus eps I: det H(k) is small but not 0."""
    rng = np.random.default_rng(seed)
    A = _rand2x2(rng); u = rng.normal(size=2) + 1j * rng.normal(size=2); v = rng.normal(size=2) + 1j * rng.normal(size=2)
    M = np.outer(u, v.conj()) / 2 + eps * np.eye(2)
    z = np.exp(-2j * np.pi * k * SUBCARRIER_HZ * d / FS_11A)
    return [0, d], [A, (M - A) / z]

def _spec_11n(mcs):
    S = [
        ("mimo4tap", 150, mimo_profile(1), 0, 30),
        ("mimo4tap_b", 150, mimo_profile(2, (0, 3, 7, 12)), 0, 30),
        ("near_singular+9", 150, mimo_near_singular(3, 9), 0, 35),
        ("near_singular-3", 150, mimo_near_singular(4, -3), 0, 35),
        ("faded_ant1", 150, ([0, 4], [np.array([[1.0, 0.4j], [0.04, 0.03j]]), np.array([[0.3, -0.2], [0.02j, 0.05]])]), 0, 30),
        ("sco+40ppm", 900, ([0], [np.array([[1.0, 0.3j], [-0.2, 0.9]])]), 40, 35),
        ("sco-40ppm", 900, ([0], [np.array([[1.0, 0.3j], [-0.2, 0.9]])]), -40, 35),
        ("mimo_sco+40ppm_snr25", 900, mimo_profile(5), 40, 25),
    ]
    return S

@functools.lru_cache(maxsize=None)
def cases_11n(mcs):
    """802.11n 2x2 at 40 Msps: one frame per case at mcs; each capture a pair (antenna 0, antenna 1)."""
    out = []
    for i, (name, L, (d, g), ppm, snr) in enumerate(_spec_11n(mcs)):
        tx = synth.modulate_11n(_psdu(L, 0xC4B00000 + 16 * mcs + i)[None, :], mcs)[0]
        y = resample(multipath(tx, d, g), 1.0 + ppm * 1e-6)
        q = quantise(y, 0.5, snr, seed=0xC4B0 + mcs + i)
        out.append((name, (q[0], q[1])))
    return out


# ---- 802.11b ------------------------------------------------------------------------------------------------------------------------
FS_11B = 44e6

def _spec_11b(rate):
    long_len = 1500 if rate in (1000, 11000) else 400
    S = [
        ("two_tap", 200, _norm([0, 4], [1, 0.3j]), 0, None, 30),                # 91 ns
        ("three_tap", 200, _norm([0, 3, 9], [1, -0.25, 0.15j]), 0, None, 30),    # 205 ns
        ("five_tap_exp", 200, exp_profile(60, FS_11B, 7, max_taps=6), 0, None, 30),
        ("preecho", 200, _norm([0, 5], [0.5, 1.0]), 0, None, 30),
        ("sco+40ppm", long_len, ([0], [1]), 40, None, 30),                     # 1500 B at 1 Mbps, 40 ppm: 0.49 us = 5.4 chips of drift
        ("sco-40ppm", long_len, ([0], [1]), -40, None, 30),
        ("sco+40ppm_cfo", long_len, ([0], [1]), 40, FC_11B, 30),               # one oscillator: 40 ppm at 2.4 GHz is -96 kHz
        ("three_tap_sco-40ppm_cfo_snr20", long_len, _norm([0, 3, 9], [1, 0.25j, -0.15]), -40, FC_11B, 20),
    ]
    return S

@functools.lru_cache(maxsize=None)
def cases_11b(rate_kbps):
    """802.11b at 44 Msps: one long-preamble frame per case at rate_kbps."""
    out = []
    for i, (name, L, (d, g), ppm, fc, snr) in enumerate(_spec_11b(rate_kbps)):
        td = synth.modulate_11b(_psdu(L, 0xC4C00000 + rate_kbps + i), rate_kbps)
        y = sco(multipath(td, d, g), ppm, FS_11B, fc)
        out.append((name, quantise(y, 0.3, snr, seed=0xC4C0 + rate_kbps + i)))
    return out


# ---- continuous captures ------------------------------------------------------------------------------------------------------------
def _pick(cases, names):
    c = dict(cases)
    return [c[n] for n in names]

def stream_11a():
    """One capture: frames of four rates through different channels, back to back (each case keeps its own noisy lead and trail)."""
    parts = _pick(cases_11a(6000), ["exp150ns", "null_pilot+7"]) + _pick(cases_11a(12000), ["echo1.2us", "preecho"]) \
        + _pick(cases_11a(24000), ["nearnull40dB", "exp50ns"]) + _pick(cases_11a(54000), ["sco-100ppm", "null_dc-1", "echo1.0us"])
    return np.concatenate(parts)

def stream_11n(mcs):
    parts = _pick(cases_11n(mcs), ["mimo4tap", "near_singular+9", "faded_ant1", "sco-40ppm", "mimo4tap_b"])
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])

def stream_11b():
    parts = _pick(cases_11b(2000), ["three_tap", "preecho"]) + _pick(cases_11b(5500), ["three_tap", "sco-40ppm"]) \
        + _pick(cases_11b(11000), ["sco+40ppm", "two_tap"])
    return np.concatenate(parts)

RATES_11A = (6000, 12000, 24000, 54000)
RATES_11B = (1000, 2000, 5500, 11000)
MCS_11N = ((8, 11), (10, 11), (14, 15))                # (mcs, ht_mcs_limit): MCS 14 needs the 16-/64-QAM branches of the HT-SIG parser


def _run_oracle():
    """Every case through the oracle entry points the device tests compare with; after each case its batch status."""
    import oracle_py
    say = lambda s: (print(s), sys.stdout.flush())
    for rate in RATES_11A:
        for (name, x), (_, x44) in zip(cases_11a(rate), cases_11a(rate, 44)):
            say(f"11a {rate} {name}")
            r, _ = oracle_py.rx11a_batch(x, [0], [len(x)], out_stride=4096)
            oracle_py.rx11a_batch(np.repeat(x[::2], 2, axis=0), [0], [len(x[::2]) * 2], out_stride=4096)
            oracle_py.rx11a_run(oracle_py.resample_44_40(x44), max_frames=1, out_stride=4096)
            oracle_py.rx11a_taps(x, max_sym=1400)
            say(f"status {int(r['status'][0]):#x}")
    say("11a stream"); oracle_py.rx11a_run(stream_11a(), max_frames=16, out_stride=4096)
    for rate in RATES_11B:
        for name, x in cases_11b(rate):
            say(f"11b {rate} {name}")
            r, _ = oracle_py.rx11b_batch(x, [0], [len(x)])
            say(f"status {int(r['status'][0]):#x}")
    say("11b stream"); oracle_py.rx11b_run(stream_11b(), max_frames=16)
    for mcs, limit in MCS_11N:
        oracle_py.set_ht_mcs_limit(limit)
        for name, (x, y) in cases_11n(mcs):
            say(f"11n {mcs} {name}")
            r, _ = oracle_py.rx11n_batch(x, y, [0], [len(x)])
            oracle_py.rx11n_taps(x, y)
            say(f"status {int(r['status'][0]):#x}")
        say(f"11n {mcs} stream"); oracle_py.rx11n_run(*stream_11n(mcs), max_frames=16)
    oracle_py.set_ht_mcs_limit(11)
    say("done")

if __name__ == "__main__":
    if len(sys.argv) > 1:
        import oracle_py
        oracle_py.use_library(sys.argv[1])
    _run_oracle()
