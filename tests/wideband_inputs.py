"""Wideband captures holding several channels, and the numpy model of sb200_channelize (test input only).

The model restates the arithmetic of include/sora_b200.h in 64-bit integers: the NCO table from its closed form, the Q14 rotation of every
sample by the phase of its absolute index, and the FIR over the rotated samples with the int32 accumulator's wrap emulated.

The captures (capture_11a, capture_11b, capture_11n) are rendered from the float modulators of synth: every channel's frames are made at
the channel rate (40 or 44 Msps), resampled by 4 with the band-limited resampler of channel_inputs, shifted to the channel's centre,
summed in float and quantised to int16 once.  Each returns the capture, the channel centres (Hz), and per channel the PSDUs (FCS
included) it carries, in order.
"""
import numpy as np
from sora_b200 import synth
import channel_inputs as CI

# ---- the model ----------------------------------------------------------------------------------------------------------------------
_I = np.arange(4096)
NCO = np.stack([np.rint(16384 * np.cos(2 * np.pi * _I / 4096)), np.rint(16384 * np.sin(2 * np.pi * _I / 4096))], 1).astype(np.int64)   # (C, S), Q14

def phase_inc(f_hz, fs_hz):
    return int(round(f_hz / fs_hz * 2 ** 32)) % 2 ** 32

def _wrap32(v):
    return ((v + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)

def rotate(iq, inc, phase0):
    """v(n) = sat16((x(n) e^{-j theta(n)} + 2^13) >> 14), theta from NCO[(phase0 + n inc) mod 2^32 >> 20]; int16 [n, 2] -> int64 [n, 2]."""
    x = np.asarray(iq, np.int64).reshape(-1, 2)
    n = np.arange(len(x), dtype=np.uint64)
    phi = (np.uint64(phase0 % 2 ** 32) + n * np.uint64(inc % 2 ** 32)) & np.uint64(0xFFFFFFFF)
    cs = NCO[(phi >> np.uint64(20)).astype(np.int64)]
    C, S = cs[:, 0], cs[:, 1]
    re = (x[:, 0] * C + x[:, 1] * S + (1 << 13)) >> 14
    im = (x[:, 1] * C - x[:, 0] * S + (1 << 13)) >> 14
    return np.clip(np.stack([re, im], 1), -32768, 32767)

def fir(v, decim, taps):
    """y[m] = sat16((sum_k taps[k] v(D m + k - c) + 2^14) >> 15), v = 0 outside, int32 accumulator; m = 0 .. ceil(n / D)."""
    taps = np.asarray(taps, np.int64); c = len(taps) // 2; n = len(v); m = -(-n // decim)
    x = np.zeros((decim * m + 2 * c + 1, 2), np.int64); x[c:c + n] = v
    acc = np.zeros((m, 2), np.int64)
    for k, t in enumerate(taps):
        if t: acc += t * x[k: k + decim * m: decim][:m]
    return np.clip(_wrap32(acc + (1 << 14)) >> 15, -32768, 32767).astype(np.int16)

def channelize(iq, channels, decim, taps):
    """The model of sb200_channelize: int16 [n, 2], [(phase_inc, phase0)] -> int16 [K, ceil(n / decim), 2]."""
    return np.stack([fir(rotate(iq, a, b), decim, taps) for a, b in channels])

def channelize_window(iq, channels, decim, taps, m0, m1):
    """Outputs m0 .. m1 of channelize(iq, channels, decim, taps), computed from the input samples they read only (the phase is a closed
    form of the absolute index), so that windows of a long capture can be checked without the whole of it."""
    x = np.asarray(iq).reshape(-1, 2); taps = np.asarray(taps, np.int64); c = len(taps) // 2; n = len(x); M = m1 - m0
    lo = decim * m0 - c; hi = decim * (m1 - 1) + c + 1; a, b = max(lo, 0), min(hi, n)
    out = []
    for inc, ph in channels:
        seg = np.zeros((hi - lo, 2), np.int64)
        if b > a: seg[a - lo:b - lo] = rotate(x[a:b], inc, (ph + a * inc) % 2 ** 32)
        acc = np.zeros((M, 2), np.int64)
        for k, t in enumerate(taps):
            if t: acc += t * seg[k: k + decim * M: decim][:M]
        out.append(np.clip(_wrap32(acc + (1 << 14)) >> 15, -32768, 32767).astype(np.int16))
    return np.stack(out)


# ---- taps ---------------------------------------------------------------------------------------------------------------------------
def lowpass(ntaps, cutoff, beta=8.0, gain=1.0):
    """Kaiser-windowed sinc low-pass of ntaps (odd) taps, cutoff as a fraction of the sample rate, DC gain `gain`, in Q15 (int16)."""
    k = np.arange(ntaps) - ntaps // 2
    h = 2 * cutoff * np.sinc(2 * cutoff * k) * np.kaiser(ntaps, beta)
    h *= gain / h.sum()
    return np.clip(np.rint(h * 32768), -32768, 32767).astype(np.int16)


# ---- captures -----------------------------------------------------------------------------------------------------------------------
def _psdu(n, seed):
    r = np.random.RandomState(seed & 0xFFFFFFFF)
    return synth.psdu_with_fcs(r.randint(0, 256, n - 4).astype(np.uint8))

def _render(parts, fs, n_total, up=4):
    """Sum of channels: parts = [(f_c Hz, [(start at the channel rate, waveform [..., n])], amplitude)] -> complex [..., n_total] at fs."""
    y = None
    for fc, frames, amp in parts:
        for start, w in frames:
            z = CI.resample(w, float(up)) * amp
            if y is None: y = np.zeros(z.shape[:-1] + (n_total,), np.complex128)
            s = up * start; z = z[..., :n_total - s]
            y[..., s:s + z.shape[-1]] += z * np.exp(2j * np.pi * fc / fs * np.arange(s, s + z.shape[-1]))
    return y

def _quantise(y, sigma, seed):
    rng = np.random.default_rng(seed)
    z = y + rng.normal(0, sigma, y.shape) + 1j * rng.normal(0, sigma, y.shape)
    return np.clip(np.round(np.stack([z.real, z.imag], -1)), -32768, 32767).astype(np.int16)

FS_11A_WIDE, CH_11A = 160e6, (-60e6, -20e6, 20e6, 60e6)
RATES_11A_WIDE = ((6000, 24000, 54000), (12000, 36000, 6000), (54000, 6000, 24000), (24000, 48000, 12000))

def capture_11a(strong=2):
    """160 Msps, four 802.11a channels at -60 / -20 / +20 / +60 MHz, three frames each at different rates, starting at different times;
    channel `strong` 20 dB above the others (it is the neighbour of channels 1 and 3).  -> (int16 [n, 2], centres, [[psdu, ...] per channel])."""
    parts, psdus, end = [], [], 0
    for ci, (fc, rates) in enumerate(zip(CH_11A, RATES_11A_WIDE)):
        t, fr, ps = 600 + 900 * ci, [], []
        for j, rate in enumerate(rates):
            p = _psdu(120 + 60 * j + 20 * ci, 0x3D1A0000 + 16 * ci + j)
            w = synth.modulate(p[None, :], rate, scramble_seeds=[1 + 7 * ci + j])[0]
            fr.append((t, w)); ps.append(p); t += w.shape[-1] + 1500
        parts.append((fc, fr, 220.0 if ci == strong else 22.0)); psdus.append(ps); end = max(end, t)
    n = 4 * (end + 600); n += (-n) % (4 * 28)
    return _quantise(_render(parts, FS_11A_WIDE, n), 10.0, 0x3D1A), CH_11A, psdus

FS_11B_WIDE, CH_11B = 176e6, (-25e6, 0.0, 25e6)

def capture_11b():
    """176 Msps, three 802.11b channels at -25 / 0 / +25 MHz (channels 1 / 6 / 11 of 2.4 GHz), two long-preamble frames each."""
    parts, psdus, end = [], [], 0
    rates = ((2000, 11000), (5500, 1000), (11000, 2000))
    for ci, fc in enumerate(CH_11B):
        t, fr, ps = 800 + 1200 * ci, [], []
        for j, rate in enumerate(rates[ci]):
            p = _psdu(60 + 40 * j + 10 * ci, 0x3D1B0000 + 16 * ci + j)
            w = synth.modulate_11b(p, rate)
            fr.append((t, w)); ps.append(p); t += w.shape[-1] + 2000
        parts.append((fc, fr, 0.3 * 256.0)); psdus.append(ps); end = max(end, t)
    n = 4 * (end + 800); n += (-n) % (4 * 28)
    return _quantise(_render(parts, FS_11B_WIDE, n), 40.0, 0x3D1B), CH_11B, psdus

CH_11N = (-20e6, 20e6)

def capture_11n(mcs=9):
    """Two antennas at 160 Msps, two 802.11n 2x2 channels at -20 / +20 MHz, two frames each through a fixed 2x2 channel per channel.
    -> ((int16 [n, 2], int16 [n, 2]), centres, psdus)."""
    parts, psdus, end = [], [], 0
    H = (np.array([[1.0, 0.3j], [-0.2, 0.9]]), np.array([[0.8, -0.4], [0.3j, 1.0]]))
    for ci, fc in enumerate(CH_11N):
        t, fr, ps = 700 + 1100 * ci, [], []
        for j in range(2):
            p = _psdu(100 + 50 * j + 30 * ci, 0x3D1C0000 + 16 * ci + j)
            w = H[ci] @ synth.modulate_11n(p[None, :], mcs, scramble_seeds=[3 + 5 * ci + j])[0]
            fr.append((t, w)); ps.append(p); t += w.shape[-1] + 1500
        parts.append((fc, fr, 0.5 * 256.0)); psdus.append(ps); end = max(end, t)
    n = 4 * (end + 600); n += (-n) % (4 * 28)
    q = _quantise(_render(parts, FS_11A_WIDE, n), 40.0, 0x3D1C)
    return (q[0], q[1]), CH_11N, psdus
