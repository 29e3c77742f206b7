"""The numpy model of sb200_channelize_rational and a 2.4 GHz capture for it (test input only).

The model restates the arithmetic of include/sora_b200.h in 64-bit integers, in the style of the channelizer's model in wideband_inputs.py,
whose NCO rotation it reuses: the rotated input is zero-stuffed by U and goes through the FIR with the int32 accumulator's wrap emulated,
decimated by D.  channelize_rational_window computes a window of outputs from the inputs it reads only, so that windows of a long device
capture can be checked without the whole of it.  capture_24ghz renders 802.11b and OFDM channels into one capture the way
wideband_inputs' captures are rendered.
"""
import numpy as np
from sora_b200 import synth
import channel_inputs as CI
from wideband_inputs import _psdu, _quantise, _wrap32, rotate

# ---- the rational-rate channelizer (sb200_channelize_rational) ---------------------------------------------------------------------
def _fir_stuffed(v, interp, decim, taps, m0, m1, i0):
    """Outputs m0 .. m1 of y[m] = sat16((sum_k taps[k] z(D m + k - c) + 2^14) >> 15), z the rotated samples v (input i0 + j at v[j], zero
    elsewhere) stuffed with interp - 1 zeros; int32 accumulator."""
    taps = np.asarray(taps, np.int64); c = len(taps) // 2; M = m1 - m0
    lo = decim * m0 - c; hi = decim * (m1 - 1) + c + 1                              # zero-stuffed indices read
    z = np.zeros((hi - lo, 2), np.int64)
    i = i0 + np.arange(len(v)); at = interp * i - lo; keep = (at >= 0) & (at < hi - lo)
    z[at[keep]] = v[keep]
    acc = np.zeros((M, 2), np.int64)
    for k, t in enumerate(taps):
        if t: acc += t * z[k: k + decim * M: decim][:M]
    return np.clip(_wrap32(acc + (1 << 14)) >> 15, -32768, 32767).astype(np.int16)

def channelize_rational(iq, channels, interp, decim, taps):
    """The model of sb200_channelize_rational: int16 [n, 2], [(phase_inc, phase0)] -> int16 [K, ceil(interp n / decim), 2]."""
    x = np.asarray(iq).reshape(-1, 2); n_out = -(-interp * len(x) // decim)
    return np.stack([_fir_stuffed(rotate(x, a, b), interp, decim, taps, 0, n_out, 0) for a, b in channels])

def channelize_rational_window(iq, channels, interp, decim, taps, m0, m1):
    """Outputs m0 .. m1 of channelize_rational, computed from the input samples they read only."""
    x = np.asarray(iq).reshape(-1, 2); c = len(taps) // 2; n = len(x)
    a = max(-(-(decim * m0 - c) // interp), 0); b = min((decim * (m1 - 1) + c) // interp + 1, n)
    out = []
    for inc, ph in channels:
        v = rotate(x[a:b], inc, (ph + a * inc) % 2 ** 32) if b > a else np.zeros((0, 2), np.int64)
        out.append(_fir_stuffed(v, interp, decim, taps, m0, m1, a))
    return np.stack(out)

# ---- a 2.4 GHz capture: 802.11b and OFDM on channels 1, 6 and 11 --------------------------------------------------------------------
CH_24 = (-25e6, 0.0, 25e6)                             # channels 1, 6, 11 around channel 6's centre
KIND_24 = ("11b", "ofdm", "11b")

def capture_24ghz(fs):
    """One capture at fs (160 or 176 Msps) of the 2.4 GHz band: 802.11b at -25 and +25 MHz (44 Msps, long preamble) and 802.11a OFDM frames
    at 0 Hz (40 Msps), several frames per channel at several rates, starting at staggered times.  Every frame starts on a 4 MHz grid of the
    capture (fs / 4 MHz = 40 or 44 samples), whole at 40 and at 44 Msps; each waveform is resampled from its own rate to fs by
    channel_inputs.resample.  -> (int16 [n, 2], centres, kinds, [[psdu, ...] per channel])."""
    grid = int(round(fs / 4e6))
    frames = ([(2000, 70), (11000, 40)], [(24000, 150), (6000, 90), (54000, 200)], [(5500, 60), (2000, 90), (11000, 50)])    # (rate kbps, bytes)
    pieces, psdus, end = [], [], 0
    for ci, (fc, kind) in enumerate(zip(CH_24, KIND_24)):
        t = (300 + 700 * ci) * grid; ps = []
        for j, (rate, nb) in enumerate(frames[ci]):
            p = _psdu(nb + 10 * j, 0x3D240000 + 16 * ci + j)
            if kind == "11b":
                w, r, amp = synth.modulate_11b(p, rate), 44e6, 0.3 * 256.0
            else:
                w, r, amp = synth.modulate(p[None, :], rate, scramble_seeds=[5 + 3 * j])[0], 40e6, 150.0
            z = CI.resample(w, fs / r) * amp
            pieces.append((fc, t, z)); ps.append(p)
            t += -(-(z.shape[-1] + 60 * grid) // grid) * grid
        psdus.append(ps); end = max(end, t)
    n = end + 400 * grid; n += (-n) % (4 * 28 * grid)
    y = np.zeros(n, np.complex128)
    for fc, s, z in pieces:
        y[s:s + len(z)] += z * np.exp(2j * np.pi * fc / fs * np.arange(s, s + len(z)))
    return _quantise(y, 20.0, 0x3D24 + int(fs // 1e6)), CH_24, KIND_24, psdus
