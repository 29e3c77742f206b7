"""The numpy model of sb200_channelize_arbitrary and a 2.4 GHz capture at a rate off the 4 MHz grid (test input only).

The model restates the arithmetic of include/sora_b200.h in 64-bit integers, reusing the channelizer model's NCO rotation: output m stands
at input time t_m = tau0 + m step (Q32.32), t' = t_m + 2^23 picks input i = t' >> 32 and row p = (t' >> 24) & 255 of the table, and the
row's taps weigh the rotated inputs i - c .. i - c + ntaps - 1.  channelize_arbitrary_window computes outputs m0 .. m1 from only the
inputs they read, in slices, so that long captures and windows of device rows can be checked without the whole of them.
capture_24ghz_grid renders the channels of rational_model.capture_24ghz at any rate on a grid of start times given in samples.
"""
import numpy as np
from sora_b200 import synth
import channel_inputs as CI
import rational_model as R
from wideband_inputs import _psdu, _quantise, rotate

SLICE = 1 << 15                                        # outputs per slice of the model

def _times(tau0, step, m0, m1):
    t = np.uint64(tau0) + np.arange(m0, m1, dtype=np.uint64) * np.uint64(step) + np.uint64(1 << 23)
    return (t >> np.uint64(32)).astype(np.int64), ((t >> np.uint64(24)) & np.uint64(255)).astype(np.int64)

def _slice(x, ch, tau0, step, H, m0, m1):
    """Outputs m0 .. m1 of one channel from the inputs they read."""
    ntaps = H.shape[1]; c = (ntaps - 1) // 2; n = len(x)
    i, p = _times(tau0, step, m0, m1)
    lo, hi = int(i[0]) - c, int(i[-1]) - c + ntaps                  # inputs read
    v = np.zeros((hi - lo, 2), np.int64)
    a, b = max(lo, 0), min(hi, n)
    if b > a: v[a - lo:b - lo] = rotate(x[a:b], ch[0], (ch[1] + a * ch[0]) % 2 ** 32)
    acc = np.full((m1 - m0, 2), 1 << 13, np.int64)
    for k in range(ntaps):
        acc += H[p, k][:, None] * v[i - c + k - lo]
    return np.clip(acc >> 14, -32768, 32767).astype(np.int16)

def channelize_arbitrary_window(iq, channels, tau0, step, taps, m0, m1):
    """Outputs m0 .. m1 of sb200_channelize_arbitrary: int16 [n, 2], [(phase_inc, phase0)], taps [256, ntaps] -> int16 [K, m1 - m0, 2]."""
    x = np.asarray(iq).reshape(-1, 2); H = np.asarray(taps, np.int64)
    out = np.zeros((len(channels), m1 - m0, 2), np.int16)
    for k, ch in enumerate(channels):
        for s in range(m0, m1, SLICE):
            e = min(s + SLICE, m1); out[k, s - m0:e - m0] = _slice(x, ch, tau0, step, H, s, e)
    return out

def channelize_arbitrary(iq, channels, tau0, step, taps, n_out):
    """The model of sb200_channelize_arbitrary: -> int16 [K, n_out, 2]."""
    return channelize_arbitrary_window(iq, channels, tau0, step, taps, 0, n_out)

def n_inside(n_in, tau0, step):
    """Outputs whose time lies inside the input (Engine.channelize_arbitrary's default n_out)."""
    return max(0, -(-((n_in << 32) - tau0) // step))

# ---- a 2.4 GHz capture at any rate ---------------------------------------------------------------------------------------------------
def capture_24ghz_grid(fs, grid):
    """rational_model.capture_24ghz's frames and channels (802.11b at -25 and +25 MHz, OFDM at 0 Hz) rendered at fs, every frame starting
    on a multiple of `grid` samples of the capture.  At 122.88 Msps a grid of 768 samples (6.25 us) is 250 samples at 40 Msps and 275 at
    44 Msps, so every frame starts on a whole sample at both rates.  -> (int16 [n, 2], centres, kinds, [[psdu, ...] per channel])."""
    frames = ([(2000, 70), (11000, 40)], [(24000, 150), (6000, 90), (54000, 200)], [(5500, 60), (2000, 90), (11000, 50)])    # (rate kbps, bytes)
    step = -(-int(round(12.5e-6 * fs)) // grid) * grid                    # at least 12.5 us between frames
    pieces, psdus, end = [], [], 0
    for ci, (fc, kind) in enumerate(zip(R.CH_24, R.KIND_24)):
        t = (1 + 2 * ci) * step; ps = []
        for j, (rate, nb) in enumerate(frames[ci]):
            p = _psdu(nb + 10 * j, 0x3D240000 + 16 * ci + j)
            if kind == "11b":
                w, r, amp = synth.modulate_11b(p, rate), 44e6, 0.3 * 256.0
            else:
                w, r, amp = synth.modulate(p[None, :], rate, scramble_seeds=[5 + 3 * j])[0], 40e6, 150.0
            z = CI.resample(w, fs / r) * amp
            pieces.append((fc, t, z)); ps.append(p)
            t += -(-(z.shape[-1] + step) // grid) * grid
        psdus.append(ps); end = max(end, t)
    n = end + 4 * step; n += (-n) % (4 * grid)
    y = np.zeros(n, np.complex128)
    for fc, s, z in pieces:
        y[s:s + len(z)] += z * np.exp(2j * np.pi * fc / fs * np.arange(s, s + len(z)))
    return _quantise(y, 20.0, 0x3D24 + int(fs // 1e6)), R.CH_24, R.KIND_24, psdus
