"""The numpy model of sb200_channelize_bank (include/sora_b200.h), in 64-bit integers, and a capture for its odd-stacked grid (test input only).

direct() restates the header's arithmetic as written: every tap's sample rotated by the channel's NCO entry, one rounding.  window() is
the polyphase form the kernel computes (bank_kernels.cuh): branch sums with the odd-stacking sign, then an M-point DFT over the Q14
table; integer arithmetic is exact, so the two agree bit for bit.  window() reads only the input samples its outputs meet, so long
captures are checked a window at a time, as wideband_inputs.channelize_window does for sb200_channelize.
"""
import numpy as np
import wideband_inputs as W
from wideband_inputs import NCO
from sora_b200 import synth

def _sat16(acc):
    return np.clip((acc + (1 << 28)) >> 29, -32768, 32767).astype(np.int16)

def direct(iq, M, D, odd, taps):
    """The stated arithmetic, tap by tap: int16 [n, 2] -> int16 [M, ceil(n / D), 2].  For small sizes."""
    x = np.asarray(iq, np.int64).reshape(-1, 2); n = len(x); taps = np.asarray(taps, np.int64); c = len(taps) // 2
    nm = -(-n // D); m = np.arange(nm)
    acc = np.zeros((M, nm, 2), np.int64)
    for k in range(M):
        for j, t in enumerate(taps):
            nj = D * m + j - c; ok = (nj >= 0) & (nj < n); v = x[np.where(ok, nj, 0)] * ok[:, None]
            C, S = NCO[((2 * k + odd) * nj * (2048 // M)) % 4096].T
            acc[k, :, 0] += t * (v[:, 0] * C + v[:, 1] * S); acc[k, :, 1] += t * (v[:, 1] * C - v[:, 0] * S)
    return _sat16(acc)

def window(iq, M, D, odd, taps, m0, m1):
    """Outputs m0 .. m1 of every channel by the polyphase form, from the input samples they read only: int16 [M, m1 - m0, 2]."""
    x = np.asarray(iq).reshape(-1, 2); n = len(x); taps = np.asarray(taps, np.int64); c = len(taps) // 2; nm = m1 - m0
    lo = D * m0 - c; hi = D * (m1 - 1) + c + 1; a, b = max(lo, 0), min(hi, n)
    seg = np.zeros((hi - lo, 2), np.int64)
    if b > a: seg[a - lo:b - lo] = x[a:b]
    seg *= np.where(odd * (((lo + np.arange(hi - lo)) // M) % 2) == 1, -1, 1)[:, None]     # sigma(n) = (-1)^(o floor(n / M))
    s = np.zeros((nm, M, 2), np.int64); rows = np.arange(nm)
    for j, t in enumerate(taps):                                   # branch sums s_p[m], p = n_j mod M
        if t: s[rows, (D * (m0 + rows) + j - c) % M] += t * seg[j: j + D * nm: D][:nm]
    assert np.abs(s).max(initial=0) < 2 ** 31
    p, k = np.arange(M)[:, None], np.arange(M)[None, :]
    T = NCO[(((2 * k + odd) * p) % (2 * M)) * (2048 // M)]          # [p, k, (C, S)]
    C, S = T[..., 0], T[..., 1]
    yr = s[..., 0] @ C + s[..., 1] @ S; yi = s[..., 1] @ C - s[..., 0] @ S
    return _sat16(np.stack([yr.T, yi.T], -1))

def bank(iq, M, D, odd, taps):
    """The whole capture: int16 [n, 2] -> int16 [M, ceil(n / D), 2]."""
    n = len(np.asarray(iq).reshape(-1, 2))
    return window(iq, M, D, odd, taps, 0, -(-n // D))

def phase_incs(M, odd):
    """sb200_channelize's channels (phase_inc, phase0) that the bank's channels are: phase_inc = (2k + o) 2^31 / M."""
    return [(((2 * k + odd) * 2 ** 31 // M) % 2 ** 32, 0) for k in range(M)]


# ---- a capture for the odd-stacked grid -----------------------------------------------------------------------------------------------
CH_11A_OCTET = (-70e6, -50e6, -30e6, -10e6, 10e6, 30e6, 50e6, 70e6)
TAPS_BANK = W.lowpass(255, 10e6 / 160e6)               # -6 dB at 10 MHz of 160 Msps: passes 8.4 MHz, stops from 11.6 MHz

def capture_11a_octet(strong=5):
    """160 Msps, eight adjacent 802.11a channels at +-10 / +-30 / +-50 / +-70 MHz (the odd-stacked grid of M = 8), one frame each at
    different rates and start times; channel `strong` (in CH_11A_OCTET order) 10 dB above its neighbours.
    -> (int16 [n, 2], centres, [[psdu] per channel])."""
    rates = (6000, 12000, 24000, 54000, 36000, 18000, 48000, 9000)
    parts, psdus, end = [], [], 0
    for ci, (fc, rate) in enumerate(zip(CH_11A_OCTET, rates)):
        t = 500 + 350 * ci
        p = W._psdu(100 + 15 * ci, 0x3D1D0000 + ci)
        w = synth.modulate(p[None, :], rate, scramble_seeds=[1 + 5 * ci])[0]
        parts.append((fc, [(t, w)], 70.0 if ci == strong else 22.0)); psdus.append([p]); end = max(end, t + w.shape[-1] + 500)
    n = 4 * end; n += (-n) % (4 * 28)
    return W._quantise(W._render(parts, W.FS_11A_WIDE, n), 10.0, 0x3D1D), CH_11A_OCTET, psdus

