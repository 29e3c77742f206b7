"""The numpy model of sb200_combine (test input only): the arithmetic of include/sora_b200.h restated in 64-bit integers, in the style of
the channelizer's model in wideband_inputs.py, whose Q14 NCO table it shares.  The zero-stuffed row goes through the FIR with the int32
accumulator's wrap emulated, then the Q14 rotation with the opposite sign by the phase of the absolute output index, the Q12 gain and the
saturating sum over the channels.  combine_window computes a window of outputs from the inputs it reads only, so that windows of a long
device capture can be checked without the whole of it."""
import numpy as np
from wideband_inputs import NCO, _wrap32

def rotate_up(u, inc, phase0, n0=0):
    """v(n) = sat16((u(n) e^{+j theta(n)} + 2^13) >> 14), theta from NCO[(phase0 + n inc) mod 2^32 >> 20], n = n0 + index; int64 [n, 2] -> int64 [n, 2]."""
    u = np.asarray(u, np.int64).reshape(-1, 2)
    n = np.arange(n0, n0 + len(u), dtype=np.uint64)
    phi = (np.uint64(phase0 % 2 ** 32) + n * np.uint64(inc % 2 ** 32)) & np.uint64(0xFFFFFFFF)
    cs = NCO[(phi >> np.uint64(20)).astype(np.int64)]
    C, S = cs[:, 0], cs[:, 1]
    re = (u[:, 0] * C - u[:, 1] * S + (1 << 13)) >> 14
    im = (u[:, 1] * C + u[:, 0] * S + (1 << 13)) >> 14
    return np.clip(np.stack([re, im], 1), -32768, 32767)

def interpolate(x, interp, taps):
    """u(n) = sat16((sum_j taps[j] z(n + j - c) + 2^14) >> 15), z = x zero-stuffed by U, int32 accumulator; n = 0 .. U n_in."""
    x = np.asarray(x, np.int64).reshape(-1, 2); taps = np.asarray(taps, np.int64); c = len(taps) // 2; N = interp * len(x)
    z = np.zeros((N + 2 * c, 2), np.int64); z[c:c + N:interp] = x                  # z[n + c] = z(n)
    acc = np.zeros((N, 2), np.int64)
    for j, t in enumerate(taps):
        if t: acc += t * z[j:j + N]
    return np.clip(_wrap32(acc + (1 << 14)) >> 15, -32768, 32767)

def _scale_sum(vs, gains):
    """y = sat16(sum_k ((v_k * gain_k + 2^11) >> 12)), int32 terms and sum."""
    acc = sum(_wrap32(v * int(g) + (1 << 11)) >> 12 for v, g in zip(vs, gains))
    return np.clip(_wrap32(acc), -32768, 32767).astype(np.int16)

def combine(rows, channels, interp, taps):
    """The model of sb200_combine: int16 [K, n_in, 2], [(phase_inc, phase0, gain)] -> int16 [interp * n_in, 2]."""
    return _scale_sum([rotate_up(interpolate(x, interp, taps), a, b) for x, (a, b, _) in zip(rows, channels)], [g for _, _, g in channels])

def combine_window(rows, channels, interp, taps, n0, n1):
    """Outputs n0 .. n1 of combine(rows, channels, interp, taps), computed from the input samples they read only (the phase is a closed
    form of the absolute index), so that windows of a long capture can be checked without the whole of it."""
    taps = np.asarray(taps, np.int64); c = len(taps) // 2; U = interp; N = n1 - n0
    vs = []
    for x, (inc, ph, _) in zip(rows, channels):
        x = np.asarray(x).reshape(-1, 2)
        i0 = max(-(-(n0 - c) // U), 0); i1 = min((n1 - 1 + c) // U + 1, len(x))   # inputs i with n0 - c <= U i <= n1 - 1 + c
        z = np.zeros((N + 2 * c, 2), np.int64)                                     # z[q] = z(n0 - c + q)
        if i1 > i0: z[U * i0 - (n0 - c):U * (i1 - 1) - (n0 - c) + 1:U] = x[i0:i1]
        acc = np.zeros((N, 2), np.int64)
        for j, t in enumerate(taps):
            if t: acc += t * z[j:j + N]
        vs.append(rotate_up(np.clip(_wrap32(acc + (1 << 14)) >> 15, -32768, 32767), inc, ph, n0))
    return _scale_sum(vs, [g for _, _, g in channels])
