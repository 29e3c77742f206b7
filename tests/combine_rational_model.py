"""The numpy model of sb200_combine_rational (test input only): the arithmetic of include/sora_b200.h restated in 64-bit integers.  The filter
is the rational channelizer's (rational_model._fir_stuffed: zero-stuffed by U, int32 accumulator with its wrap emulated, decimated by D),
the rotation is sb200_combine's (combine_model.rotate_up, by the phase of the absolute output index), then the Q12 gain, the sum over the
channels and, with accumulate, the caller's samples, under one saturation.  combine_rational_window computes a window of outputs from the
inputs it reads only, so that windows of a long device capture can be checked without the whole of it."""
import numpy as np
from combine_model import rotate_up
from rational_model import _fir_stuffed
from wideband_inputs import _wrap32

def _sum(vs, gains, acc):
    """y = sat16(a + sum_k ((v_k * gain_k + 2^11) >> 12)), int32 terms and sum; a = acc or 0."""
    s = sum(_wrap32(v.astype(np.int64) * int(g) + (1 << 11)) >> 12 for v, g in zip(vs, gains))
    if acc is not None: s = s + np.asarray(acc, np.int64).reshape(-1, 2)
    return np.clip(_wrap32(s), -32768, 32767).astype(np.int16)

def combine_rational_window(rows, channels, U, D, taps, n0, n1, acc=None):
    """Outputs n0 .. n1 of combine_rational(rows, ...), from the input samples they read only; acc: the caller's samples n0 .. n1 (int16
    [n1 - n0, 2]) when accumulating."""
    c = len(taps) // 2; vs = []
    for x, (inc, ph, _) in zip(rows, channels):
        x = np.asarray(x, np.int64).reshape(-1, 2)
        a = max(-(-(D * n0 - c) // U), 0); b = min((D * (n1 - 1) + c) // U + 1, len(x))   # inputs i with D n0 - c <= U i <= D (n1 - 1) + c
        v = x[a:b] if b > a else np.zeros((0, 2), np.int64)
        vs.append(rotate_up(_fir_stuffed(v, U, D, taps, n0, n1, a), inc, ph, n0))
    return _sum(vs, [g for _, _, g in channels], acc)

def combine_rational(rows, channels, U, D, taps, n_out=None, acc=None):
    """The model of sb200_combine_rational: int16 [K, n_in, 2], [(phase_inc, phase0, gain)] -> int16 [n_out, 2] (n_out None:
    ceil(U n_in / D)); acc: the output buffer's samples before the call (int16 [n_out, 2]) for accumulate = 1, None for 0."""
    n_in = np.asarray(rows[0]).reshape(-1, 2).shape[0]
    n_out = -(-U * n_in // D) if n_out is None else n_out
    return combine_rational_window(rows, channels, U, D, taps, 0, n_out, acc)
