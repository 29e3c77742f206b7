"""The numpy model of sb200_combine_arbitrary (test input only): the arithmetic of include/sora_b200.h restated in 64-bit integers from the
models it is built of.  The resampler is the arbitrary-rate channelizer's (arbitrary_model._slice with channel (0, 0), whose rotation is
the identity), the rotation is sb200_combine's (combine_model.rotate_up, by the phase of the absolute output index), and the Q12 gain, the
sum over the channels and, with accumulate, the caller's samples under one saturation are sb200_combine_rational's
(combine_rational_model._sum).  combine_arbitrary_window computes a window of outputs from the inputs it reads only, so that windows of a
long device capture can be checked without the whole of it."""
import numpy as np
import arbitrary_model as A
from combine_model import rotate_up
from combine_rational_model import _sum

def combine_arbitrary_window(rows, channels, tau0, step, taps, n0, n1, acc=None):
    """Outputs n0 .. n1 of combine_arbitrary(rows, ...): int16 [K, n_in, 2], [(phase_inc, phase0, gain)], taps int16 [256, ntaps]
    -> int16 [n1 - n0, 2]; acc: the caller's samples n0 .. n1 (int16 [n1 - n0, 2]) when accumulating."""
    H = np.asarray(taps, np.int64); vs = []
    for x, (inc, ph, _) in zip(rows, channels):
        x = np.asarray(x).reshape(-1, 2)
        u = [A._slice(x, (0, 0), tau0, step, H, s, min(s + A.SLICE, n1)) for s in range(n0, n1, A.SLICE)]
        vs.append(rotate_up(np.concatenate(u) if u else np.zeros((0, 2), np.int64), inc, ph, n0))
    return _sum(vs, [g for _, _, g in channels], acc)

def combine_arbitrary(rows, channels, tau0, step, taps, n_out=None, acc=None):
    """The model of sb200_combine_arbitrary -> int16 [n_out, 2]; n_out None: the outputs whose time lies inside the rows
    (arbitrary_model.n_inside); acc: the output buffer's samples before the call (int16 [n_out, 2]) for accumulate = 1, None for 0."""
    n_in = np.asarray(rows[0]).reshape(-1, 2).shape[0]
    n_out = A.n_inside(n_in, tau0, step) if n_out is None else n_out
    return combine_arbitrary_window(rows, channels, tau0, step, taps, 0, n_out, acc)
