"""The numpy model of sb200_combine_bank (include/sora_b200.h), in 64-bit integers (test input only).

direct() restates the header's arithmetic output by output: the IDFT value W_{n mod M}(i) of every input time the output meets, each
rounded once, then the branch of taps, sigma and the second rounding.  window() is the vectorised form: the IDFT of the input times a
window of outputs meets (a matrix product over the Q14 table), then the taps one at a time over all outputs.  It reads only those input
times, so long device captures are checked a window at a time.  combine_bank() covers the whole capture.
"""
import numpy as np
from wideband_inputs import NCO

def _twiddles(M, odd):
    """T[(2k + o) p mod 2M] as int64 C and S, indexed [k, p]."""
    k, p = np.arange(M)[:, None], np.arange(M)[None, :]
    T = NCO[(((2 * k + odd) * p) % (2 * M)) * (2048 // M)].astype(np.int64)
    return T[..., 0], T[..., 1]

def _finish(acc, n, M, odd, a):
    """y(n) = sat16(a(n) + ((sigma(n) acc(n) + 2^14) >> 15)) for int64 acc [N, 2] at outputs n."""
    sigma = np.where(odd * ((n // M) % 2) == 1, -1, 1)[:, None]
    y = (sigma * acc + (1 << 14)) >> 15
    if a is not None: y = y + np.asarray(a, np.int64).reshape(-1, 2)
    return np.clip(y, -32768, 32767).astype(np.int16)

def direct(rows, U, odd, taps, n_out, acc=None):
    """The stated arithmetic, output by output: int16 [M, n_in, 2] -> int16 [n_out, 2]; acc: out before the call (accumulate).  For small sizes."""
    x = np.asarray(rows, np.int64); M, n_in = x.shape[:2]; taps = [int(t) for t in taps]; c = len(taps) // 2
    C, S = _twiddles(M, odd)
    def W(p, i):
        re = sum(int(x[k, i, 0]) * int(C[k, p]) - int(x[k, i, 1]) * int(S[k, p]) for k in range(M))
        im = sum(int(x[k, i, 1]) * int(C[k, p]) + int(x[k, i, 0]) * int(S[k, p]) for k in range(M))
        return (re + (1 << 13)) >> 14, (im + (1 << 13)) >> 14
    out = np.zeros((n_out, 2), np.int64)
    for n in range(n_out):
        p = n % M; ar = ai = 0
        for i in range(n_in):
            j = c + U * i - n
            if 0 <= j < len(taps) and taps[j]:
                wr, wi = W(p, i); ar += taps[j] * wr; ai += taps[j] * wi
        out[n] = ar, ai
    return _finish(out, np.arange(n_out), M, odd, acc)

def window(rows, M, U, odd, taps, n0, n1, acc=None):
    """Outputs n0 .. n1, from the input times they meet only: int16 [n1 - n0, 2]; acc: out[n0:n1] before the call (accumulate)."""
    taps = np.asarray(taps, np.int64); c = len(taps) // 2; N = n1 - n0
    n_in = rows.shape[1]
    if N <= 0: return np.zeros((0, 2), np.int16)
    lo = -(-(n0 - c) // U); hi = (n1 - 1 + c) // U + 1                 # input times i with n0 - c <= U i <= n1 - 1 + c
    seg = np.zeros((M, hi - lo, 2), np.int64); a, b = max(lo, 0), min(hi, n_in)
    if b > a: seg[:, a - lo:b - lo] = np.asarray(rows[:, a:b], np.int64)
    C, S = _twiddles(M, odd)
    xr, xi = seg[..., 0].T, seg[..., 1].T                                # [i, k]
    Wr = (xr @ C - xi @ S + (1 << 13)) >> 14; Wi = (xi @ C + xr @ S + (1 << 13)) >> 14   # [i, p]
    n = np.arange(n0, n1); p = n % M
    accr = np.zeros(N, np.int64); acci = np.zeros(N, np.int64)
    for j, t in enumerate(taps):                                         # tap j meets input i = (n - c + j) / U where U divides it
        if not t: continue
        m = n - c + j; ok = m % U == 0; i = m[ok] // U - lo
        accr[ok] += t * Wr[i, p[ok]]; acci[ok] += t * Wi[i, p[ok]]
    return _finish(np.stack([accr, acci], 1), n, M, odd, acc)

def combine_bank(rows, U, odd, taps, n_out=None, acc=None):
    """The whole capture: int16 [M, n_in, 2] -> int16 [n_out, 2], n_out = U n_in by default."""
    rows = np.asarray(rows); M, n_in = rows.shape[:2]
    return window(rows, M, U, odd, taps, 0, U * n_in if n_out is None else n_out, acc)

def channels(M, odd):
    """sb200_combine's channels (phase_inc, phase0, gain) that the bank's rows are: phase_inc = (2k + o) 2^31 / M, unity gain."""
    return [(((2 * k + odd) * 2 ** 31 // M) % 2 ** 32, 0, 4096) for k in range(M)]

def combine_bound(rows, taps, U):
    """The header's bound on |bank - sb200_combine| per component where nothing saturates: 1.2072 K + 0.5 B / 32768 + 0.5."""
    K = int(sum(np.any(np.asarray(r) != 0) for r in rows))
    B = max(int(np.abs(np.asarray(taps, np.int64)[r::U]).sum()) for r in range(U))
    return 1.2072 * K + 0.5 * B / 32768 + 0.5
