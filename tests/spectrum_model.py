"""numpy restatement of sb200_spectrum and sb200_power_meter (include/sora_b200.h): the reference's FFT<N> (kernel/core/inc/fft_r4dif.h)
on int arrays, vectorised over frames, and TSpecMeter<N> / TPowerMeter<N> (kernel/sdl/inc/sdlmeasure.hpp) around it.  Samples are int
arrays [..., 2] (re, im); every intermediate is kept in int64 and brought back to int16 or int32 exactly where the SSE code narrows."""
import numpy as np

def _sat(v): return np.clip(v, -32768, 32767)
def _sx16(v): return ((v + 32768) & 0xFFFF) - 32768
def _w32(v): return ((v + 2 ** 31) & 0xFFFFFFFF) - 2 ** 31

def gen_twiddle(N, M):
    """FFT_GetTwiddleConst<N, M>() as N / 4 (re, im) pairs: (trunc(32767 cos(2 pi j M / N)), trunc(-32767 sin(2 pi j M / N)))."""
    j = np.arange(N // 4)
    return np.stack([np.trunc(32767.0 * np.cos(2 * np.pi * j * M / N)), np.trunc(-32767.0 * np.sin(2 * np.pi * j * M / N))], 1).astype(np.int64)

def bitrev(N):
    """FFTLUTMapTable<N>: the plain log2(N)-bit reversal of the index."""
    b = N.bit_length() - 1
    i = np.arange(N)
    return np.array([int(format(k, "0%db" % b)[::-1], 2) if b else 0 for k in i], np.int64)

# The SSE operations, per lane on (re, im) pairs of int64 arrays
def _adds(a, b): return (_sat(a[0] + b[0]), _sat(a[1] + b[1]))
def _subs(a, b): return (_sat(a[0] - b[0]), _sat(a[1] - b[1]))
def _cnot(a): return (~a[0], ~a[1])                      # XOR with all ones
def _sra(a, n): return (a[0] >> n, a[1] >> n)
def _mulj(a): return (~a[1], a[0])                       # mul_j: flip, then XOR of the real halves
def _mulmj(a): return (a[1], ~a[0])                      # permutate_high<0xb1> then XOR of the imaginary halves: times -j
def _mul_shift(a, w):
    """mul_shift(a, w, 15): pmaddwd with conj (XOR) and flip of w, >> 15, the wrapping pack."""
    re = _w32(a[0] * w[0] + a[1] * ~w[1]); im = _w32(a[0] * w[1] + a[1] * w[0])
    return (_sx16(re >> 15), _sx16(im >> 15))

def _dft4(v, shift):
    x0, x1, x2, x3 = (_sra(u, shift) for u in v)
    s0, s1, s2, s3 = _adds(x0, x2), _adds(x1, x3), _adds(_cnot(x2), x0), _adds(_cnot(x3), x1)
    t3 = _mulmj(s3)
    return [_adds(s0, s1), _adds(_cnot(s1), s0), _adds(s2, t3), _adds(_cnot(t3), s2)]

def _dft8(v):
    a = [_sra(v[i], 3) for i in range(4)]; b = [_sra(v[4 + i], 3) for i in range(4)]
    d = [_subs(a[i], b[i]) for i in range(4)]; s = [_adds(a[i], b[i]) for i in range(4)]
    W0, W1, W3 = (32767, 0), (23169, -23169), (-23169, -23169)     # wFFTLUT8: W^0, W^1, W^0, W^3 of N = 8
    t2, t3 = _mulmj(d[2]), _mulmj(d[3])
    m0, m1 = _mul_shift(_adds(d[0], t2), W0), _mul_shift(_adds(d[1], t3), W1)
    m2, m3 = _mul_shift(_adds(_cnot(t2), d[0]), W0), _mul_shift(_adds(_cnot(t3), d[1]), W3)
    odd = [_adds(m0, m1), _adds(_cnot(m1), m0), _adds(m2, m3), _adds(_cnot(m3), m2)]
    return _dft4(s, 0) + odd

def fft(x):
    """FFT<N> (FFTSSEEx<N> then the FFTLUTMapTable read-out) of int [F, N, 2] frames -> int64 [F, N, 2] in natural bin order."""
    x = np.asarray(x, np.int64)
    F, N = x.shape[:2]
    re, im = x[..., 0].copy(), x[..., 1].copy()
    L = N
    while L >= 16:                                       # FFTSSE<L> on every block of L samples
        Q = L // 4
        r = re.reshape(F, N // L, 4, Q); i = im.reshape(F, N // L, 4, Q)
        a, b, c, d = [(_sra((r[:, :, k], i[:, :, k]), 2)) for k in range(4)]
        ac, bd, a_c, b_d = _adds(a, c), _adds(b, d), _subs(a, c), _subs(b, d)
        jbd = _mulj(b_d)
        w = [gen_twiddle(L, M) for M in (1, 2, 3)]
        y0 = _adds(ac, bd)
        y1 = _mul_shift(_subs(ac, bd), (w[1][:, 0], w[1][:, 1]))
        y2 = _mul_shift(_subs(a_c, jbd), (w[0][:, 0], w[0][:, 1]))
        y3 = _mul_shift(_adds(a_c, jbd), (w[2][:, 0], w[2][:, 1]))
        re = np.stack([y0[0], y1[0], y2[0], y3[0]], 2).reshape(F, N); im = np.stack([y0[1], y1[1], y2[1], y3[1]], 2).reshape(F, N)
        L = Q
    B = L
    r = re.reshape(F, N // B, B); i = im.reshape(F, N // B, B)
    v = [(r[:, :, k], i[:, :, k]) for k in range(B)]
    out = _dft4(v, 2) if B == 4 else _dft8(v)
    re = np.stack([o[0] for o in out], 2).reshape(F, N); im = np.stack([o[1] for o in out], 2).reshape(F, N)
    m = bitrev(N)
    return np.stack([re[:, m], im[:, m]], 2)

def window(x, w):
    """(x w[n] + 2^14) >> 15 per component, w Q15 in [0, 32767]."""
    w = np.asarray(w, np.int64)[:, None]
    return (np.asarray(x, np.int64) * w + 16384) >> 15

def squared_norm(y):
    """SquaredNorm per bin: re^2 + im^2 in wrapping int32 (pmaddwd(x, x))."""
    return _w32(y[..., 0] * y[..., 0] + y[..., 1] * y[..., 1])

def spec_meter(frames):
    """TSpecMeter<N> of int [F, N, 2] frames -> int64 [F, N]: FFT<N>, SquaredNorm, bin 0 cleared."""
    p = squared_norm(fft(frames))
    p[:, 0] = 0
    return p

def frames_of(n_in, N, hop):
    return (n_in - N) // hop + 1 if n_in >= N else 0

def spectrum(rows, N, hop=None, avg=1, win=None):
    """sb200_spectrum of int16 rows [R, n_in, 2] -> int64 [R, ngroups, N]."""
    rows = np.asarray(rows, np.int64)
    if rows.ndim == 2: rows = rows[None]
    hop = N if hop is None else hop
    R, n_in = rows.shape[:2]
    ng = frames_of(n_in, N, hop) // avg
    out = np.zeros((R, ng, N), np.int64)
    if ng == 0: return out
    idx = (np.arange(ng * avg) * hop)[:, None] + np.arange(N)[None, :]
    for r in range(R):
        fr = rows[r][idx]
        if win is not None: fr = window(fr, win)
        out[r] = spec_meter(fr).reshape(ng, avg, N).sum(1)
    return out

def power_meter_blocks(blocks):
    """TPowerMeter<N> of int [B, N, 2] blocks -> uint32 [B]: per 4-sample vector the wrapping int32 sum of SquaredNorm (hadd), converted to
    the 64-bit size_t of N (a negative sum as 2^64 + v) and divided by N, summed in uint; the tail samples one by one the same way."""
    blocks = np.asarray(blocks, np.int64)
    B, N = blocks.shape[:2]
    e = squared_norm(blocks)
    vlen = N // 4
    def share(v): return (v.astype(np.int64).astype(np.uint64) // np.uint64(N)).astype(np.uint64) & np.uint64(0xFFFFFFFF)
    tot = np.zeros(B, np.uint64)
    if vlen:
        s = _w32(e[:, :4 * vlen].reshape(B, vlen, 4).sum(2))
        tot += share(s).sum(1, dtype=np.uint64)
    if N % 4:
        tot += share(e[:, 4 * vlen:]).sum(1, dtype=np.uint64)
    return (tot & np.uint64(0xFFFFFFFF)).astype(np.uint32)

def power_meter(rows, N):
    """sb200_power_meter of int16 rows [R, n_in, 2] -> uint32 [R, n_in // N]."""
    rows = np.asarray(rows, np.int64)
    if rows.ndim == 2: rows = rows[None]
    R, n_in = rows.shape[:2]
    nb = n_in // N
    return np.stack([power_meter_blocks(rows[r, :nb * N].reshape(nb, N, 2)) for r in range(R)])
