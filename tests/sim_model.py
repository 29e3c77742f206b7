"""The numpy model of sb200_channel_sim (test input only): the arithmetic of include/sora_b200.h restated in 64-bit integers.  A vectorised
Philox4x32-10, the tables H and LNT from their closed forms (I0 summed as the same power series as the library's), the channelizer model's
NCO table, and the four stages: interpolation at the link's sample clock, multipath, carrier rotation and fixed-point Box-Muller noise.
sim computes whole rows; sim_window computes outputs m0 .. m1 of every row from the closed forms alone, so windows of a long device
capture can be checked without the whole of it."""
import numpy as np
from wideband_inputs import NCO

M32 = np.uint64(0xFFFFFFFF)

# ---- Philox4x32-10 ------------------------------------------------------------------------------------------------------------------
def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Random123's Philox4x32 with 10 rounds over arrays (broadcast): uint32 counter words and key words -> (w0, w1, w2, w3) uint32."""
    c = [np.asarray(v, np.uint64) & M32 for v in (c0, c1, c2, c3)]
    k0 = np.asarray(k0, np.uint64) & M32; k1 = np.asarray(k1, np.uint64) & M32
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]; p1 = np.uint64(0xCD9E8D57) * c[2]          # < 2^64: exact in uint64
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & M32]
        k0 = (k0 + np.uint64(0x9E3779B9)) & M32; k1 = (k1 + np.uint64(0xBB67AE85)) & M32
    return tuple(np.asarray(v, np.uint64).astype(np.uint32) for v in c)


# ---- tables -------------------------------------------------------------------------------------------------------------------------
def _i0(x):
    s = np.ones_like(x); t = np.ones_like(x); q = x * x / 4.0
    for k in range(1, 32):
        t = t * (q / (float(k) * k)); s = s + t
    return s

def _h_table():
    d = np.arange(8)[None, :] - 3 - (np.arange(256) / 256.0)[:, None]
    with np.errstate(invalid="ignore", divide="ignore"):
        sinc = np.where(d == 0.0, 1.0, np.sin(np.pi * d) / (np.pi * d))
    return np.rint(16384.0 * sinc * _i0(5.0 * np.sqrt(1.0 - (d / 4.0) * (d / 4.0))) / _i0(np.array(5.0))).astype(np.int64)

H = _h_table()                                                          # [256, 8] Q14: row p weights x(i - 3 .. i + 4)
LNT = np.rint(-np.log((2048.0 + np.arange(2048) + 0.5) / 4096.0) * 16777216.0).astype(np.int64)


# ---- the stages ---------------------------------------------------------------------------------------------------------------------
def _sat(v):
    return np.clip(v, -32768, 32767)

def interpolate(x, tau0, step, m):
    """Stage 1 for one input row x (int [n_in, 2]) at outputs m (int64 array, may be negative) -> int64 [len(m), 2]."""
    x = np.asarray(x, np.int64).reshape(-1, 2); n_in = len(x); m = np.asarray(m, np.int64)
    ok = m >= 0; mm = np.where(ok, m, 0).astype(np.uint64)
    tp = np.uint64(tau0) + mm * np.uint64(step) + np.uint64(1 << 23)
    i = (tp >> np.uint64(32)).astype(np.int64); p = ((tp >> np.uint64(24)) & np.uint64(255)).astype(np.int64)
    idx = i[:, None] - 3 + np.arange(8)[None, :]
    xv = np.where(((idx >= 0) & (idx < n_in))[..., None], x[np.clip(idx, 0, max(n_in - 1, 0))] if n_in else 0, 0)
    acc = (H[p][..., None] * xv).sum(1) + (1 << 13)
    return np.where(ok[:, None], _sat(acc >> 14), 0)

def multipath(s, g, L):
    """Stage 2 for one output row: s int64 [T, M + L - 1, 2] (s[t, L - 1 + k] = s_t(m0 + k)), g int [T, L, 2] -> int64 [M, 2]."""
    T, n = s.shape[:2]; M = n - (L - 1)
    re = np.full(M, 1 << 13, np.int64); im = np.full(M, 1 << 13, np.int64)
    for t in range(T):
        for j in range(L):
            gr, gi = int(g[t, j, 0]), int(g[t, j, 1])
            if gr == 0 and gi == 0: continue
            sv = s[t, L - 1 - j:L - 1 - j + M]
            re += gr * sv[:, 0] - gi * sv[:, 1]; im += gr * sv[:, 1] + gi * sv[:, 0]
    return np.stack([_sat(re >> 14), _sat(im >> 14)], 1)

def rotate(u, phase_inc, phase0, m):
    """Stage 3: u * e^{+j theta(m)} in Q14 (the combiner's sign)."""
    th = (np.uint64(phase0 % 2 ** 32) + np.asarray(m, np.uint64) * np.uint64(phase_inc % 2 ** 32)) & M32
    cs = NCO[(th >> np.uint64(20)).astype(np.int64)]
    C, S = cs[:, 0], cs[:, 1]
    return np.stack([_sat((u[:, 0] * C - u[:, 1] * S + (1 << 13)) >> 14), _sat((u[:, 1] * C + u[:, 0] * S + (1 << 13)) >> 14)], 1)

def gauss(wa, wb, sigma):
    """Stage 4's Gaussian pair from the uint32 words (wa, wb): int64 [n, 2], standard deviation sigma / 256 per component."""
    a = np.asarray(wa, np.uint64) | np.uint64(1)
    e = 32 - np.frexp(a.astype(np.float64))[1].astype(np.int64)          # clz32: a < 2^32 is exact in float64, frexp's exponent its bit length
    mant = (((a << e.astype(np.uint64)) & M32) >> np.uint64(20)).astype(np.int64)
    v = 2 * (11629080 * e + LNT[mant - 2048])
    r = np.floor(np.sqrt(v.astype(np.float64))).astype(np.int64)
    r -= (r * r > v); r += ((r + 1) * (r + 1) <= v)
    cs = NCO[(np.asarray(wb, np.uint64) >> np.uint64(20)).astype(np.int64)]
    q = int(sigma) * r
    return np.stack([(q * cs[:, 0] + (1 << 33)) >> 34, (q * cs[:, 1] + (1 << 33)) >> 34], 1)

def noise_words(m, r, l, seed):
    """(wa, wb) of output m of row r of link l."""
    m = np.asarray(m, np.uint64); pr = m >> np.uint64(1)
    w0, w1, w2, w3 = philox4x32_10(pr & M32, pr >> np.uint64(32), r, l, seed & 0xFFFFFFFF, seed >> 32)
    odd = (m & np.uint64(1)).astype(bool)
    return np.where(odd, w2, w0), np.where(odd, w3, w1)

def noise(m, r, l, seed, sigma):
    wa, wb = noise_words(m, r, l, seed)
    return gauss(wa, wb, sigma)


# ---- the whole -------------------------------------------------------------------------------------------------------------------------
def _link(rec):
    if isinstance(rec, np.void): return int(rec["tau0"]), int(rec["step"]), int(rec["phase_inc"]), int(rec["phase0"]), int(rec["noise_q8"])
    return tuple(int(v) for v in rec[:5])

def sim_window(x, links, taps, seed, m0, m1, link_ids=None):
    """Outputs m0 .. m1 of every row of every link: x int [nlinks, T, n_in, 2], links records (tau0, step, phase_inc, phase0, noise_q8) or a
    LINK_DTYPE array, taps int [nlinks, R, T, L, 2] or [R, T, L, 2] -> int16 [nlinks, R, m1 - m0, 2].  link_ids: the index of each link in
    its call (the noise counter's fourth word), 0 .. nlinks - 1 by default, so that a few links of a large call can be modelled alone."""
    x = np.asarray(x); nl, T = x.shape[:2]
    taps = np.asarray(taps, np.int64)
    if taps.ndim == 4: taps = np.broadcast_to(taps, (nl,) + taps.shape)
    R, L = taps.shape[1], taps.shape[3]
    m = np.arange(m0 - (L - 1), m1, dtype=np.int64); mo = np.arange(m0, m1, dtype=np.int64)
    out = np.zeros((nl, R, m1 - m0, 2), np.int16)
    for l in range(nl):
        tau0, step, inc, ph, sig = _link(links[l])
        s = np.stack([interpolate(x[l, t], tau0, step, m) for t in range(T)])
        for r in range(R):
            v = multipath(s, taps[l, r], L)
            if inc % 2 ** 32 or (ph % 2 ** 32) >> 20: v = rotate(v, inc, ph, mo)
            if sig: v = _sat(v + noise(mo, r, l if link_ids is None else int(link_ids[l]), seed, sig))
            out[l, r] = v
    return out

def sim(x, links, taps, n_out, seed=0):
    """The model of sb200_channel_sim: -> int16 [nlinks, R, n_out, 2]."""
    return sim_window(x, links, taps, seed, 0, n_out)
