"""What the GPU tests of the wideband calls share (test input and checks only): random channels, rows and taps for the channelizers and the
combiners, device rows and slot tables, the device transmitters, the stream receivers run over device rows, and their comparison with the
CPU oracle on the host rows."""
import ctypes as C
import numpy as np
import torch
import oracle_py
import wideband_inputs as W
from sora_b200 import api
from test_cpu_channelize import _full_scale, decode_11a

V, U32, U64 = C.c_void_p, C.c_uint32, C.c_uint64
FRAMES = 16                                            # results per stream of the receivers
OUT_11A, OUT_11B, OUT_11N = 4096, 4096, 1536           # delivered bytes per frame

def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count

# ---- random inputs of the channelizers ----------------------------------------------------------------------------------------------
DDC_INCS = [0, 2 ** 30, 2 ** 31, W.phase_inc(-20e6, 160e6), W.phase_inc(-60e6, 160e6), W.phase_inc(25e6, 176e6), 0x9E3779B9, 3 * 2 ** 30]

def ddc_channels(k, seed):
    rng = np.random.default_rng(seed)
    return [(DDC_INCS[i % len(DDC_INCS)], int(rng.integers(0, 2 ** 32)) if i % 3 else 0) for i in range(k)]

def ddc_taps(n, seed, total=40000):
    """n random Q15 taps, sum |t| = total (rounded down), the centre one largest."""
    rng = np.random.default_rng(seed)
    t = rng.integers(-1000, 1000, n).astype(np.float64); t[n // 2] = 5000.0
    return np.trunc(t * total / np.abs(t).sum()).astype(np.int16)

# A capture of at least 4 x SMs tiles runs every channel of a channelizer call in one CTA (the launch splits the channels into groups only
# until there are four CTAs per multiprocessor), and one of G tiles with 4 x SMs / G < K splits them into groups of several.  Identity and
# rotating channels are mixed within a group, and most increments are multiples of 2^29 (the channel plan of a 160 Msps capture), whose
# phases hit NCO[0] on every eighth sample.
GROUP_CH = [(0, 0), (2 ** 29, 0), (W.phase_inc(-60e6, 160e6), 0), (2 ** 30, 0xDEADBEEF), (0, 0x000FFFFF), (2 ** 31, 0), (0x9E3779B9, 12345),
            (3 * 2 ** 29, 1 << 29), (0, 1 << 20), (W.phase_inc(20e6, 160e6), 7), (W.phase_inc(-20e6, 160e6), 0), (0, 0), (5 * 2 ** 29, 0),
            (W.phase_inc(25e6, 176e6), 0x80000000), (7 * 2 ** 29, 99), (2 ** 32 - 2 ** 30, 0)]

# ---- random inputs of the combiners -------------------------------------------------------------------------------------------------
DUC_INCS = [0, 2 ** 30, 2 ** 31, 3 * 2 ** 30, W.phase_inc(-20e6, 160e6), W.phase_inc(-60e6, 160e6), W.phase_inc(25e6, 176e6), 0x9E3779B9]
GAINS = [4096, 0, 65535, 4096, 1, 30000, 4096, 8191]

def duc_channels(k, seed):
    rng = np.random.default_rng(seed)
    return [(DUC_INCS[i % len(DUC_INCS)], int(rng.integers(0, 2 ** 32)) if i % 3 else 0, GAINS[(i + seed) % len(GAINS)]) for i in range(k)]

def duc_rows(k, n, seed):
    return np.stack([_full_scale(n, seed + 1000 * i) for i in range(k)])

def duc_taps(n, U, seed, total=50000):
    """n random Q15 taps, the centre one largest, every branch j = r (mod U) with sum |t| <= total."""
    rng = np.random.default_rng(seed)
    t = rng.integers(-1000, 1000, n).astype(np.float64); t[n // 2] = 5000.0
    worst = max(np.abs(t[r::U]).sum() for r in range(min(U, n)))
    return np.trunc(t * min(total / worst, 32767 / 5000)).astype(np.int16)

# ---- device rows and slot tables ----------------------------------------------------------------------------------------------------
def ceil4(n):
    return (n + 3) // 4 * 4

def dev_rows(K, n, pad=0):
    """K zeroed device rows of n samples, ceil4(n) + pad apart: int16 [K, stride, 2] (stride = its shape[1])."""
    return torch.zeros((K, ceil4(n) + pad, 2), dtype=torch.int16, device="cuda")

def tables(K, stride, n):
    """The slot table of K streams of n samples, stride apart."""
    return np.arange(K, dtype=np.uint64) * stride, np.full(K, n, np.uint32)

# ---- the device transmitters --------------------------------------------------------------------------------------------------------
def tx11a(eng, mpdu, rate, seed):
    """One frame of k_tx11a into device memory -> int8 [ns, 2] device tensor."""
    flat, offs, lens = api._payload_table([mpdu]); sd = np.array([seed], np.uint8); ns = np.zeros(1, np.uint32)
    stride = api.Engine.tx11a_out_stride(len(mpdu), rate)
    out = torch.zeros((1, stride, 2), dtype=torch.int8, device="cuda")
    eng.tx11a_raw(api._ptr(flat), flat.size, api._ptr(offs), api._ptr(lens), api._ptr(sd), 1, rate, 0, 8, out.data_ptr(), stride, api._ptr(ns))
    return out[0, :int(ns[0])]

def tx11b(eng, mpdu, rate):
    flat, offs, lens = api._payload_table([mpdu]); ns = np.zeros(1, np.uint32)
    stride = api.Engine.tx11b_out_stride(len(mpdu), rate)
    out = torch.zeros((1, stride, 2), dtype=torch.int8, device="cuda")
    eng.tx11b_raw(api._ptr(flat), flat.size, api._ptr(offs), api._ptr(lens), 1, rate, 0, 0, 8, out.data_ptr(), stride, api._ptr(ns))
    return out[0, :int(ns[0])]

def tx11n(eng, mpdu, mcs, seed):
    flat, offs, lens = api._payload_table([mpdu]); sd = np.array([seed], np.uint8); ns = np.zeros(1, np.uint32)
    stride = api.Engine.tx11n_out_stride(len(mpdu), mcs)
    o0 = torch.zeros((1, stride, 2), dtype=torch.int16, device="cuda"); o1 = torch.zeros_like(o0)
    eng.tx11n_raw(api._ptr(flat), flat.size, api._ptr(offs), api._ptr(lens), api._ptr(sd), 1, mcs, 0, o0.data_ptr(), o1.data_ptr(), stride, api._ptr(ns))
    return o0[0, :int(ns[0])], o1[0, :int(ns[0])]

# ---- the stream receivers over K device rows of n samples, stride apart -> (res, out, sidx, cnt) -------------------------------------
def _results(K, dtype, nbytes):
    return np.zeros((K, FRAMES), dtype), np.zeros((K, FRAMES, nbytes), np.uint8), np.zeros((K, FRAMES), np.uint32), np.zeros(K, np.uint32)

def rx11a(e, d, stride, n, K):
    off, ln = tables(K, stride, n); res, out, sidx, cnt = _results(K, api.RESULT_DTYPE, OUT_11A)
    e._check(e._lib.sb200_rx11a_streams(e._h, V(d.data_ptr()), U64(K * stride), V(off.ctypes.data), V(ln.ctypes.data), U32(K), U32(FRAMES), V(out.ctypes.data),
                                        U32(OUT_11A), V(res.ctypes.data), V(sidx.ctypes.data), V(cnt.ctypes.data), V(0)), "sb200_rx11a_streams")
    return res, out, sidx, cnt

def rx11b(e, d, stride, n, K):
    """sidx: the sample_index of the results (the 802.11b receiver reports it there)."""
    off, ln = tables(K, stride, n); res, out, _, cnt = _results(K, api.RESULT11B_DTYPE, OUT_11B)
    e._check(e._lib.sb200_rx11b_streams(e._h, V(d.data_ptr()), U64(K * stride), V(off.ctypes.data), V(ln.ctypes.data), U32(K), U32(FRAMES), V(out.ctypes.data),
                                        U32(OUT_11B), V(res.ctypes.data), V(cnt.ctypes.data), V(0)), "sb200_rx11b_streams")
    return res, out, res["sample_index"], cnt

def rx11n(e, d0, d1, stride, n, K):
    off, ln = tables(K, stride, n); res, out, sidx, cnt = _results(K, api.RESULT11N_DTYPE, OUT_11N)
    e._check(e._lib.sb200_rx11n_streams(e._h, V(d0.data_ptr()), V(d1.data_ptr()), U64(K * stride), V(off.ctypes.data), V(ln.ctypes.data), U32(K), U32(FRAMES),
                                        V(out.ctypes.data), U32(OUT_11N), V(res.ctypes.data), V(sidx.ctypes.data), V(cnt.ctypes.data), V(0)), "sb200_rx11n_streams")
    return res, out, sidx, cnt

# ---- the receivers' results against the CPU oracle on the host rows; each returns the oracle's [(results, bytes)] per row ------------
def equal_11a(rows, got):
    """Frame count, status, rate, length, CRC, symbol count, CFO, sample_index, detect_index (re-based: the oracle counts 20 Msps vectors
    from the capture's start) and every delivered byte."""
    res, out, sidx, cnt = got; dec = decode_11a(rows)
    for c, (o, ob) in enumerate(dec):
        assert cnt[c] == len(o), (c, cnt[c], o)
        r = res[c, :cnt[c]]
        for k in ("status", "rate_kbps", "length", "crc32", "nsym", "cfo_est"): assert (r[k] == o[k]).all(), (c, k)
        assert (sidx[c, :cnt[c]] == o["sample_index"]).all(), c
        seg = np.diff(np.concatenate([[0], o["sample_index"].astype(np.int64)]))
        assert (r["detect_index"] + np.concatenate([[0], np.cumsum(4 * (seg // 8))[:-1]]).astype(np.int64) == o["detect_index"]).all(), c
        for i in range(len(o)):
            L = int(o["length"][i]); assert (out[c, i, :L] == ob[i, :L]).all(), (c, i)
    return dec

def equal_11b(rows, got):
    """Frame count, status, rate, length, CRC, sample_index, detect_vec and every delivered byte (the FCS's last byte excepted)."""
    res, out, _, cnt = got; dec = [oracle_py.rx11b_run(r, max_frames=FRAMES, out_stride=OUT_11B) for r in rows]
    for c, (o, ob) in enumerate(dec):
        assert cnt[c] == len(o), (c, cnt[c], o)
        r = res[c, :cnt[c]]
        for k in ("status", "rate_kbps", "length", "crc32", "sample_index", "detect_vec"): assert (r[k] == o[k]).all(), (c, k)
        for i in range(len(o)):
            L = int(o["length"][i]) - 1; assert (out[c, i, :L] == ob[i, :L]).all(), (c, i)
    return dec

def equal_11n(rows0, rows1, got):
    """Frame count, status, MCS, length, CRC, symbol count, CFO, L-SIG length, sample_index, detect_index (re-based as for 802.11a) and
    every delivered byte."""
    res, out, sidx, cnt = got; dec = [oracle_py.rx11n_run(a, b, max_frames=FRAMES, out_stride=OUT_11N) for a, b in zip(rows0, rows1)]
    for c, (o, ob) in enumerate(dec):
        assert cnt[c] == len(o), (c, cnt[c], o)
        vec_base = 0; prev = 0
        for k in range(len(o)):
            for f in ("status", "mcs", "length", "crc32", "nsym", "cfo_est", "lsig_length"): assert res[c, k][f] == o[k][f], (c, k, f)
            assert sidx[c, k] == o[k]["sample_index"], (c, k)
            assert vec_base + res[c, k]["detect_index"] == o[k]["detect_index"], (c, k)
            vec_base += 4 * ((int(sidx[c, k]) - prev) // 8); prev = int(sidx[c, k])
            L = int(o[k]["length"]); assert (out[c, k, :L] == ob[k, :L]).all(), (c, k)
    return dec
