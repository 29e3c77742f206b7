"""ctypes binding of oracle/libsora_oracle.so — TEST INFRASTRUCTURE (checker only, never the product path)."""
import ctypes as C, os, subprocess, numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = None

class FrameResult(C.Structure):
    _fields_ = [("status", C.c_uint32), ("rate_kbps", C.c_uint32), ("length", C.c_uint32), ("crc32", C.c_uint32),
                ("nsym", C.c_uint32), ("sample_index", C.c_uint32), ("detect_index", C.c_uint32),
                ("cfo_est", C.c_int16), ("peak_index", C.c_uint16)]

RES_DTYPE = np.dtype([("status", "<u4"), ("rate_kbps", "<u4"), ("length", "<u4"), ("crc32", "<u4"), ("nsym", "<u4"),
                      ("sample_index", "<u4"), ("detect_index", "<u4"), ("cfo_est", "<i2"), ("peak_index", "<u2")])

E_FRAME_OK, E_CRC32_FAIL, E_PLCP_FAIL, E_NO_FRAME = 1, 0x80000006, 0x80000005, 0x8000F001

def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(ROOT, "oracle", "libsora_oracle.so")
        srcs = [os.path.join(ROOT, "oracle", f) for f in os.listdir(os.path.join(ROOT, "oracle")) if f.endswith((".cpp", ".h", ".inc"))]
        stale = lambda: not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)
        if stale():                                     # several ranks / test workers may get here at once: one builds, the others wait for it
            import fcntl
            with open(os.path.join(ROOT, "oracle", ".build.lock"), "w") as lk:
                fcntl.flock(lk, fcntl.LOCK_EX)
                try:
                    if stale(): subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
                finally: fcntl.flock(lk, fcntl.LOCK_UN)
        use_library(so)
    return _LIB

def use_library(so):
    """Bind the oracle library at path `so` (a build of oracle/ with other compiler flags, for instance) instead of oracle/libsora_oracle.so."""
    global _LIB
    _LIB = C.CDLL(so)
    _LIB.sbo_viterbi_block.restype = C.c_uint64
    _LIB.sbo_uatan2.restype = C.c_int16; _LIB.sbo_usin.restype = C.c_int16; _LIB.sbo_ucos.restype = C.c_int16
    _LIB.sbo_uatan2.argtypes = [C.c_int, C.c_int]; _LIB.sbo_usin.argtypes = [C.c_int16]; _LIB.sbo_ucos.argtypes = [C.c_int16]
    _LIB.sbo_sts_pattern.restype = C.POINTER(C.c_int16)
    _LIB.sbo_crc32.restype = C.c_uint32
    _LIB.sbo_viterbi_signal.restype = C.c_uint32
    return _LIB

def _p(a, t=C.c_void_p):
    return a.ctypes.data_as(t)

def rx11a_run(iq, max_frames=16, out_stride=4096):
    """iq: int16 array [n,2] (40 Msps). Returns (results structured array, bytes [nf, stride])."""
    iq = np.ascontiguousarray(iq, dtype=np.int16)
    res = np.zeros(max_frames, dtype=RES_DTYPE); out = np.zeros((max_frames, out_stride), dtype=np.uint8)
    n = lib().sbo_rx11a_run(_p(iq), C.c_uint64(iq.shape[0]), C.c_int(max_frames), _p(res), _p(out), C.c_uint64(out_stride))
    return res[:n], out[:n]

def rx11a_batch(iq, off, length, out_stride=2048, nthreads=1):
    iq = np.ascontiguousarray(iq, dtype=np.int16)
    off = np.ascontiguousarray(off, dtype=np.uint64); length = np.ascontiguousarray(length, dtype=np.uint32)
    nf = len(off)
    res = np.zeros(nf, dtype=RES_DTYPE); out = np.zeros((nf, out_stride), dtype=np.uint8)
    lib().sbo_rx11a_batch(_p(iq), _p(off), _p(length), C.c_uint32(nf), _p(res), _p(out), C.c_uint64(out_stride), C.c_int(nthreads))
    return res, out

def rx11a_batch_2t(iq, off, length, out_stride=2048, npipes=1):
    """The same batch through the reference's two-thread topology (front end | Viterbi thread per pipeline), npipes pipelines."""
    iq = np.ascontiguousarray(iq, dtype=np.int16)
    off = np.ascontiguousarray(off, dtype=np.uint64); length = np.ascontiguousarray(length, dtype=np.uint32)
    nf = len(off)
    res = np.zeros(nf, dtype=RES_DTYPE); out = np.zeros((nf, out_stride), dtype=np.uint8)
    lib().sbo_rx11a_batch_2t(_p(iq), _p(off), _p(length), C.c_uint32(nf), _p(res), _p(out), C.c_uint64(out_stride), C.c_int(npipes))
    return res, out

def rx11a_taps(iq, max_sym=600):
    iq = np.ascontiguousarray(iq, dtype=np.int16)
    res = np.zeros(1, dtype=RES_DTYPE)
    fc = np.zeros((64, 2), np.int16); cc = np.zeros((64, 2), np.int16)
    fo = np.zeros((max_sym, 64, 2), np.int16); eq = np.zeros_like(fo); tr = np.zeros_like(fo)
    soft = np.zeros(max_sym * 288, np.uint8); so = np.zeros(max_sym + 1, np.uint32)
    fi = np.zeros_like(fo); li = np.zeros((144, 2), np.int16); si = np.zeros((max_sym, 80, 2), np.int16)
    ns = lib().sbo_rx11a_taps_blocks(_p(iq), C.c_uint64(iq.shape[0]), _p(res), _p(fc), _p(cc), _p(fo), _p(eq), _p(tr), _p(soft), _p(so),
                                     C.c_int(max_sym), _p(fi), _p(li), _p(si))
    return dict(res=res[0], freq_coeffs=fc, chan_coeffs=cc, fft_in=fi[:ns], fft_out=fo[:ns], equalized=eq[:ns], tracked=tr[:ns],
                soft=soft[:so[ns]], soft_off=so[:ns + 1], nsym=ns, lts_in=li, sym_in=si[:ns])

def viterbi_block(soft, code_rate, frame_len_bytes, depth=256, lookahead=24):
    soft = np.ascontiguousarray(soft, dtype=np.uint8)
    out = np.zeros(frame_len_bytes + 2 + 64, dtype=np.uint8)
    n = lib().sbo_viterbi_block(_p(soft), C.c_uint64(len(soft)), C.c_int(code_rate), C.c_uint32(frame_len_bytes),
                                C.c_uint32(depth), C.c_uint32(lookahead), _p(out))
    return out[:n]

def viterbi_blocks(soft2d, code_rate, frame_len_bytes, depth=256, lookahead=24, nthreads=1):
    soft2d = np.ascontiguousarray(soft2d, dtype=np.uint8)
    nb, ns = soft2d.shape
    stride = frame_len_bytes + 2
    out = np.zeros((nb, stride), dtype=np.uint8)
    lib().sbo_viterbi_blocks(_p(soft2d), C.c_uint64(ns), C.c_uint32(nb), C.c_int(code_rate), C.c_uint32(frame_len_bytes),
                             C.c_uint32(depth), C.c_uint32(lookahead), _p(out), C.c_uint64(stride), C.c_int(nthreads))
    return out

def viterbi_blocks_n(soft2d, code_rate, frame_len_bytes, depth=256, lookahead=24, nthreads=1):
    """viterbi_blocks, plus the bytes each block produced: fewer than L + 2 when its soft values end before the flush point
    (only out[i, :n[i]] is defined then; the rest of the row is zero)."""
    soft2d = np.ascontiguousarray(soft2d, dtype=np.uint8)
    nb, ns = soft2d.shape
    stride = frame_len_bytes + 2
    out = np.zeros((nb, stride), dtype=np.uint8); n = np.zeros(nb, dtype=np.uint32)
    lib().sbo_viterbi_blocks_n(_p(soft2d), C.c_uint64(ns), C.c_uint32(nb), C.c_int(code_rate), C.c_uint32(frame_len_bytes),
                               C.c_uint32(depth), C.c_uint32(lookahead), _p(out), C.c_uint64(stride), _p(n), C.c_int(nthreads))
    return out, n

def descramble(decoded):
    """The receive chains' descrambler (oracle/rx11a.cpp sink_byte) on Viterbi output (SERVICE + PSDU): the PSDU bytes."""
    d = np.ascontiguousarray(decoded, dtype=np.uint8); out = np.zeros(max(len(d) - 2, 0), np.uint8)
    lib().sbo_descramble(_p(d), C.c_uint32(len(d)), _p(out))
    return out

def _xform(fn, x, N):
    """x: int16 [..., N, 2], any number of leading axes; one transform per vector, same shape out."""
    x = np.ascontiguousarray(x, dtype=np.int16); assert x.shape[-2:] == (N, 2), x.shape
    o = np.zeros_like(x); fn(C.c_uint64(x.size // (2 * N)), _p(x), _p(o)); return o
def fft64(x): return _xform(lib().sbo_fft64_n, x, 64)
def ifft64(x): return _xform(lib().sbo_ifft64_n, x, 64)
def crc32(b):
    b = np.ascontiguousarray(b, dtype=np.uint8); return int(lib().sbo_crc32(_p(b), C.c_uint64(len(b))))

RES11B_DTYPE = np.dtype([("status", "<u4"), ("rate_kbps", "<u4"), ("length", "<u4"), ("crc32", "<u4"), ("sample_index", "<u4"), ("detect_vec", "<u4")])

def rx11b_run(iq, max_frames=8, out_stride=4096):
    iq = np.ascontiguousarray(iq, dtype=np.int16)
    res = np.zeros(max_frames, dtype=RES11B_DTYPE); out = np.zeros((max_frames, out_stride), dtype=np.uint8)
    n = lib().sbo_rx11b_run(_p(iq), C.c_uint64(iq.shape[0]), C.c_int(max_frames), _p(res), _p(out), C.c_uint64(out_stride))
    return res[:n], out[:n]

def rx11b_batch(iq, off, length, out_stride=4096, nthreads=1):
    iq = np.ascontiguousarray(iq, dtype=np.int16)
    off = np.ascontiguousarray(off, dtype=np.uint64); length = np.ascontiguousarray(length, dtype=np.uint32)
    nf = len(off)
    res = np.zeros(nf, dtype=RES11B_DTYPE); out = np.zeros((nf, out_stride), dtype=np.uint8)
    lib().sbo_rx11b_batch(_p(iq), _p(off), _p(length), C.c_uint32(nf), _p(res), _p(out), C.c_uint64(out_stride), C.c_int(nthreads))
    return res, out

def resample_44_40(iq44):
    iq44 = np.ascontiguousarray(iq44, dtype=np.int16)
    out = np.zeros_like(iq44)
    lib().sbo_resample_44_40.restype = C.c_uint64
    n = lib().sbo_resample_44_40(_p(iq44), C.c_uint64(iq44.shape[0]), _p(out))
    return out[:n].copy()


# ---- 802.11n 2x2 ------------------------------------------------------------------------------------------------------
RES11N_DTYPE = np.dtype([("status", "<u4"), ("mcs", "<u4"), ("length", "<u4"), ("crc32", "<u4"), ("nsym", "<u4"),
                         ("sample_index", "<u4"), ("detect_index", "<u4"), ("cfo_est", "<i2"), ("lsig_length", "<u2")])

def rx11n_run(iq0, iq1, max_frames=8, out_stride=2048):
    iq0 = np.ascontiguousarray(iq0, dtype=np.int16); iq1 = np.ascontiguousarray(iq1, dtype=np.int16)
    res = np.zeros(max_frames, dtype=RES11N_DTYPE); out = np.zeros((max_frames, out_stride), dtype=np.uint8)
    n = lib().sbo_rx11n_run(_p(iq0), _p(iq1), C.c_uint64(iq0.reshape(-1, 2).shape[0]), C.c_int(max_frames), _p(res), _p(out), C.c_uint64(out_stride))
    return res[:n], out[:n]

def rx11n_batch(iq0, iq1, off, length, out_stride=1536, nthreads=1):
    iq0 = np.ascontiguousarray(iq0, dtype=np.int16); iq1 = np.ascontiguousarray(iq1, dtype=np.int16)
    off = np.ascontiguousarray(off, dtype=np.uint64); length = np.ascontiguousarray(length, dtype=np.uint32); nf = len(off)
    res = np.zeros(nf, dtype=RES11N_DTYPE); out = np.zeros((nf, out_stride), dtype=np.uint8)
    lib().sbo_rx11n_batch(_p(iq0), _p(iq1), _p(off), _p(length), C.c_uint32(nf), _p(res), _p(out), C.c_uint64(out_stride), C.c_int(nthreads))
    return res, out

def rx11n_taps(iq0, iq1, max_sym=300):
    iq0 = np.ascontiguousarray(iq0, dtype=np.int16); iq1 = np.ascontiguousarray(iq1, dtype=np.int16)
    res = np.zeros(1, dtype=RES11N_DTYPE)
    siso = np.zeros((2, 64, 2), np.int16); hinv = np.zeros((4, 64, 2), np.int16)
    fo = np.zeros((2, max_sym, 64, 2), np.int16); eq = np.zeros((2, max_sym, 64, 2), np.int16); fi = np.zeros_like(fo)
    soft = np.zeros(max_sym * 624, np.uint8); nsoft = C.c_uint32(0); theta = np.zeros(max_sym, np.int16); sig = np.zeros(9, np.uint8); nfft = C.c_int(0)
    nd = lib().sbo_rx11n_taps_in(_p(iq0), _p(iq1), C.c_uint64(iq0.reshape(-1, 2).shape[0]), _p(res), _p(siso), _p(hinv), _p(fo), _p(eq), _p(soft),
                              C.byref(nsoft), _p(theta), _p(sig), C.c_int(max_sym), C.byref(nfft), _p(fi))
    return dict(res=res[0], siso=siso, hinv=hinv, fft_in=fi[:, :nfft.value], fft_out=fo[:, :nfft.value], eq=eq[:, :nd], soft=soft[:nsoft.value], theta=theta[:nd], sig=sig, ndata=nd)

def tables11n():
    sc = np.zeros((65536, 2), np.int16); at = np.zeros(4097, np.int16); dm = np.zeros(256, np.uint8); c8 = np.zeros(256, np.uint8)
    di = np.zeros((4, 2, 312), np.uint16); ls = np.zeros(64, np.uint8); hs = np.zeros(64, np.uint8)
    lib().sbo_tables11n(_p(sc), _p(at), _p(dm), _p(c8), _p(di), _p(ls), _p(hs))
    d16 = np.zeros((2, 256), np.uint8); d64 = np.zeros((3, 288), np.uint8); lib().sbo_tables11n_qam(_p(d16), _p(d64))
    return dict(sincos=sc, atan=at, demap=dm, crc8=c8, deint=di, lltf_sign=ls, htltf_sign=hs, demap16=d16, demap64=d64)

def set_ht_mcs_limit(first_refused=11):
    """11 = the reference's HT-SIG parser as shipped (MCS 8..10); 15 = the 16-/64-QAM branches enabled (MCS 8..14)."""
    lib().sbo_set_ht_mcs_limit(C.c_uint32(first_refused))


# ---- 802.11a transmit (brick modulator restatement) ---------------------------------------------------------------------
def tx11a_modulate(payload, rate_kbps, seed=0xFF, tail_zeros=32):
    """payload: MPDU bytes without FCS.  Returns int8 [n, 2] complex samples at 40 Msps (what `demod11 -m` writes)."""
    payload = np.ascontiguousarray(payload, dtype=np.uint8); L = lib(); L.sbo_tx11a_modulate.restype = C.c_uint64
    nsym = L.sbo_tx11a_nsym(C.c_uint32(len(payload)), C.c_uint32(rate_kbps)); cap = 640 + 160 * (1 + nsym) + tail_zeros
    out = np.zeros((cap, 2), np.int8)
    n = L.sbo_tx11a_modulate(_p(payload), C.c_uint32(len(payload)), C.c_uint32(rate_kbps), C.c_uint8(seed), _p(out), C.c_uint64(cap), C.c_uint32(tail_zeros))
    assert n == cap, (n, cap)
    return out

def tx11a_scramble(data, ctrl, seed):
    """The oracle's T11aSc: uint8 [n] under the per-byte scramble_ctrl ctrl (0 none, 1 scramble, 2 tail), register from seed."""
    d = np.ascontiguousarray(data, np.uint8); c = np.ascontiguousarray(np.broadcast_to(ctrl, d.shape), np.uint8); out = np.zeros_like(d)
    lib().sbo_tx11a_scramble_n(_p(d), _p(c), C.c_uint64(len(d)), C.c_uint8(seed), _p(out)); return out
def tx11a_encode_bits(data, cr):
    """The oracle's convolutional encoder and puncturing (cr 0 = 1/2, 1 = 2/3, 2 = 3/4) from state 0: coded bits, one per byte."""
    d = np.ascontiguousarray(data, np.uint8); out = np.zeros(16 * len(d) + 8, np.uint8); L = lib(); L.sbo_tx11a_encode_bits.restype = C.c_uint64
    m = L.sbo_tx11a_encode_bits(_p(d), C.c_uint64(len(d)), C.c_int(cr), _p(out)); return out[:m]
def tx11a_interleave(bits, nbpsc):
    """The oracle's 802.11a interleaver on bits [nsym, 48 nbpsc] (one per byte): the on-air bits."""
    b = np.ascontiguousarray(bits, np.uint8).reshape(-1, 48 * nbpsc); out = np.zeros_like(b)
    lib().sbo_tx11a_interleave_n(_p(b), C.c_uint64(len(b)), C.c_int(nbpsc), _p(out)); return out
def tx11a_map(bits, nbpsc):
    """The oracle's 802.11a mapper on on-air bits [nsym, 48 nbpsc]: int16 [nsym, 48, 2]."""
    b = np.ascontiguousarray(bits, np.uint8).reshape(-1, 48 * nbpsc); out = np.zeros((len(b), 48, 2), np.int16)
    lib().sbo_tx11a_map_n(_p(b), C.c_uint64(len(b)), C.c_int(nbpsc), _p(out)); return out
def tx11a_add_pilot(data48):
    """The oracle's pilot inserter on int16 [nsym, 48, 2] (pilot index 127 first): int16 [nsym, 64, 2]."""
    d = np.ascontiguousarray(data48, np.int16).reshape(-1, 48, 2); out = np.zeros((len(d), 64, 2), np.int16)
    lib().sbo_tx11a_add_pilot_n(_p(d), C.c_uint64(len(d)), _p(out)); return out
def tx11a_ifftx(spec64):
    """The oracle's TIFFTx on int16 [nsym, 64, 2]: int16 [nsym, 160, 2]."""
    d = np.ascontiguousarray(spec64, np.int16).reshape(-1, 64, 2); out = np.zeros((len(d), 160, 2), np.int16)
    lib().sbo_tx11a_ifftx_n(_p(d), C.c_uint64(len(d)), _p(out)); return out
def tx11a_pack8(x):
    """The oracle's TPackSample16to8 on int16 [n, 2]: int8 [n, 2]."""
    d = np.ascontiguousarray(x, np.int16).reshape(-1, 2); out = np.zeros(d.shape, np.int8)
    lib().sbo_tx11a_pack8_n(_p(d), C.c_uint64(len(d)), _p(out)); return out

def tx11a_legacy_modulate(body, rate_kbps, append_crc=True):
    """The reference's LEGACY transmitter (BB11ATxFrameMod; oracle/tx11a_legacy.cpp).  Returns int8 [n, 2]: 640 + 160 (1 + nsym) + 8 samples at 40 Msps."""
    body = np.ascontiguousarray(body, dtype=np.uint8); L = lib(); L.sbo_tx11a_legacy_modulate.restype = C.c_uint64
    pre = np.fromfile(os.path.join(ROOT, "tests", "golden", "preamble40_11a.i16"), np.int16)
    nsym = L.sbo_tx11a_legacy_nsym(C.c_uint32(len(body) + (4 if append_crc else 0)), C.c_uint32(rate_kbps)); assert nsym, "not an 802.11a rate"
    cap = 640 + 160 * (1 + nsym) + 8
    out = np.zeros((cap, 2), np.int8)
    n = L.sbo_tx11a_legacy_modulate(_p(body), C.c_uint32(len(body)), C.c_int(1 if append_crc else 0), C.c_uint32(rate_kbps), _p(pre), _p(out), C.c_uint64(cap))
    assert n == cap, (n, cap)
    return out

def ifft128(x): return _xform(lib().sbo_ifft128_n, x, 128)
def ifft128_inputs(fn, *args, **kw):
    """Run fn(*args, **kw) (an oracle transmitter) and return (its result, int16 [n, 128, 2]: the input of every ifft128 it made, in order)."""
    L = lib(); L.sbo_ifft128_log_end.restype = C.c_uint64; L.sbo_ifft128_log_begin()
    try: r = fn(*args, **kw)
    finally: n = L.sbo_ifft128_log_end(None, C.c_uint64(0))
    x = np.zeros((n, 128, 2), np.int16); L.sbo_ifft128_log_end(_p(x), C.c_uint64(n))   # the log stays until the next _begin
    return r, x


# ---- 802.11b transmit (brick modulator restatement) ---------------------------------------------------------------------
def tx11b_modulate(payload, rate_kbps, init_phase=0, return_phase=False):
    """payload: MPDU bytes without FCS.  Returns int8 [n, 2] complex samples at 44 Msps (the COMPLEX8 buffer TModSink fills)."""
    payload = np.ascontiguousarray(payload, dtype=np.uint8); L = lib(); L.sbo_tx11b_modulate.restype = C.c_uint64
    cap = L.sbo_tx11b_nsamples(C.c_uint32(len(payload)), C.c_uint32(rate_kbps)); assert cap, "not an 802.11b rate"
    out = np.zeros((cap, 2), np.int8)
    fin = C.c_uint32(0)
    n = L.sbo_tx11b_modulate(_p(payload), C.c_uint32(len(payload)), C.c_uint32(rate_kbps), C.c_uint32(init_phase), _p(out), C.c_uint64(cap), C.byref(fin))
    assert n == cap, (n, cap)
    return (out, fin.value) if return_phase else out

def tx11b_taps():
    o = np.zeros(20, np.int16); lib().sbo_tx11b_taps(_p(o)); return o


# ---- 802.11n transmit (brick modulator restatement) ---------------------------------------------------------------------
def tx11n_modulate(payload, mcs, seed=0xAB):
    """payload: MPDU bytes without FCS.  Returns two int16 [n, 2] streams at 40 Msps (what `demod11` writes to *_0.dmp / *_1.dmp)."""
    payload = np.ascontiguousarray(payload, dtype=np.uint8); L = lib(); L.sbo_tx11n_modulate.restype = C.c_uint64
    sig = C.c_uint32(0); nsym = L.sbo_tx11n_nsym(C.c_uint32(len(payload)), C.c_uint32(mcs), C.byref(sig)); assert nsym, "mcs must be 8 .. 14"
    cap = 640 + 480 + 480 + 160 * nsym
    o0 = np.zeros((cap, 2), np.int16); o1 = np.zeros((cap, 2), np.int16)
    n = L.sbo_tx11n_modulate(_p(payload), C.c_uint32(len(payload)), C.c_uint32(mcs), C.c_uint8(seed), _p(o0), _p(o1), C.c_uint64(cap))
    assert n == cap, (n, cap)
    return o0, o1

def tx11n_preamble_tables():
    a = np.zeros((320, 2), np.int16); b = np.zeros((320, 2), np.int16); c = np.zeros((160, 2), np.int16); d = np.zeros((160, 2), np.int16)
    lib().sbo_tx11n_preamble_tables(_p(a), _p(b), _p(c), _p(d)); return a, b, c, d


def fir37_legacy(chips, variant=0):
    """oracle/tx11b_legacy.cpp: BB11BPMDSpreadFIR4SSE (variant 0) / BB11BPMDSpreadFIR4ASM (variant 1) restated.  int8 [n,2] -> int8 [n,2] (n % 8 == 0)."""
    x = np.ascontiguousarray(chips, dtype=np.int8).reshape(-1, 2); out = np.zeros_like(x)
    lib().sbo_fir37_legacy(C.c_void_p(x.ctypes.data), C.c_uint32(len(x)), C.c_int(variant), C.c_void_p(out.ctypes.data))
    return out

_REF_FIR = None
def ref_fir37_available():
    return os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libfir37_ref.so"))
def ref_fir37(chips):
    """oracle/_ref/libfir37_ref.so: the reference's own FIR37SSE_INTRINSIC body + coefficient table, compiled by oracle/build_ref.sh."""
    global _REF_FIR
    if _REF_FIR is None: _REF_FIR = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libfir37_ref.so"))
    x = np.ascontiguousarray(chips, dtype=np.int8).reshape(-1, 2); out = np.zeros_like(x)
    _REF_FIR.ref_fir37(C.c_void_p(x.ctypes.data), C.c_uint(len(x)), C.c_void_p(out.ctypes.data))
    return out

_REF_VIT = None
REF_VITERBI_INSTS = {0: (48, 256, 24), 1: (312, 192, 36), 2: (48, 24, 24)}   # inst -> (N_INPUT, TRELLIS_DEPTH, TRELLIS_LOOKAHEAD)
REF_TRELLIS_MAX = 5000 * 8
def ref_viterbi_available():
    return os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libviterbi_ref.so"))
def _ref_vit():
    global _REF_VIT
    if _REF_VIT is None:
        L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libviterbi_ref.so"))
        L.ref_viterbi_sig11.restype = C.c_uint32; L.ref_viterbi_sig11.argtypes = [C.c_void_p]
        L.ref_viterbi_block.restype = C.c_size_t
        L.ref_viterbi_block.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_uint32, C.c_void_p]
        L.ref_viterbi_debug.argtypes = [C.c_void_p]
        _REF_VIT = L
    return _REF_VIT
def ref_viterbi_sig11(soft48):
    """oracle/_ref/libviterbi_ref.so: the reference's own Viterbi_sig11 (viterbicore.h) on 48 soft values, >> 6 as T11aViterbiSig does."""
    s = np.ascontiguousarray(soft48, dtype=np.uint8); assert s.shape == (48,)
    return int(_ref_vit().ref_viterbi_sig11(s.ctypes.data))
def ref_viterbi_block(inst, soft, code_rate, frame_len, debug=False):
    """oracle/_ref/libviterbi_ref.so: the reference's own T11aViterbi<...>::Filter (viterbi.hpp), fresh context, fed len(soft) / N_INPUT
    bursts.  inst picks the instantiation (REF_VITERBI_INSTS).  Returns the bytes it emitted; with debug=True also (max_min, max_any):
    the largest unwrapped minimum Normalize subtracted and the largest unwrapped metric of any state at a normalisation (> 255: wrapped)."""
    s = np.ascontiguousarray(soft, dtype=np.uint8).ravel()
    out = np.zeros(frame_len + 2 + 64, np.uint8)
    n = _ref_vit().ref_viterbi_block(inst, s.ctypes.data, len(s), code_rate, frame_len, out.ctypes.data)
    assert n != C.c_size_t(-1).value, "nsoft must be a multiple of N_INPUT and stay within TRELLIS_MAX trellis columns"
    if not debug: return out[:n].copy()
    d = np.zeros(2, np.uint32); _ref_vit().ref_viterbi_debug(d.ctypes.data)
    return out[:n].copy(), (int(d[0]), int(d[1]))

_REF_FFT = None
REF_FFT_COUNTERS = ("sat_add", "sat_sub", "pack", "madd")   # the order of ref_fft_debug's counts
def ref_fft_available():
    return os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libfft_ref.so"))
def _ref_fft():
    global _REF_FFT
    if _REF_FFT is None:
        L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libfft_ref.so"))
        for f in (L.ref_fft64, L.ref_ifft64, L.ref_ifft128): f.argtypes = [C.c_size_t, C.c_void_p, C.c_void_p]; f.restype = None
        L.ref_fft_debug.argtypes = [C.c_void_p]; L.ref_fft_debug.restype = None
        _REF_FFT = L
    return _REF_FFT
def _ref_xform(fn, x, N):
    x = np.ascontiguousarray(x, dtype=np.int16); assert x.shape[-2:] == (N, 2), x.shape
    o = np.zeros_like(x); fn(x.size // (2 * N), x.ctypes.data, o.ctypes.data); return o
def ref_fft64(x):
    """oracle/_ref/libfft_ref.so: the reference's own FFTSafe<64> (fft_r4dif.h) on int16 [..., 64, 2], one transform per vector."""
    return _ref_xform(_ref_fft().ref_fft64, x, 64)
def ref_ifft64(x):
    """The reference's own IFFTSafe<64> (ifft_r4dif.h) on int16 [..., 64, 2]."""
    return _ref_xform(_ref_fft().ref_ifft64, x, 64)
def ref_ifft128(x):
    """The reference's own IFFTSafe<128> (ifft_r4dif.h) on int16 [..., 128, 2]."""
    return _ref_xform(_ref_fft().ref_ifft128, x, 128)
def ref_fft_debug():
    """What the tap counted over the last ref_fft64 / ref_ifft64 / ref_ifft128 call of this thread, as {name: lanes} (REF_FFT_COUNTERS):
    saturated_add / saturated_sub lanes that clipped, pack lanes whose 32-bit value did not fit int16, pmaddwd lanes that wrapped."""
    d = np.zeros(4, np.uint64); _ref_fft().ref_fft_debug(d.ctypes.data)
    return dict(zip(REF_FFT_COUNTERS, (int(v) for v in d)))

# ---- oracle/_ref/librx11a_ref.so: the reference's own 802.11a front-end bricks (oracle/build_ref_rx11a.sh) ----
_REF_RX = None
REF_RX11A_COUNTERS = ("lts_e0", "lts_pack", "eq_pack", "mul_pack", "demap_clamp", "madd")   # the order of ref_rx11a_debug's counts
def ref_rx11a_available():
    return os.path.exists(os.path.join(ROOT, "oracle", "_ref", "librx11a_ref.so"))
def _ref_rx():
    global _REF_RX
    if _REF_RX is None:
        L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "librx11a_ref.so"))
        L.ref_rx11a_lts.argtypes = [C.c_void_p] * 4; L.ref_rx11a_lts.restype = None
        L.ref_rx11a_symbols.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint] + [C.c_void_p] * 11; L.ref_rx11a_symbols.restype = C.c_int
        L.ref_resample_44_40.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]; L.ref_resample_44_40.restype = C.c_size_t
        L.ref_rx11a_debug.argtypes = [C.c_void_p]; L.ref_rx11a_debug.restype = None
        _REF_RX = L
    return _REF_RX
def ref_rx11a_lts(lts144):
    """T11aLTS (channel_11a.hpp) on the 144 samples int16 [144, 2] it is handed, fresh context: (CFO_est, FreqCoeffs, ChannelCoeffs)."""
    x = np.ascontiguousarray(lts144, np.int16).reshape(144, 2)
    cfo = np.zeros(1, np.int16); fc = np.zeros((64, 2), np.int16); cc = np.zeros((64, 2), np.int16)
    _ref_rx().ref_rx11a_lts(_p(x), _p(cfo), _p(fc), _p(cc))
    return int(cfo[0]), fc, cc
def ref_rx11a_symbols(lts144, sym80, rate_kbps):
    """T11aLTS on lts144, then the 80-sample blocks sym80 int16 [n, 80, 2] through the reference's own per-symbol bricks; symbol 0 is
    SIGNAL.  Returns a dict of every intermediate (see ref_rx11a_symbols in oracle/build_ref_rx11a.sh); soft and demapped are cut to
    N_CBPS per symbol."""
    x = np.ascontiguousarray(lts144, np.int16).reshape(144, 2); s = np.ascontiguousarray(sym80, np.int16).reshape(-1, 80, 2); n = len(s)
    cfo = np.zeros(1, np.int16); fc = np.zeros((64, 2), np.int16); cc = np.zeros((64, 2), np.int16)
    v = {k: np.zeros((n, 64, 2), np.int16) for k in ("fft_in", "fft_out", "equalized", "phase_comp", "tracked")}
    dm = np.zeros((n, 288), np.uint8); so = np.zeros((n, 288), np.uint8); st = np.zeros((n, 5), np.int32)
    rc = _ref_rx().ref_rx11a_symbols(_p(x), n, _p(s), rate_kbps, _p(cfo), _p(fc), _p(cc), _p(v["fft_in"]), _p(v["fft_out"]),
                                     _p(v["equalized"]), _p(v["phase_comp"]), _p(v["tracked"]), _p(dm), _p(so), _p(st))
    assert rc == 0, rate_kbps
    nb = {6000: 1, 9000: 1, 12000: 2, 18000: 2, 24000: 4, 36000: 4, 48000: 6, 54000: 6}[rate_kbps]
    ncb = [48] + [48 * nb] * (n - 1)
    v.update(cfo_est=int(cfo[0]), freq_coeffs=fc, chan_coeffs=cc, state=st, ncbps=ncb,
             demapped=[dm[i, :ncb[i]] for i in range(n)], soft=[so[i, :ncb[i]] for i in range(n)])
    return v
def ref_rx11a_debug():
    """What the tap counted over the last ref_rx11a_lts / ref_rx11a_symbols call of this thread, as {name: lanes} (REF_RX11A_COUNTERS)."""
    d = np.zeros(6, np.uint64); _ref_rx().ref_rx11a_debug(d.ctypes.data)
    return dict(zip(REF_RX11A_COUNTERS, (int(v) for v in d)))
def ref_resample_44_40(iq44):
    """TDownSample44_40 / Down44to40 (sampling.hpp, 44MTo40M.hpp) over int16 [n, 2] fed in 28-sample blocks: the 40 Msps samples it emits."""
    x = np.ascontiguousarray(iq44, np.int16).reshape(-1, 2); out = np.zeros_like(x)
    m = _ref_rx().ref_resample_44_40(_p(x), len(x), _p(out))
    return out[:m]
CS_FIELDS = ("cca_state", "error_code", "dc", "cca_peak_index", "cca_pwr_reading", "vec20")   # a carrier-sense record: 13 int32
def rx11a_cs_trace(iq, max_vec=1 << 20):
    """The oracle's carrier sense up to the first frame event: (records int32 [n, 13], index of the first vector past the detection or -1)."""
    iq = np.ascontiguousarray(iq, np.int16); rec = np.zeros((max_vec, 13), np.int32); det = np.zeros(1, np.int64)
    L = lib(); L.sbo_rx11a_cs_trace.restype = C.c_uint64
    n = L.sbo_rx11a_cs_trace(_p(iq), C.c_uint64(iq.shape[0]), _p(rec), C.c_uint64(max_vec), _p(det))
    return rec[:n], int(det[0])
def ref_rx11a_carrier_sense(iq, cca_pwr_threshold=1000 * 1000, max_vec=1 << 20):
    """TDownSample2 -> TDCRemoveEx<4> -> TCCA11a -> TDCEstimator of the reference (oracle/build_ref_rx11a.sh) over 40 Msps int16 [n, 2]:
    the same records as rx11a_cs_trace, and the detection index."""
    iq = np.ascontiguousarray(iq, np.int16); rec = np.zeros((max_vec, 13), np.int32); det = np.zeros(1, np.int64)
    L = _ref_rx(); L.ref_rx11a_carrier_sense.restype = C.c_size_t
    L.ref_rx11a_carrier_sense.argtypes = [C.c_void_p, C.c_size_t, C.c_uint, C.c_void_p, C.c_size_t, C.c_void_p]
    n = L.ref_rx11a_carrier_sense(_p(iq), len(iq), cca_pwr_threshold, _p(rec), max_vec, _p(det))
    return rec[:n], int(det[0])

# ---- the header parsers and the descrambler / frame sink alone: the oracle's, and the reference's own (oracle/build_ref_rx11n.sh) ----
PLCP11A_FIELDS = ("accepted", "error_code", "rate_kbps", "frame_length", "total_symbols", "code_rate")
SIG11N_FIELDS = PLCP11A_FIELDS + ("ht_mcs", "ht_length")
def _parse_words(fn, words):
    w = np.ascontiguousarray(words, np.uint32).reshape(-1); out = np.zeros((len(w), 6), np.uint32)
    fn(_p(w), C.c_uint64(len(w)), _p(out)); return out
def _parse_sig9(fn, sig9):
    s = np.ascontiguousarray(sig9, np.uint8).reshape(-1, 9); out = np.zeros((len(s), 8), np.uint32)
    fn(_p(s), C.c_uint64(len(s)), _p(out)); return out
def plcp11a_parse(words):
    """The oracle's 802.11a SIGNAL parse on each word, from a context just reset: uint32 [n, 6] (PLCP11A_FIELDS)."""
    return _parse_words(lib().sbo_plcp11a_parse, words)
def sig11n_parse(sig9):
    """The oracle's L-SIG + HT-SIG parse on uint8 [n, 9] blocks in turn, one context (the HT fields carry over): uint32 [n, 8] (SIG11N_FIELDS)."""
    return _parse_sig9(lib().sbo_sig11n_parse, sig9)
def desc_sink(chain, decoded, frame_length):
    """The oracle's descrambler and frame sink of the 802.11a (chain 0) or 802.11n (chain 1) receiver, fed the decoded bytes of a frame of
    frame_length bytes: (error code, CF_11aRxVector::crc32, the frame buffer's first frame_length bytes)."""
    d = np.ascontiguousarray(decoded, np.uint8); out = np.zeros(frame_length, np.uint8); crc = np.zeros(1, np.uint32)
    L = lib(); L.sbo_desc_sink.restype = C.c_uint32
    e = L.sbo_desc_sink(C.c_int(chain), _p(d), C.c_uint64(len(d)), C.c_uint16(frame_length), _p(out), _p(crc))
    return int(e), int(crc[0]), out

_REF_RX11N = None
REF_RX11N_COUNTERS = ("lsig_reserved", "lsig_parity", "lsig_rate", "lsig_length", "htsig_crc8", "htsig_mcs", "htsig_length", "accepted",
                      "fcs_ok", "fcs_fail")   # the order of ref_rx11n_debug's counts
def ref_rx11n_available():
    return os.path.exists(os.path.join(ROOT, "oracle", "_ref", "librx11n_ref.so"))
def _ref_rx11n():
    global _REF_RX11N
    if _REF_RX11N is None:
        L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "librx11n_ref.so"))
        L.ref_plcp11a_parse.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]; L.ref_plcp11a_parse.restype = None
        L.ref_sig11n_parse.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]; L.ref_sig11n_parse.restype = None
        L.ref_desc_sink.argtypes = [C.c_void_p, C.c_size_t, C.c_uint16, C.c_void_p, C.c_void_p]; L.ref_desc_sink.restype = C.c_uint32
        L.ref_rx11n_debug.argtypes = [C.c_void_p]; L.ref_rx11n_debug.restype = None
        L.ref_rx11n_debug_reset.argtypes = []; L.ref_rx11n_debug_reset.restype = None
        _REF_RX11N = L
    return _REF_RX11N
def ref_plcp11a_parse(words):
    """T11aPLCPParser (PHY_11a.hpp) on each word, from a context just Reset: uint32 [n, 6] (PLCP11A_FIELDS)."""
    return _parse_words(_ref_rx11n().ref_plcp11a_parse, words)
def ref_sig11n_parse(sig9):
    """T11nSigParser (PHY_11n.hpp) on uint8 [n, 9] blocks in turn, one context: uint32 [n, 8] (SIG11N_FIELDS)."""
    return _parse_sig9(_ref_rx11n().ref_sig11n_parse, sig9)
def ref_desc_sink(decoded, frame_length):
    """T11aDesc -> TBB11aFrameSink (scramble.hpp, PHY_11a.hpp), fresh, fed the decoded bytes: (error code, crc32, frame bytes)."""
    d = np.ascontiguousarray(decoded, np.uint8); out = np.zeros(max(frame_length, 1), np.uint8); crc = np.zeros(1, np.uint32)
    e = _ref_rx11n().ref_desc_sink(_p(d), len(d), frame_length, _p(out), _p(crc))
    return int(e), int(crc[0]), out[:frame_length]
def ref_rx11n_debug_reset():
    _ref_rx11n().ref_rx11n_debug_reset()
def ref_rx11n_debug():
    """What the tap counted since the last ref_rx11n_debug_reset on this thread, as {name: count} (REF_RX11N_COUNTERS)."""
    d = np.zeros(10, np.uint64); _ref_rx11n().ref_rx11n_debug(d.ctypes.data)
    return dict(zip(REF_RX11N_COUNTERS, (int(v) for v in d)))

# ---- the reference's own 802.11b receiver bricks and graph (oracle/build_ref_rx11b.sh) ----
_REF_RX11B = None
REF_RX11B_COUNTERS = ("cck_int_min", "cck_tie", "dqpsk_re_wrap", "dqpsk_sum_wrap", "sfd_found", "sfd_fail", "sfd_timeout", "sync_timeout",
                      "plcp_crc16", "plcp_unknown_rate", "plcp_short_length", "fcs_ok", "fcs_fail", "cs_timeout")   # ref_rx11b_debug's order
def ref_rx11b_available():
    return os.path.exists(os.path.join(ROOT, "oracle", "_ref", "librx11b_ref.so"))
def _ref_rx11b():
    global _REF_RX11B
    if _REF_RX11B is None:
        L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "librx11b_ref.so"))
        for f in ("ref_cck11_decode", "ref_cck5_decode", "ref_dqpsk_demap", "ref_dbpsk_demap"):
            getattr(L, f).argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]; getattr(L, f).restype = None
        L.ref_despread.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]; L.ref_despread.restype = None
        L.ref_plcp11b_parse.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]; L.ref_plcp11b_parse.restype = None
        L.ref_desc_sink.argtypes = [C.c_void_p, C.c_size_t, C.c_uint8, C.c_uint16, C.c_void_p, C.c_void_p]; L.ref_desc_sink.restype = C.c_uint32
        L.ref_rx11b_run.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]; L.ref_rx11b_run.restype = C.c_int
        L.ref_rx11b_debug.argtypes = [C.c_void_p]; L.ref_rx11b_debug.restype = None
        L.ref_rx11b_debug_reset.argtypes = []; L.ref_rx11b_debug_reset.restype = None
        _REF_RX11B = L
    return _REF_RX11B
def _ref_decode(fn, x, per, last):
    x = np.ascontiguousarray(x, np.int16).reshape(-1, per, 2); out = np.zeros(len(x), np.uint8)
    l = np.ascontiguousarray(last, np.int16).reshape(2); lo = np.zeros(2, np.int16)
    getattr(_ref_rx11b(), fn)(_p(x), len(x), _p(l), _p(out), _p(lo)); return out, lo
def ref_cck11_decode(chips, last=(0, 0)):
    """TCCK11Decoder (cck.hpp), one instance, on int16 [n, 8, 2] symbols: (bytes [n], last_symbol after)."""
    return _ref_decode("ref_cck11_decode", chips, 8, last)
def ref_cck5_decode(chips, last=(0, 0)):
    """TCCK5P5Decoder (cck.hpp) on int16 [n, 16, 2]: (bytes [n], last_symbol after)."""
    return _ref_decode("ref_cck5_decode", chips, 16, last)
def ref_dqpsk_demap(sym, last=(0, 0)):
    """TDQPSKDemap (barkerspread.hpp) on int16 [n, 4, 2] symbols: (bytes [n], last_symbol after)."""
    return _ref_decode("ref_dqpsk_demap", sym, 4, last)
def ref_dbpsk_demap(sym, last=(0, 0)):
    """TDBPSKDemap (barkerspread.hpp) on int16 [n, 8, 2] symbols: (bytes [n], last_symbol after)."""
    return _ref_decode("ref_dbpsk_demap", sym, 8, last)
def ref_despread(chips):
    """TBB11bDespread (barkerspread.hpp) on int16 [n, 11, 2] chips: int16 [n, 2] symbols."""
    x = np.ascontiguousarray(chips, np.int16).reshape(-1, 11, 2); out = np.zeros((len(x), 2), np.int16)
    _ref_rx11b().ref_despread(_p(x), len(x), _p(out)); return out
PLCP11B_FIELDS = ("error_code", "plcp_state", "rxrate_state", "rate_kbps", "frame_length")
def ref_plcp11b_parse(hdr6, prev=(0, 0, 0)):
    """TBB11bPlcpParser (PHY_11b.hpp) on uint8 [n, 6] headers in turn through one context (CF_11bRxVector and CF_11bRxMRSel carry over
    from `prev` = (rxrate_state, rate_kbps, frame_length)): uint32 [n, 5] (PLCP11B_FIELDS)."""
    h = np.ascontiguousarray(hdr6, np.uint8).reshape(-1, 6); out = np.zeros((len(h), 5), np.uint32); pv = np.asarray(prev, np.uint32)
    _ref_rx11b().ref_plcp11b_parse(_p(h), len(h), _p(pv), _p(out)); return out
def ref_desc_sink11b(scrambled, seed, frame_length):
    """TDesc741 -> TBB11bFrameSink (scramble.hpp, PHY_11b.hpp), fresh, byte_reg = seed: (error code, crc32 low 24 bits, frame bytes)."""
    d = np.ascontiguousarray(scrambled, np.uint8); out = np.zeros(max(frame_length, 1), np.uint8); crc = np.zeros(1, np.uint32)
    e = _ref_rx11b().ref_desc_sink(_p(d), len(d), seed, frame_length, _p(out), _p(crc))
    return int(e), int(crc[0]), out[:frame_length]
def ref_rx11b_run(iq, max_frames=8, out_stride=4096):
    """CreateDemodGraph driven as MAC11b_Receive drives it, on one 44 Msps capture: (RES11B_DTYPE events, bytes [ne, out_stride])."""
    iq = np.ascontiguousarray(iq, np.int16).reshape(-1, 2)
    res = np.zeros(max_frames, dtype=RES11B_DTYPE); out = np.zeros((max_frames, out_stride), np.uint8)
    n = _ref_rx11b().ref_rx11b_run(_p(iq), iq.shape[0], _p(res), _p(out), out_stride, max_frames)
    return res[:n], out[:n]
def ref_rx11b_batch(iq, off, length, out_stride=4096):
    """ref_rx11b_run on each slot, first event only, shaped like rx11b_batch (a slot without an event reports E_NO_FRAME)."""
    iq = np.ascontiguousarray(iq, np.int16).reshape(-1, 2)
    res = np.zeros(len(off), dtype=RES11B_DTYPE); out = np.zeros((len(off), out_stride), np.uint8); res["status"] = E_NO_FRAME
    for i, (o, n) in enumerate(zip(off, length)):
        r, b = ref_rx11b_run(iq[int(o):int(o) + int(n)], 1, out_stride)
        if len(r): res[i] = r[0]; out[i] = b[0]
    return res, out
def ref_rx11b_debug_reset():
    _ref_rx11b().ref_rx11b_debug_reset()
def ref_rx11b_debug():
    """What the tap counted since the last ref_rx11b_debug_reset on this thread, as {name: count} (REF_RX11B_COUNTERS)."""
    d = np.zeros(len(REF_RX11B_COUNTERS), np.uint64); _ref_rx11b().ref_rx11b_debug(d.ctypes.data)
    return dict(zip(REF_RX11B_COUNTERS, (int(v) for v in d)))
def _cck_n(fn, x, per, last):
    x = np.ascontiguousarray(x, np.int16).reshape(-1, per, 2); out = np.zeros(len(x), np.uint8); l = np.array(last, np.int16).reshape(2).copy()
    fn(_p(x), C.c_uint64(len(x)), _p(l), _p(out)); return out, l
def cck11_decode_n(chips, last=(0, 0)):
    """The oracle's CCK-11 decoder on int16 [n, 8, 2] symbols in turn (is_even from 0): (bytes [n], last_symbol after)."""
    return _cck_n(lib().sbo_cck11_decode_n, chips, 8, last)
def dbpsk_demap_n(sym, last=(0, 0)):
    """The oracle's DBPSK demapper on int16 [n, 8, 2] symbols in turn: (bytes [n], last_symbol after)."""
    return _cck_n(lib().sbo_dbpsk_demap_n, sym, 8, last)
def dqpsk_demap_n(sym, last=(0, 0)):
    """The oracle's DQPSK demapper on int16 [n, 4, 2] symbols in turn: (bytes [n], last_symbol after)."""
    return _cck_n(lib().sbo_dqpsk_demap_n, sym, 4, last)
def despread_n(chips):
    """The oracle's Barker despreader on int16 [n, 11, 2] chips: int16 [n, 2] symbols."""
    x = np.ascontiguousarray(chips, np.int16).reshape(-1, 11, 2); out = np.zeros((len(x), 2), np.int16)
    lib().sbo_despread_n(_p(x), C.c_uint64(len(x)), _p(out)); return out
def cck5_decode_n(chips, last=(0, 0)):
    """The oracle's CCK-5.5 decoder on int16 [n, 16, 2] bytes in turn: (bytes [n], last_symbol after)."""
    return _cck_n(lib().sbo_cck5_decode_n, chips, 16, last)


# ---- oracle/_ref/libmod_ref.so: the reference's own 802.11a brick modulator (oracle/build_ref_mod.sh) ----
_REF_MOD = None
REF_MOD_COUNTERS = ("pack_saturated", "pad_9m_pair", "nsym_over_standard")
def ref_mod_available():
    return os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libmod_ref.so"))
def _ref_mod():
    global _REF_MOD
    if _REF_MOD is None:
        L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libmod_ref.so"))
        L.ref_mod11a_frame.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint8, C.c_void_p, C.c_size_t]; L.ref_mod11a_frame.restype = C.c_int64
        L.ref_mod11a_scramble.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint8, C.c_void_p]; L.ref_mod11a_scramble.restype = None
        L.ref_mod11a_encode.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]; L.ref_mod11a_encode.restype = C.c_size_t
        L.ref_mod11a_interleave.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]; L.ref_mod11a_interleave.restype = None
        L.ref_mod11a_map.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]; L.ref_mod11a_map.restype = C.c_size_t
        for f in ("ref_mod11a_add_pilot", "ref_mod11a_ifftx", "ref_pack16to8"):
            getattr(L, f).argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]; getattr(L, f).restype = None
        L.ref_mod_debug.argtypes = [C.c_void_p]; L.ref_mod_debug.restype = None
        L.ref_mod_debug_reset.argtypes = []; L.ref_mod_debug_reset.restype = None
        _REF_MOD = L
    return _REF_MOD
def ref_mod11a_frame(payload, rate_kbps, seed=0xFF):
    """CreatePreamble11a_40M then CreateModGraph11a_40M, driven as Test11A_FB_Mod drives them, with sc_seed = seed: int8 [n, 2] at 40 Msps
    (what TModSink wrote: preamble, SIGNAL and DATA, no trailing zeros)."""
    p = np.ascontiguousarray(payload, np.uint8)
    # room for the preamble, SIGNAL, the standard's N_SYM and two symbols more: the reference pads to at most a 9 Mbps symbol pair and
    # counts the tail as a whole byte, one symbol each at most.  The library sizes its own buffer the same way and reports how many
    # samples it wrote, so a graph that wrote more would fail the assert below rather than be cut short.
    std_nsym = -(-(16 + 8 * (len(p) + 4) + 6) // (rate_kbps // 250))
    cap = 640 + 160 * (1 + std_nsym + 2); out = np.zeros((cap, 2), np.int8)
    n = _ref_mod().ref_mod11a_frame(_p(p), len(p), rate_kbps, seed, _p(out), cap)
    assert 0 < n <= cap, (n, cap)
    return out[:n]
def ref_mod11a_scramble(data, ctrl, seed):
    """T11aSc, fresh, sc_seed = seed, on uint8 [n] with the scramble_ctrl ctrl[i] (0 none, 1 scramble, 2 tail) in force for byte i."""
    d = np.ascontiguousarray(data, np.uint8); c = np.ascontiguousarray(np.broadcast_to(ctrl, d.shape), np.uint8); out = np.zeros_like(d)
    _ref_mod().ref_mod11a_scramble(_p(d), _p(c), len(d), seed, _p(out))
    return out
def ref_mod11a_encode(cr, data):
    """TConvEncode_12 (cr 0), _23 (1), _34 (2), fresh, on uint8 [n] (whole input bursts of 1, 2, 3 bytes): the coded bytes."""
    d = np.ascontiguousarray(data, np.uint8); out = np.zeros(2 * len(d) + 8, np.uint8)
    m = _ref_mod().ref_mod11a_encode(cr, _p(d), len(d), _p(out)); return out[:m]
def ref_mod11a_interleave(nbpsc, data):
    """T11aInterleave{BPSK,QPSK,QAM16,QAM64} on uint8 [nsym, 6 * nbpsc] (coded bits packed LSB first)."""
    d = np.ascontiguousarray(data, np.uint8).reshape(-1, 6 * nbpsc); out = np.zeros_like(d)
    _ref_mod().ref_mod11a_interleave(nbpsc, _p(d), len(d), _p(out)); return out
def ref_mod11a_map(nbpsc, data):
    """TMap11a{BPSK,QPSK,QAM16,QAM64}<> on uint8 input bursts (1 byte; 3 bytes at QAM64): int16 [m, 2] constellation points."""
    d = np.ascontiguousarray(data, np.uint8); per = 3 if nbpsc == 6 else 1; out = np.zeros((8 * len(d), 2), np.int16)
    m = _ref_mod().ref_mod11a_map(nbpsc, _p(d), len(d) // per, _p(out)); return out[:m]
def ref_mod11a_add_pilot(data48):
    """T11aAddPilot<>, fresh (pilot index 127 first), on int16 [nsym, 48, 2]: int16 [nsym, 64, 2]."""
    d = np.ascontiguousarray(data48, np.int16).reshape(-1, 48, 2); out = np.zeros((len(d), 64, 2), np.int16)
    _ref_mod().ref_mod11a_add_pilot(_p(d), len(d), _p(out)); return out
def ref_mod11a_ifftx(spec64):
    """TIFFTx on int16 [nsym, 64, 2] spectra: int16 [nsym, 160, 2] (32-sample GI, windowed)."""
    d = np.ascontiguousarray(spec64, np.int16).reshape(-1, 64, 2); out = np.zeros((len(d), 160, 2), np.int16)
    _ref_mod().ref_mod11a_ifftx(_p(d), len(d), _p(out)); return out
def ref_pack16to8(x):
    """TPackSample16to8 on int16 [8 n, 2]: int8 [8 n, 2]."""
    d = np.ascontiguousarray(x, np.int16).reshape(-1, 8, 2); out = np.zeros((len(d) * 8, 2), np.int8)
    _ref_mod().ref_pack16to8(_p(d), len(d), _p(out)); return out
def ref_mod_debug_reset():
    _ref_mod().ref_mod_debug_reset()
def ref_mod_debug():
    """What the tap counted since the last ref_mod_debug_reset on this thread, as {name: count} (REF_MOD_COUNTERS)."""
    d = np.zeros(len(REF_MOD_COUNTERS), np.uint64); _ref_mod().ref_mod_debug(d.ctypes.data)
    return dict(zip(REF_MOD_COUNTERS, (int(v) for v in d)))
