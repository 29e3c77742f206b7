"""The legacy 802.11a transmitter at 40 and 44 Msps (BB11ATxFrameMod / BB11AModulateACK) — TEST INFRASTRUCTURE.

- `modulate` binds `sbo_tx11a_legacy_modulate_ex` (oracle/tx11a_legacy44.cpp, built into oracle/libsora_oracle_tx11a44.so by
  oracle/tx11a_legacy44.mk): the whole transmitter, RCB padding included.
- `up160` / `up3` bind its SSE restatement of the 40 -> 44 Msps upsampler (Upsample40MTo44M_160 / _3, upsample.h:44-144).
- `up160_numpy` / `up3_numpy` are a second, scalar reading of the same code: every output is at most two rounded Q15 products of
  neighbouring inputs, summed with a 16-bit wrap.
- `ref_up160` / `ref_up3` drive the reference's own upsampler body where oracle/build_ref_tx11a44.sh could compile it (oracle/_ref).
- `ref_modulate`, `ref_frame_mod_raw`, `ref_ack` drive the reference's own BB11ATxFrameMod / BB11AModulateACK as a whole, where
  oracle/build_ref_tx11a_legacy.sh could compile them (oracle/_ref/libtx11a_legacy_ref.so), with `ref_preamble`, `ref_set_pad` and the
  debug tap `ref_debug`.
"""
import ctypes as C, os, subprocess, zlib
import numpy as np
import oracle_py

ROOT = oracle_py.ROOT
ORACLE = os.path.join(ROOT, "oracle")
SO = os.path.join(ORACLE, "libsora_oracle_tx11a44.so")
PREAMBLE = os.path.join(ROOT, "tests", "golden", "preamble40_11a.i16")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libupsample44_ref.so")
RATES = [6000, 9000, 12000, 18000, 24000, 36000, 48000, 54000]
NDBPS = {6000: 24, 9000: 36, 12000: 48, 18000: 72, 24000: 96, 36000: 144, 48000: 192, 54000: 216}
CODE = {6000: 0xB, 9000: 0xF, 12000: 0xA, 18000: 0xE, 24000: 0x9, 36000: 0xD, 48000: 0x8, 54000: 0xC}


_LIB = None
def lib():
    """oracle/libsora_oracle_tx11a44.so, (re)built first when one of its sources is newer (one process builds, the others wait)."""
    global _LIB
    if _LIB is None:
        srcs = [os.path.join(ORACLE, f) for f in ("tx11a_legacy44.mk", "tx11a_legacy44.cpp", "tables.cpp", "tx11a.cpp", "ops.h", "tables.h", "tx11a.h", "rx11a.h", "viterbi.h")]
        stale = lambda: not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in srcs)
        if stale():
            import fcntl
            with open(os.path.join(ORACLE, ".build.lock"), "w") as lk:
                fcntl.flock(lk, fcntl.LOCK_EX)
                try:
                    if stale(): subprocess.check_call(["make", "-C", ORACLE, "-f", "tx11a_legacy44.mk"], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
                finally: fcntl.flock(lk, fcntl.LOCK_UN)
        _LIB = C.CDLL(SO)
        _LIB.sbo_tx11a_legacy_modulate_ex.restype = C.c_uint64
    return _LIB


def preamble():
    """The 640 COMPLEX16 samples of PREAMBLE40_11A_LUT, int16 [640, 2]."""
    return np.fromfile(PREAMBLE, np.int16).reshape(640, 2)


def nsym(psdu_len, rate_kbps):
    return (16 + 6 + 8 * psdu_len + NDBPS[rate_kbps] - 1) // NDBPS[rate_kbps]


def signal_samples(psdu_len, rate_kbps, sample_rate):
    """GetSignalBytes / 2 (atx_tpl.h:69-83): preamble, SIGNAL and data symbols (x 11/10 at 44 Msps) and the 8-sample tail."""
    n = 640 + 160 * (1 + nsym(psdu_len, rate_kbps))
    return (n // 10 * 11 if sample_rate == 44 else n) + 8


def padded_samples(psdu_len, rate_kbps, sample_rate):
    """The signal rounded up to 128 bytes (ALIGN_WITH_RCB_BUFFER_PADDING_ZERO): what SoraPacketSetSignalLength stores, / 2."""
    return (signal_samples(psdu_len, rate_kbps, sample_rate) + 63) // 64 * 64


def modulate(body, rate_kbps, sample_rate=40, append_crc=True, pre=None):
    """MPDU (append_crc) or MPDU + FCS sent as it is -> int8 [padded, 2]: the signal and its RCB zero padding."""
    body = np.ascontiguousarray(body, dtype=np.uint8)
    pre = np.ascontiguousarray(preamble() if pre is None else pre, dtype=np.int16)
    f = lib().sbo_tx11a_legacy_modulate_ex
    cap = padded_samples(len(body) + (4 if append_crc else 0), rate_kbps, sample_rate)
    out = np.full((cap, 2), 0x55, np.int8); sig = C.c_uint64(0)
    n = f(oracle_py._p(body), C.c_uint32(len(body)), C.c_int(1 if append_crc else 0), C.c_uint32(rate_kbps), C.c_uint32(sample_rate),
          oracle_py._p(pre), oracle_py._p(out), C.c_uint64(cap), C.byref(sig))
    assert n == cap, (n, cap)
    return out


def ack_frame(ra):
    """DOT11_MAC_ACK_FRAME as BB11AModulateACK builds it (atx_fe.c:175-186): FC 0xD4 0x00, Duration 0, RA, CRC-32."""
    b = bytes([0xD4, 0x00, 0, 0]) + bytes(ra)
    return np.frombuffer(b + zlib.crc32(b).to_bytes(4, "little"), np.uint8)


def up160(x164):
    """SSE restatement.  x164: int16 [164, 2] (what the reference's loads see: 160 inputs and the vector behind them) -> int16 [176, 2]."""
    x = np.ascontiguousarray(x164, dtype=np.int16); assert x.shape == (164, 2)
    o = np.zeros((176, 2), np.int16); lib().sbo_tx11a_legacy_upsample44_160(oracle_py._p(x), oracle_py._p(o)); return o


def up3(x4):
    x = np.ascontiguousarray(x4, dtype=np.int16); o = np.zeros((4, 2), np.int16)
    lib().sbo_tx11a_legacy_upsample44_3(oracle_py._p(x), oracle_py._p(o)); return o


def _s1(x):
    return x * 0x7FFF // 11                             # S1(x) = short(x * SONE / 11); S1(11) = SONE


def _mulhrs(x, c):
    return (x.astype(np.int64) * c + (1 << 14)) >> 15  # pmulhrsw for c in [0, 32767]: never leaves int16


def _wrap16(v):
    return ((v + 32768) & 0xFFFF) - 32768


def up160_numpy(x164):
    """Output k = 11 h + s of the 176 (h = 0 .. 15): s = 0 -> M(x[10 h], 11); s >= 1 -> M(x[10 h + s - 1], s) + M(x[10 h + s], 11 - s),
    M(x, a) = mulhrs(x, S1(a)).  Output 175 reads x[160], the sample behind the chunk."""
    x = np.asarray(x164, np.int64)
    out = np.zeros((176, 2), np.int64)
    for k in range(176):
        h, s = divmod(k, 11); b = 10 * h
        out[k] = _mulhrs(x[b], _s1(11)) if s == 0 else _wrap16(_mulhrs(x[b + s - 1], _s1(s)) + _mulhrs(x[b + s], _s1(11 - s)))
    return out.astype(np.int16)


def up3_numpy(x4):
    """Upsample40MTo44M_3: the first four outputs of the rule above over the window tail (x[3] = 0)."""
    x = np.asarray(x4, np.int64); out = np.zeros((4, 2), np.int64)
    out[0] = _mulhrs(x[0], _s1(11))
    for s in (1, 2, 3): out[s] = _wrap16(_mulhrs(x[s - 1], _s1(s)) + _mulhrs(x[s], _s1(11 - s)))
    return out.astype(np.int16)


_REF = None
def ref_available():
    return os.path.exists(REF_SO)


def _ref():
    global _REF
    if _REF is None: _REF = C.CDLL(REF_SO)
    return _REF


def ref_up160(x160, in_place_tail=True, behind=None):
    """The reference's Upsample40MTo44M_160, compiled from upsample.h.  With in_place_tail the input lies in a cSymbol[160] that is
    immediately followed by cSymbol44M[177] (BB11A_TX_VECTOR), so the over-read sees the call's own first outputs; otherwise `behind`
    (int16 [4, 2]) is placed after the input."""
    x = np.ascontiguousarray(x160, dtype=np.int16); o = np.zeros((176, 2), np.int16)
    b = np.zeros((4, 2), np.int16) if behind is None else np.ascontiguousarray(behind, dtype=np.int16)
    _ref().ref_upsample44_160(oracle_py._p(x), oracle_py._p(b), C.c_int(1 if in_place_tail else 0), oracle_py._p(o))
    return o


def ref_up3(x4):
    x = np.ascontiguousarray(x4, dtype=np.int16); o = np.zeros((4, 2), np.int16)
    _ref().ref_upsample44_3(oracle_py._p(x), oracle_py._p(o)); return o


# ---- the reference's own transmitter, compiled from atx_*.c by oracle/build_ref_tx11a_legacy.sh -------------------------------------------
REF_TX_SO = os.path.join(ROOT, "oracle", "_ref", "libtx11a_legacy_ref.so")
REF_TX_COUNTERS = ("window_sat", "window_wrap", "pack_sat", "ifft_shl_loss", "ifft_sat")    # the order of ref_tx11a_legacy_debug's counts


class MDL(C.Structure):
    pass
MDL._fields_ = [("Next", C.POINTER(MDL)), ("StartVa", C.c_void_p), ("ByteOffset", C.c_uint32), ("ByteCount", C.c_uint32)]


def ref_tx_available():
    return os.path.exists(REF_TX_SO)


_REFTX = None
def _reftx():
    global _REFTX
    if _REFTX is None:
        L = C.CDLL(REF_TX_SO)
        L.ref_tx11a_legacy_ctx_new.restype = C.c_void_p
        L.ref_tx11a_legacy_ctx_free.argtypes = [C.c_void_p]
        L.ref_tx11a_legacy_frame_mod.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
        L.ref_tx11a_legacy_frame_mod.restype = C.c_int32
        L.ref_tx11a_legacy_ack.argtypes = [C.c_uint, C.c_void_p, C.c_void_p]; L.ref_tx11a_legacy_ack.restype = C.c_uint32
        for f in (L.ref_tx11a_legacy_preamble, L.ref_tx11a_legacy_set_pad, L.ref_tx11a_legacy_debug): f.argtypes = [C.c_void_p]; f.restype = None
        _REFTX = L
    return _REFTX


class RefContext:
    """One BB11A_TX_VECTOR of the compiled transmitter, kept across frames (as BB11ATxContextInit leaves it when made)."""
    def __init__(self): self.p = _reftx().ref_tx11a_legacy_ctx_new()
    def __del__(self):
        if getattr(self, "p", None): _reftx().ref_tx11a_legacy_ctx_free(self.p); self.p = None


def ref_frame_mod_raw(parts, fcs, rate_code, sample_rate, ctx=None, offsets=None, out=None):
    """BB11ATxFrameMod compiled from the reference: the MPDU in MDLs over `parts` (uint8 arrays; StartVa + ByteOffset = the part's first byte,
    ByteOffset = offsets[i]), FCS = Reserved1.  out: uint8 buffer the transmitter writes (default: 0x55 bytes enough for LENGTH 4096).
    Returns (HRESULT, out, SignalLength in bytes)."""
    parts = [np.ascontiguousarray(p, dtype=np.uint8) for p in parts]
    offsets = offsets or [0] * len(parts)
    mdls = [MDL(None, C.c_void_p(p.ctypes.data - o if p.size else 0x1000), o, p.size) for p, o in zip(parts, offsets)]
    for a, b in zip(mdls, mdls[1:]): a.Next = C.pointer(b)
    if out is None: out = np.full(4 * padded_samples(4096, 6000, 44), 0x55, np.uint8)
    sl = C.c_uint32(0)
    hr = _reftx().ref_tx11a_legacy_frame_mod(ctx.p if ctx else None, rate_code, sample_rate, C.addressof(mdls[0]) if mdls else None,
                                             C.c_uint32(fcs), out.ctypes.data, out.size, C.byref(sl))
    return hr, out, sl.value


def ref_modulate(psdu, rate_kbps, sample_rate=40, ctx=None):
    """The compiled transmitter on MPDU + FCS (its last 4 bytes, sent as Reserved1): int8 [SignalLength / 2, 2], what `modulate(..,
    append_crc=False)` returns."""
    psdu = np.ascontiguousarray(psdu, dtype=np.uint8); assert psdu.size >= 4
    hr, out, sl = ref_frame_mod_raw([psdu[:-4]], int.from_bytes(bytes(psdu[-4:]), "little"), CODE[rate_kbps], sample_rate, ctx)
    assert hr == 0 and sl % 128 == 0, (hr, sl)
    assert (out[sl:] == 0x55).all()
    return out[:sl].view(np.int8).reshape(-1, 2)


def ref_ack(ra, sample_rate):
    """BB11AModulateACK compiled from the reference: (return value, uint8 buffer it wrote, pre-filled 0x55)."""
    buf = np.full(2 * padded_samples(14, 6000, 44) + 256, 0x55, np.uint8)
    off = (-buf.ctypes.data) % 16                                       # Copy_NT streams: 16-byte aligned
    r = np.ascontiguousarray(ra, dtype=np.uint8)
    n = _reftx().ref_tx11a_legacy_ack(sample_rate, r.ctypes.data, buf[off:].ctypes.data)
    return n, buf[off:off + 2 * padded_samples(14, 6000, 44) + 128]


def ref_preamble():
    """The compiled PREAMBLE40_11A_LUT (lutst/preamble40_11a.c), int16 [640, 2]."""
    o = np.zeros((640, 2), np.int16); _reftx().ref_tx11a_legacy_preamble(o.ctypes.data); return o


def ref_set_pad(pad):
    """The 8 samples the compiled transmitter reads behind PREAMBLE40_11A_LUT (int16 [8, 2]; zeros unless set)."""
    p = np.ascontiguousarray(pad, dtype=np.int16); assert p.shape == (8, 2); _reftx().ref_tx11a_legacy_set_pad(p.ctypes.data)


def ref_debug_reset():
    _reftx().ref_tx11a_legacy_debug_reset()


def ref_debug():
    """The tap's lane counts since ref_debug_reset, as {name: lanes} (REF_TX_COUNTERS)."""
    d = np.zeros(5, np.uint64); _reftx().ref_tx11a_legacy_debug(d.ctypes.data)
    return dict(zip(REF_TX_COUNTERS, (int(x) for x in d)))
