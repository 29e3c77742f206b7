"""Python binding of the product C ABI (include/sora_b200.h) — thin ctypes, no compute here.

The CUDA library is the only implementation: a missing `libsora_b200.so` or a box without a usable GPU raises.
There is deliberately no CPU fallback (oracle/ is test infrastructure and is never imported from this package).
"""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsora_b200.so")

FRAME_OK, FRAME_FAILED, FRAME_PLCP_FAIL, FRAME_CRC32_FAIL, FRAME_NONE = 1, 0x8000FFFF, 0x80000005, 0x80000006, 0x8000F001
CR_12, CR_23, CR_34 = 0, 1, 2

RESULT_DTYPE = np.dtype([("status", "<u4"), ("rate_kbps", "<u4"), ("length", "<u4"), ("crc32", "<u4"), ("nsym", "<u4"),
                         ("detect_index", "<u4"), ("cfo_est", "<i2"), ("peak_index", "<u2")])

RESULT11B_DTYPE = np.dtype([("status", "<u4"), ("rate_kbps", "<u4"), ("length", "<u4"), ("crc32", "<u4"), ("sample_index", "<u4"), ("detect_vec", "<u4")])

RESULT11N_DTYPE = np.dtype([("status", "<u4"), ("mcs", "<u4"), ("length", "<u4"), ("crc32", "<u4"), ("nsym", "<u4"),
                            ("detect_index", "<u4"), ("cfo_est", "<i2"), ("lsig_length", "<u2")])

EXPORTS = ["sb200_create", "sb200_destroy", "sb200_last_error", "sb200_launch_count", "sb200_last_kernel_ms",
           "sb200_last_kernel_times", "sb200_set_option", "sb200_rx11a_batch", "sb200_rx11a_batch_ex", "sb200_rx11a_stream", "sb200_rx11a_streams", "sb200_rx11b_batch", "sb200_viterbi_k7", "sb200_rx11a_taps",
           "sb200_rx11n_batch", "sb200_rx11n_taps", "sb200_rxblocks_unpack", "sb200_tx11a_batch", "sb200_tx11b_batch", "sb200_rx11b_streams", "sb200_rx11n_streams", "sb200_tx11n_batch", "sb200_rxblocks_desc", "sb200_fir_decimate2", "sb200_channelize", "sb200_tx11b_fir37", "sb200_tx11b_legacy_batch", "sb200_tx11a_legacy_batch", "sb200_host_alloc", "sb200_host_free", "sb200_last_transfer", "sb200_last_viterbi_kernel"]

class Sb200Error(RuntimeError):
    pass

_lib = None
def load_library():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise Sb200Error(f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'` (no CPU fallback exists)")
        lib = C.CDLL(LIB_PATH)
        lib.sb200_create.argtypes = [C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]; lib.sb200_create.restype = C.c_int
        lib.sb200_destroy.argtypes = [C.c_void_p]; lib.sb200_destroy.restype = None
        lib.sb200_last_error.argtypes = [C.c_void_p]; lib.sb200_last_error.restype = C.c_char_p
        lib.sb200_launch_count.argtypes = [C.c_void_p]; lib.sb200_launch_count.restype = C.c_uint64
        lib.sb200_last_kernel_ms.argtypes = [C.c_void_p]; lib.sb200_last_kernel_ms.restype = C.c_float
        lib.sb200_last_kernel_times.argtypes = [C.c_void_p, C.c_void_p]; lib.sb200_last_kernel_times.restype = C.c_int
        lib.sb200_last_viterbi_kernel.argtypes = [C.c_void_p]; lib.sb200_last_viterbi_kernel.restype = C.c_char_p
        lib.sb200_last_transfer.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]; lib.sb200_last_transfer.restype = C.c_int
        lib.sb200_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64]; lib.sb200_set_option.restype = C.c_int
        lib.sb200_rx11a_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32,
                                          C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        lib.sb200_rx11a_batch.restype = C.c_int
        lib.sb200_rx11a_batch_ex.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                             C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        lib.sb200_rx11a_batch_ex.restype = C.c_int
        lib.sb200_rx11a_stream.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.sb200_rx11a_stream.restype = C.c_int
        lib.sb200_rx11b_batch.argtypes = lib.sb200_rx11a_batch.argtypes; lib.sb200_rx11b_batch.restype = C.c_int
        lib.sb200_viterbi_k7.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32,
                                         C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p]
        lib.sb200_viterbi_k7.restype = C.c_int
        lib.sb200_rx11a_taps.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                         C.c_void_p] + [C.c_void_p] * 6 + [C.c_uint64]
        lib.sb200_rx11a_taps.restype = C.c_int
        _lib = lib
    return _lib

def _payload_table(payloads):
    """List of payloads -> (flat uint8 bytes, offsets uint64, lengths uint32); one zero byte stands for an all-empty list."""
    lens = np.array([len(p) for p in payloads], np.uint32); offs = np.concatenate([[0], np.cumsum(lens[:-1])]).astype(np.uint64)
    flat = np.ascontiguousarray(np.concatenate([np.asarray(p, np.uint8) for p in payloads]) if lens.sum() else np.zeros(1, np.uint8))
    return flat, offs, lens

def phase_inc(f_hz, fs_hz):
    """NCO increment of sb200_channelize for a channel centred at f_hz in a capture at fs_hz: round(f / fs * 2^32) mod 2^32 (negative f wraps)."""
    return int(round(f_hz / fs_hz * 2 ** 32)) % 2 ** 32

class DdcChannel(C.Structure):
    _fields_ = [("phase_inc", C.c_uint32), ("phase0", C.c_uint32)]

_NDBPS_11A = {6000: 24, 9000: 36, 12000: 48, 18000: 72, 24000: 96, 36000: 144, 48000: 192, 54000: 216}   # 802.11a data bits per OFDM symbol

def _ptr(a):
    """numpy array -> host pointer; torch tensor / int -> raw (device or pinned) pointer."""
    if a is None:
        return None
    if isinstance(a, int):
        return a
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    if hasattr(a, "data_ptr"):
        return a.data_ptr()
    raise TypeError(type(a))

class Engine:
    """One sb200 handle = one GPU context (BB11aDemodContext analogue: fb11ademod_config.hpp:20-123)."""
    def __init__(self, device=0, cca_pwr_threshold=0):
        lib = load_library()
        cfg = (C.c_uint32 * 8)(cca_pwr_threshold, 0, 0, 0, 0, 0, 0, 0)
        h = C.c_void_p()
        rc = lib.sb200_create(device, C.cast(cfg, C.c_void_p), C.byref(h))
        if rc != 0:
            raise Sb200Error(f"sb200_create(device={device}) failed with {rc} (no CUDA device / no CPU fallback)")
        self._h, self._lib, self.device = h, lib, device

    def close(self):
        if getattr(self, "_h", None):
            self._lib.sb200_destroy(self._h); self._h = None
    __del__ = close

    def _check(self, rc, what):
        if rc != 0:
            raise Sb200Error(f"{what} failed ({rc}): {self._lib.sb200_last_error(self._h).decode()}")

    @property
    def launches(self):
        return int(self._lib.sb200_launch_count(self._h))
    def last_kernel_ms(self):
        return float(self._lib.sb200_last_kernel_ms(self._h))

    def set_option(self, name, value):
        self._check(self._lib.sb200_set_option(self._h, name.encode(), int(value)), "sb200_set_option")

    def last_kernel_times(self):
        t = (C.c_float * 4)()
        self._check(self._lib.sb200_last_kernel_times(self._h, C.cast(t, C.c_void_p)), "sb200_last_kernel_times")
        return [float(x) for x in t]

    def last_viterbi_kernel(self):
        return self._lib.sb200_last_viterbi_kernel(self._h).decode()

    def last_transfer(self):
        """(sample bytes copied host -> device, pipeline chunks, chunks gathered on the host first) of the last host-buffer rx11a call."""
        b = C.c_uint64(0); c = C.c_uint32(0); g = C.c_uint32(0)
        self._check(self._lib.sb200_last_transfer(self._h, C.addressof(b), C.addressof(c), C.addressof(g)), "sb200_last_transfer")
        return int(b.value), int(c.value), int(g.value)

    def rx11a_raw(self, iq_ptr, iq_total, off_ptr, len_ptr, nframes, out_ptr, out_stride, res_ptr, stream=0):
        """Pointer-level call (host or device pointers), used by bench.py with torch buffers."""
        self._check(self._lib.sb200_rx11a_batch(self._h, iq_ptr, iq_total, off_ptr, len_ptr, nframes, out_ptr, out_stride, res_ptr, stream), "sb200_rx11a_batch")

    def rx11a_batch(self, iq, frame_off, frame_len, out_stride=2560, sample_rate_mhz=40):
        """iq: int16 [n,2] numpy; returns (results structured array [F], bytes uint8 [F, out_stride])."""
        iq = np.ascontiguousarray(iq, dtype=np.int16).reshape(-1, 2)
        off = np.ascontiguousarray(frame_off, dtype=np.uint64); ln = np.ascontiguousarray(frame_len, dtype=np.uint32)
        nf = len(off)
        res = np.zeros(nf, dtype=RESULT_DTYPE); out = np.zeros((nf, out_stride), dtype=np.uint8)
        if sample_rate_mhz == 40:
            self.rx11a_raw(_ptr(iq), iq.shape[0], _ptr(off), _ptr(ln), nf, _ptr(out), out_stride, _ptr(res))
        else:
            self._check(self._lib.sb200_rx11a_batch_ex(self._h, _ptr(iq), iq.shape[0], _ptr(off), _ptr(ln), nf, sample_rate_mhz, _ptr(out), out_stride, _ptr(res), 0), "sb200_rx11a_batch_ex")
        return res, out

    def rx11a_stream(self, iq, max_frames=16, out_stride=2560):
        """One continuous capture -> (results [n], bytes [n, out_stride], sample_index [n]) in RxThread order."""
        iq = np.ascontiguousarray(iq, dtype=np.int16).reshape(-1, 2)
        res = np.zeros(max_frames, dtype=RESULT_DTYPE); out = np.zeros((max_frames, out_stride), dtype=np.uint8)
        sidx = np.zeros(max_frames, np.uint32); n = C.c_uint32(0)
        self._check(self._lib.sb200_rx11a_stream(self._h, _ptr(iq), iq.shape[0], max_frames, _ptr(out), out_stride, _ptr(res), _ptr(sidx), C.addressof(n), 0), "sb200_rx11a_stream")
        return res[:n.value], out[:n.value], sidx[:n.value]

    def rx11a_streams(self, iq, stream_off, stream_len, max_frames=16, out_stride=2560):
        """Many continuous captures -> (results [S, max_frames], bytes [S, max_frames, out_stride], sample_index [S, max_frames], counts [S])."""
        iq = np.ascontiguousarray(iq, dtype=np.int16).reshape(-1, 2)
        off = np.ascontiguousarray(stream_off, dtype=np.uint64); ln = np.ascontiguousarray(stream_len, dtype=np.uint32); S = len(off)
        res = np.zeros((S, max_frames), dtype=RESULT_DTYPE); out = np.zeros((S, max_frames, out_stride), dtype=np.uint8)
        sidx = np.zeros((S, max_frames), np.uint32); cnt = np.zeros(S, np.uint32)
        self._check(self._lib.sb200_rx11a_streams(self._h, C.c_void_p(_ptr(iq)), C.c_uint64(iq.shape[0]), C.c_void_p(_ptr(off)), C.c_void_p(_ptr(ln)), C.c_uint32(S), C.c_uint32(max_frames),
                                                  C.c_void_p(_ptr(out)), C.c_uint32(out_stride), C.c_void_p(_ptr(res)), C.c_void_p(_ptr(sidx)), C.c_void_p(_ptr(cnt)), C.c_void_p(0)), "sb200_rx11a_streams")
        return res, out, sidx, cnt

    def rx11b_raw(self, iq_ptr, iq_total, off_ptr, len_ptr, nframes, out_ptr, out_stride, res_ptr, stream=0):
        self._check(self._lib.sb200_rx11b_batch(self._h, iq_ptr, iq_total, off_ptr, len_ptr, nframes, out_ptr, out_stride, res_ptr, stream), "sb200_rx11b_batch")

    def tx11a_raw(self, pay_ptr, pay_total, off_ptr, len_ptr, seed_ptr, nframes, rate_kbps, lead, bits, out_ptr, out_stride, ns_ptr, stream=0):
        self._check(self._lib.sb200_tx11a_batch(self._h, C.c_void_p(pay_ptr), C.c_uint64(pay_total), C.c_void_p(off_ptr), C.c_void_p(len_ptr), C.c_void_p(seed_ptr),
                                                C.c_uint32(nframes), C.c_uint32(rate_kbps), C.c_uint32(lead), C.c_uint32(bits), C.c_void_p(out_ptr), C.c_uint64(out_stride),
                                                C.c_void_p(ns_ptr), C.c_void_p(stream)), "sb200_tx11a_batch")

    def tx11a_batch(self, payloads, rate_kbps, seeds=None, lead=0, sample_bits=8, out_stride=None):
        """payloads: list of uint8 arrays (MPDUs without FCS) -> (samples [F, out_stride, 2] int8 or int16, nsamples [F])."""
        flat, offs, lens = _payload_table(payloads)
        from math import ceil
        if out_stride is None:
            nd = _NDBPS_11A[rate_kbps]
            out_stride = lead + 640 + 160 * (2 + ceil((int(lens.max()) + 7) * 8 / nd) + 1) + 32
        out = np.zeros((len(lens), out_stride, 2), np.int8 if sample_bits == 8 else np.int16); ns = np.zeros(len(lens), np.uint32)
        sd = None if seeds is None else np.ascontiguousarray(seeds, dtype=np.uint8)
        self.tx11a_raw(_ptr(flat), flat.size, _ptr(offs), _ptr(lens), 0 if sd is None else _ptr(sd), len(lens), rate_kbps, lead, sample_bits, _ptr(out), out_stride, _ptr(ns))
        return out, ns

    def tx11n_raw(self, pay_ptr, pay_total, off_ptr, len_ptr, seed_ptr, nframes, mcs, lead, out0_ptr, out1_ptr, out_stride, ns_ptr, stream=0):
        self._check(self._lib.sb200_tx11n_batch(self._h, C.c_void_p(pay_ptr), C.c_uint64(pay_total), C.c_void_p(off_ptr), C.c_void_p(len_ptr), C.c_void_p(seed_ptr), C.c_uint32(nframes),
                                                C.c_uint32(mcs), C.c_uint32(lead), C.c_void_p(out0_ptr), C.c_void_p(out1_ptr), C.c_uint64(out_stride), C.c_void_p(ns_ptr),
                                                C.c_void_p(stream)), "sb200_tx11n_batch")

    def tx11n_batch(self, payloads, mcs, seeds=None, lead=0, out_stride=None):
        """payloads: list of uint8 arrays (MPDUs without FCS) -> (stream 0 [F, out_stride, 2] int16, stream 1, nsamples [F]) at 40 Msps."""
        flat, offs, lens = _payload_table(payloads)
        if out_stride is None:
            nd = {8: 52, 9: 104, 10: 156}.get(mcs, 52)
            out_stride = lead + 1600 + 160 * (-(-((int(lens.max()) + 4) * 8 + 22) // nd) + 1)
        o0 = np.zeros((len(lens), out_stride, 2), np.int16); o1 = np.zeros_like(o0); ns = np.zeros(len(lens), np.uint32)
        sd = None if seeds is None else np.ascontiguousarray(seeds, dtype=np.uint8)
        self.tx11n_raw(_ptr(flat), flat.size, _ptr(offs), _ptr(lens), 0 if sd is None else _ptr(sd), len(lens), mcs, lead, _ptr(o0), _ptr(o1), out_stride, _ptr(ns))
        return o0, o1, ns

    def tx11b_raw(self, pay_ptr, pay_total, off_ptr, len_ptr, nframes, rate_kbps, init_phase, lead, bits, out_ptr, out_stride, ns_ptr, stream=0, fp_ptr=0):
        self._check(self._lib.sb200_tx11b_batch(self._h, C.c_void_p(pay_ptr), C.c_uint64(pay_total), C.c_void_p(off_ptr), C.c_void_p(len_ptr), C.c_uint32(nframes),
                                                C.c_uint32(rate_kbps), C.c_uint32(init_phase), C.c_uint32(lead), C.c_uint32(bits), C.c_void_p(out_ptr),
                                                C.c_uint64(out_stride), C.c_void_p(ns_ptr), C.c_void_p(fp_ptr), C.c_void_p(stream)), "sb200_tx11b_batch")

    def tx11b_batch(self, payloads, rate_kbps, init_phase=0, lead=0, sample_bits=8, out_stride=None, return_phase=False):
        """payloads: list of uint8 arrays (MPDUs without FCS) -> (samples [F, out_stride, 2] int8 or int16 at 44 Msps, nsamples [F])."""
        flat, offs, lens = _payload_table(payloads)
        if out_stride is None:
            cpb = {1000: 88, 2000: 44, 5500: 16, 11000: 8}.get(rate_kbps, 8)      # an unknown rate is the library's error to report
            out_stride = (lead + (24 * 88 + (int(lens.max()) + 4) * cpb + 5) * 4 + 15) // 8 * 8
        out = np.zeros((len(lens), out_stride, 2), np.int8 if sample_bits == 8 else np.int16); ns = np.zeros(len(lens), np.uint32)
        fp = np.zeros(len(lens), np.uint32)
        self.tx11b_raw(_ptr(flat), flat.size, _ptr(offs), _ptr(lens), len(lens), rate_kbps, init_phase, lead, sample_bits, _ptr(out), out_stride, _ptr(ns), 0, _ptr(fp))
        return (out, ns, fp) if return_phase else (out, ns)

    def rxblocks_desc(self, raw):
        """raw: uint8 array of whole 128-byte RX_BLOCKs -> (VStreamBits uint32 [nblocks], TimeStamp uint32 [nblocks])."""
        raw = np.ascontiguousarray(raw, dtype=np.uint8); nblk = len(raw) // 128
        vb = np.zeros(nblk, np.uint32); ts = np.zeros(nblk, np.uint32)
        self._check(self._lib.sb200_rxblocks_desc(self._h, C.c_void_p(_ptr(raw)), C.c_uint64(nblk), C.c_void_p(_ptr(vb)), C.c_void_p(_ptr(ts)), C.c_void_p(0)), "sb200_rxblocks_desc")
        return vb, ts

    def fir_decimate2_raw(self, in_ptr, n_in, taps_ptr, ntaps, out_ptr, stream=0):
        self._check(self._lib.sb200_fir_decimate2(self._h, C.c_void_p(in_ptr), C.c_uint64(n_in), C.c_void_p(taps_ptr), C.c_uint32(ntaps), C.c_void_p(out_ptr), C.c_void_p(stream)), "sb200_fir_decimate2")

    def fir_decimate2(self, iq, taps=None):
        """2:1 anti-alias FIR decimator: int16 [n,2] -> int16 [(n+1)//2, 2]; taps int16 Q15 (odd count <= 63) or None for the built-in half-band."""
        iq = np.ascontiguousarray(iq, dtype=np.int16).reshape(-1, 2)
        out = np.zeros(((len(iq) + 1) // 2, 2), np.int16)
        t = None if taps is None else np.ascontiguousarray(taps, dtype=np.int16)
        self.fir_decimate2_raw(_ptr(iq), len(iq), _ptr(t) if t is not None else 0, 0 if t is None else len(t), _ptr(out))
        return out

    def channelize_raw(self, in_ptr, n_in, channels, decim, taps, out_ptr, out_stride, stream=0):
        """Pointer-level sb200_channelize: in_ptr / out_ptr host or device addresses; channels a list of (phase_inc, phase0); taps int16 Q15."""
        ch = (DdcChannel * max(len(channels), 1))(*[DdcChannel(int(a) % 2 ** 32, int(b) % 2 ** 32) for a, b in channels])
        t = np.ascontiguousarray(taps, dtype=np.int16)
        self._check(self._lib.sb200_channelize(self._h, C.c_void_p(in_ptr), C.c_uint64(n_in), C.cast(ch, C.c_void_p), C.c_uint32(len(channels)), C.c_uint32(decim),
                                               C.c_void_p(_ptr(t)), C.c_uint32(len(t)), C.c_void_p(out_ptr), C.c_uint64(out_stride), C.c_void_p(stream)), "sb200_channelize")

    def channelize(self, iq, channels, decim, taps):
        """Wideband channelizer: int16 [n,2] and K channels (phase_inc, phase0) -> int16 [K, ceil(n / decim), 2], channel k shifted to 0 Hz,
        filtered by taps (int16 Q15, odd count <= 255, sum |t| <= 65535) and decimated."""
        iq = np.ascontiguousarray(iq, dtype=np.int16).reshape(-1, 2)
        n_out = -(-len(iq) // decim); stride = (n_out + 3) // 4 * 4
        out = np.zeros((len(channels), stride, 2), np.int16)
        self.channelize_raw(_ptr(iq), len(iq), channels, decim, taps, _ptr(out), stride)
        return out[:, :n_out]

    def tx11b_fir37_raw(self, in_ptr, total, off_ptr, len_ptr, nframes, variant, out_ptr, stream=0):
        self._check(self._lib.sb200_tx11b_fir37(self._h, C.c_void_p(in_ptr), C.c_uint64(total), C.c_void_p(off_ptr), C.c_void_p(len_ptr), C.c_uint32(nframes),
                                                C.c_uint32(variant), C.c_void_p(out_ptr), C.c_void_p(stream)), "sb200_tx11b_fir37")

    def tx11b_fir37(self, chips, variant=0, frame_len=None):
        """Legacy 37-tap transmit filter.  chips int8 [n, 2] (one frame) or [F, L, 2] (F frames of L samples, L % 8 == 0) -> same shape."""
        x = np.ascontiguousarray(chips, dtype=np.int8)
        fr = x.reshape(1, -1, 2) if x.ndim == 2 else x
        F, L, _ = fr.shape
        off = (np.arange(F, dtype=np.uint64) * L); ln = np.full(F, L if frame_len is None else frame_len, np.uint32)
        out = np.zeros_like(fr)
        self.tx11b_fir37_raw(_ptr(fr), F * L, _ptr(off), _ptr(ln), F, variant, _ptr(out))
        return out.reshape(x.shape)

    TX11B_LEGACY_FCS_IN_PAYLOAD = 1

    def tx11b_legacy_raw(self, pay_ptr, pay_total, off_ptr, len_ptr, nframes, rate_kbps, short_preamble, flags, filt, out_ptr, out_stride, ns_ptr, stream=0):
        self._check(self._lib.sb200_tx11b_legacy_batch(self._h, C.c_void_p(pay_ptr), C.c_uint64(pay_total), C.c_void_p(off_ptr), C.c_void_p(len_ptr), C.c_uint32(nframes),
                                                       C.c_uint32(rate_kbps), C.c_uint32(short_preamble), C.c_uint32(flags), C.c_uint32(filt), C.c_void_p(out_ptr),
                                                       C.c_uint64(out_stride), C.c_void_p(ns_ptr), C.c_void_p(stream)), "sb200_tx11b_legacy_batch")

    def tx11b_legacy_batch(self, payloads, rate_kbps, short_preamble=False, filter=1, fcs_in_payload=False, out_stride=None):
        """The legacy 802.11b transmitter (BB11BPMDBufferTx4X* and, filter 1 / 2, the SSE / ASM 37-tap filter).  payloads: list of uint8 arrays,
        MPDUs without FCS (or with it, fcs_in_payload=True) -> (COMPLEX8 samples int8 [F, out_stride, 2] at 44 Msps, nsamples [F])."""
        flat, offs, lens = _payload_table(payloads)
        if out_stride is None:
            size = int(lens.max()) + (0 if fcs_in_payload else 4)
            cpb = {1000: 0 if short_preamble else 88, 2000: 44, 5500: 16, 11000: 8}.get(rate_kbps, 8)     # an unknown rate is the library's error to report
            out_stride = (4 * ((1056 if short_preamble else 2112) + size * cpb) + 37 + 127) // 128 * 128
        out = np.zeros((len(lens), out_stride, 2), np.int8); ns = np.zeros(len(lens), np.uint32)
        self.tx11b_legacy_raw(_ptr(flat), flat.size, _ptr(offs), _ptr(lens), len(lens), rate_kbps, int(bool(short_preamble)),
                              self.TX11B_LEGACY_FCS_IN_PAYLOAD if fcs_in_payload else 0, filter, _ptr(out), out_stride, _ptr(ns))
        return out, ns

    TX11A_LEGACY_FCS_IN_PAYLOAD = 1

    def tx11a_legacy_raw(self, pay_ptr, pay_total, off_ptr, len_ptr, nframes, rate_kbps, sample_rate_mhz, flags, pre_ptr, out_ptr, out_stride, ns_ptr, stream=0):
        self._check(self._lib.sb200_tx11a_legacy_batch(self._h, C.c_void_p(pay_ptr), C.c_uint64(pay_total), C.c_void_p(off_ptr), C.c_void_p(len_ptr), C.c_uint32(nframes),
                                                       C.c_uint32(rate_kbps), C.c_uint32(sample_rate_mhz), C.c_uint32(flags), C.c_void_p(pre_ptr), C.c_void_p(out_ptr),
                                                       C.c_uint64(out_stride), C.c_void_p(ns_ptr), C.c_void_p(stream)), "sb200_tx11a_legacy_batch")

    @staticmethod
    def tx11a_legacy_nsamples(psdu_len, rate_kbps, sample_rate_mhz=40):
        """Samples BB11ATxFrameMod writes for a PSDU of psdu_len bytes (FCS included): the signal rounded up to 128 bytes."""
        ndbps = _NDBPS_11A.get(rate_kbps, 24)             # an unknown rate is the library's error
        nsym = (22 + 8 * psdu_len + ndbps - 1) // ndbps
        return ((176 if sample_rate_mhz == 44 else 160) * (5 + nsym) + 8 + 63) // 64 * 64

    def tx11a_legacy_batch(self, payloads, rate_kbps, preamble, sample_rate_mhz=40, fcs_in_payload=False, out_stride=None):
        """The legacy 802.11a transmitter (BB11ATxFrameMod).  payloads: list of uint8 arrays, MPDUs without FCS (or with it, fcs_in_payload=True);
        preamble: the reference's 640-sample PREAMBLE40_11A_LUT, int16 [640, 2] -> (COMPLEX8 samples int8 [F, out_stride, 2], nsamples [F])."""
        flat, offs, lens = _payload_table(payloads)
        pre = np.ascontiguousarray(preamble, dtype=np.int16)
        if pre.size != 1280: raise Sb200Error("preamble must be 640 COMPLEX16 samples")
        if out_stride is None:
            out_stride = self.tx11a_legacy_nsamples(int(lens.max()) + (0 if fcs_in_payload else 4), rate_kbps, sample_rate_mhz)
        out = np.zeros((len(lens), out_stride, 2), np.int8); ns = np.zeros(len(lens), np.uint32)
        self.tx11a_legacy_raw(_ptr(flat), flat.size, _ptr(offs), _ptr(lens), len(lens), rate_kbps, sample_rate_mhz,
                              self.TX11A_LEGACY_FCS_IN_PAYLOAD if fcs_in_payload else 0, _ptr(pre), _ptr(out), out_stride, _ptr(ns))
        return out, ns

    def rxblocks_unpack(self, raw, left_shift=0):
        """raw: uint8 array of whole 128-byte RX_BLOCKs (a *.dmp file) -> int16 [28*nblocks, 2] via the device gather."""
        raw = np.ascontiguousarray(raw, dtype=np.uint8); nblk = len(raw) // 128
        out = np.zeros((nblk * 28, 2), np.int16)
        self._check(self._lib.sb200_rxblocks_unpack(self._h, C.c_void_p(_ptr(raw)), C.c_uint64(nblk), C.c_uint32(left_shift), C.c_void_p(_ptr(out)), C.c_void_p(0)), "sb200_rxblocks_unpack")
        return out

    def rx11n_raw(self, iq0_ptr, iq1_ptr, iq_total, off_ptr, len_ptr, nframes, out_ptr, out_stride, res_ptr, stream=0):
        self._check(self._lib.sb200_rx11n_batch(self._h, C.c_void_p(iq0_ptr), C.c_void_p(iq1_ptr), C.c_uint64(iq_total), C.c_void_p(off_ptr), C.c_void_p(len_ptr),
                                                C.c_uint32(nframes), C.c_void_p(out_ptr), C.c_uint32(out_stride), C.c_void_p(res_ptr), C.c_void_p(stream)), "sb200_rx11n_batch")

    def rx11n_batch(self, iq0, iq1, frame_off, frame_len, out_stride=1536):
        """802.11n 2x2: iq0 / iq1 int16 [n,2] at 40 Msps (the two antennas); returns (results RESULT11N_DTYPE [F], bytes [F, out_stride])."""
        iq0 = np.ascontiguousarray(iq0, dtype=np.int16).reshape(-1, 2); iq1 = np.ascontiguousarray(iq1, dtype=np.int16).reshape(-1, 2)
        assert iq0.shape == iq1.shape
        off = np.ascontiguousarray(frame_off, dtype=np.uint64); ln = np.ascontiguousarray(frame_len, dtype=np.uint32); nf = len(off)
        res = np.zeros(nf, dtype=RESULT11N_DTYPE); out = np.zeros((nf, out_stride), dtype=np.uint8)
        self.rx11n_raw(_ptr(iq0), _ptr(iq1), iq0.shape[0], _ptr(off), _ptr(ln), nf, _ptr(out), out_stride, _ptr(res))
        return res, out

    def rx11n_taps(self, iq0, iq1, frame_off, frame_len, max_sym=300):
        iq0 = np.ascontiguousarray(iq0, dtype=np.int16).reshape(-1, 2); iq1 = np.ascontiguousarray(iq1, dtype=np.int16).reshape(-1, 2)
        off = np.ascontiguousarray(frame_off, dtype=np.uint64); ln = np.ascontiguousarray(frame_len, dtype=np.uint32); nf = len(off)
        res = np.zeros(nf, dtype=RESULT11N_DTYPE)
        siso = np.zeros((nf, 2, 64, 2), np.int16); hinv = np.zeros((nf, 4, 64, 2), np.int16); eq = np.zeros((nf, 2, max_sym, 64, 2), np.int16)
        theta = np.zeros((nf, max_sym), np.int16); sig = np.zeros((nf, 16), np.uint8); sstride = max_sym * 624; soft = np.zeros((nf, sstride), np.uint8)
        self._check(self._lib.sb200_rx11n_taps(self._h, C.c_void_p(_ptr(iq0)), C.c_void_p(_ptr(iq1)), C.c_uint64(iq0.shape[0]), C.c_void_p(_ptr(off)), C.c_void_p(_ptr(ln)),
                                               C.c_uint32(nf), C.c_uint32(max_sym), C.c_void_p(_ptr(res)), C.c_void_p(_ptr(siso)), C.c_void_p(_ptr(hinv)), C.c_void_p(_ptr(eq)),
                                               C.c_void_p(_ptr(theta)), C.c_void_p(_ptr(sig)), C.c_void_p(_ptr(soft)), C.c_uint64(sstride)), "sb200_rx11n_taps")
        return dict(res=res, siso=siso, hinv=hinv, eq=eq, theta=theta, sig=sig[:, :9], soft=soft)

    def rx11b_batch(self, iq, frame_off, frame_len, out_stride=4096):
        """802.11b: iq int16 [n,2] at 44 Msps; returns (results RESULT11B_DTYPE [F], bytes uint8 [F, out_stride])."""
        iq = np.ascontiguousarray(iq, dtype=np.int16).reshape(-1, 2)
        off = np.ascontiguousarray(frame_off, dtype=np.uint64); ln = np.ascontiguousarray(frame_len, dtype=np.uint32)
        nf = len(off)
        res = np.zeros(nf, dtype=RESULT11B_DTYPE); out = np.zeros((nf, out_stride), dtype=np.uint8)
        self.rx11b_raw(_ptr(iq), iq.shape[0], _ptr(off), _ptr(ln), nf, _ptr(out), out_stride, _ptr(res))
        return res, out

    def rx11n_streams(self, iq0, iq1, stream_off, stream_len, max_frames=8, out_stride=1536):
        """802.11n continuous captures -> (results RESULT11N_DTYPE [S, max_frames], bytes [S, max_frames, out_stride], sample_index [S, max_frames], counts [S])."""
        iq0 = np.ascontiguousarray(iq0, dtype=np.int16).reshape(-1, 2); iq1 = np.ascontiguousarray(iq1, dtype=np.int16).reshape(-1, 2)
        off = np.ascontiguousarray(stream_off, dtype=np.uint64); ln = np.ascontiguousarray(stream_len, dtype=np.uint32); S = len(off)
        res = np.zeros((S, max_frames), dtype=RESULT11N_DTYPE); out = np.zeros((S, max_frames, out_stride), dtype=np.uint8)
        sidx = np.zeros((S, max_frames), np.uint32); cnt = np.zeros(S, np.uint32)
        self._check(self._lib.sb200_rx11n_streams(self._h, C.c_void_p(_ptr(iq0)), C.c_void_p(_ptr(iq1)), C.c_uint64(iq0.shape[0]), C.c_void_p(_ptr(off)), C.c_void_p(_ptr(ln)), C.c_uint32(S),
                                                  C.c_uint32(max_frames), C.c_void_p(_ptr(out)), C.c_uint32(out_stride), C.c_void_p(_ptr(res)), C.c_void_p(_ptr(sidx)), C.c_void_p(_ptr(cnt)),
                                                  C.c_void_p(0)), "sb200_rx11n_streams")
        return res, out, sidx, cnt

    def rx11b_streams(self, iq, stream_off, stream_len, max_frames=8, out_stride=4096):
        """802.11b continuous captures -> (results RESULT11B_DTYPE [S, max_frames], bytes [S, max_frames, out_stride], counts [S])."""
        iq = np.ascontiguousarray(iq, dtype=np.int16).reshape(-1, 2)
        off = np.ascontiguousarray(stream_off, dtype=np.uint64); ln = np.ascontiguousarray(stream_len, dtype=np.uint32); S = len(off)
        res = np.zeros((S, max_frames), dtype=RESULT11B_DTYPE); out = np.zeros((S, max_frames, out_stride), dtype=np.uint8); cnt = np.zeros(S, np.uint32)
        self._check(self._lib.sb200_rx11b_streams(self._h, C.c_void_p(_ptr(iq)), C.c_uint64(iq.shape[0]), C.c_void_p(_ptr(off)), C.c_void_p(_ptr(ln)), C.c_uint32(S), C.c_uint32(max_frames),
                                                  C.c_void_p(_ptr(out)), C.c_uint32(out_stride), C.c_void_p(_ptr(res)), C.c_void_p(_ptr(cnt)), C.c_void_p(0)), "sb200_rx11b_streams")
        return res, out, cnt

    def rx11a_taps(self, iq, frame_off, frame_len, max_sym):
        iq = np.ascontiguousarray(iq, dtype=np.int16).reshape(-1, 2)
        off = np.ascontiguousarray(frame_off, dtype=np.uint64); ln = np.ascontiguousarray(frame_len, dtype=np.uint32)
        nf = len(off)
        res = np.zeros(nf, dtype=RESULT_DTYPE)
        fc = np.zeros((nf, 64, 2), np.int16); cc = np.zeros_like(fc)
        fo = np.zeros((nf, max_sym, 64, 2), np.int16); eq = np.zeros_like(fo); tr = np.zeros_like(fo)
        sstride = max_sym * 288
        soft = np.zeros((nf, sstride), np.uint8)
        self._check(self._lib.sb200_rx11a_taps(self._h, _ptr(iq), iq.shape[0], _ptr(off), _ptr(ln), nf, max_sym, _ptr(res),
                                               _ptr(fc), _ptr(cc), _ptr(fo), _ptr(eq), _ptr(tr), _ptr(soft), sstride), "sb200_rx11a_taps")
        return dict(res=res, freq_coeffs=fc, chan_coeffs=cc, fft_out=fo, equalized=eq, tracked=tr, soft=soft)

    def viterbi_raw(self, soft_ptr, soft_stride, nsoft, nblocks, code_rate, frame_len, out_ptr, out_stride, depth=256, lookahead=24, stream=0):
        self._check(self._lib.sb200_viterbi_k7(self._h, soft_ptr, soft_stride, nsoft, nblocks, code_rate, frame_len, depth, lookahead,
                                               out_ptr, out_stride, stream), "sb200_viterbi_k7")

    def viterbi_k7(self, soft, code_rate, frame_len_bytes, depth=256, lookahead=24):
        """soft: uint8 [nblocks, nsoft]; returns uint8 [nblocks, frame_len_bytes+2] (SERVICE + PSDU, still scrambled)."""
        soft = np.ascontiguousarray(soft, dtype=np.uint8)
        nb, ns = soft.shape
        out = np.zeros((nb, frame_len_bytes + 2), np.uint8)
        self.viterbi_raw(_ptr(soft), ns, ns, nb, code_rate, frame_len_bytes, _ptr(out), frame_len_bytes + 2, depth, lookahead)
        return out
