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
           "sb200_rx11n_batch", "sb200_rx11n_taps", "sb200_rxblocks_unpack", "sb200_tx11a_batch", "sb200_tx11b_batch", "sb200_rx11b_streams", "sb200_rx11n_streams", "sb200_tx11n_batch", "sb200_rxblocks_desc", "sb200_fir_decimate2", "sb200_channelize", "sb200_channelize_rational", "sb200_channelize_bank", "sb200_channelize_arbitrary", "sb200_combine", "sb200_combine_rational", "sb200_combine_bank", "sb200_combine_arbitrary", "sb200_channel_sim", "sb200_spectrum", "sb200_power_meter", "sb200_tx11b_fir37", "sb200_tx11b_legacy_batch", "sb200_tx11a_legacy_batch", "sb200_host_alloc", "sb200_host_free", "sb200_last_transfer", "sb200_last_viterbi_kernel"]

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
    """NCO increment of sb200_channelize and sb200_combine for a channel centred at f_hz in a capture at fs_hz: round(f / fs * 2^32) mod 2^32 (negative f wraps)."""
    return int(round(f_hz / fs_hz * 2 ** 32)) % 2 ** 32

def bank_centres(nchannels, fs_hz, odd=False):
    """Centre frequencies (Hz) of sb200_channelize_bank's channels k = 0 .. M-1 in a capture at fs_hz: (k + o/2) fs / M, wrapped to
    [-fs/2, fs/2) (channels k >= M/2 are the negative frequencies)."""
    f = (np.arange(nchannels) + 0.5 * bool(odd)) * fs_hz / nchannels
    return np.where(np.arange(nchannels) >= nchannels // 2, f - fs_hz, f)

def arbitrary_step(fs_in, fs_out):
    """Input samples per output of sb200_channelize_arbitrary for a capture at fs_in brought to fs_out, and of sb200_combine_arbitrary for
    rows at fs_in put into a capture at fs_out: round(2^32 fs_in / fs_out) (Q32.32)."""
    return int(round(2 ** 32 * fs_in / fs_out))

def _kaiser_beta(atten_db):
    """Kaiser's window parameter for a stop-band attenuation of atten_db."""
    if atten_db > 50: return 0.1102 * (atten_db - 8.7)
    if atten_db > 21: return 0.5842 * (atten_db - 21) ** 0.4 + 0.07886 * (atten_db - 21)
    return 0.0

def arbitrary_taps(fs_in, fs_out, ntaps, passband_hz, stopband_hz=None, beta=None):
    """The 256 x ntaps Q14 table H of sb200_channelize_arbitrary for a capture at fs_in brought to fs_out, and of sb200_combine_arbitrary
    for rows at fs_in put into a capture at fs_out (there the default stop band puts the cut at the rows' Nyquist rate): a low-pass Kaiser-windowed sinc
    cut halfway between passband_hz and stopband_hz, row p evaluated at d = k - c - p / 256 (c = (ntaps - 1) // 2), where the output at
    input time i + p / 256 meets input i - c + k.  stopband_hz defaults to min(fs_in, fs_out) - passband_hz, the lowest frequency that
    the rate change folds (decimation) or images (interpolation) into the passband; beta defaults to the Kaiser value for the attenuation
    that ntaps buys over that transition band.  Every row is scaled to a DC gain of exactly 16384 (unity), so the gain does not depend on
    the phase.  -> int16 [256, ntaps].  Raises ValueError when the band edges do not fit the rates or a row's sum |H| exceeds 65535."""
    f_lo = min(fs_in, fs_out)
    stopband_hz = f_lo - passband_hz if stopband_hz is None else stopband_hz
    if not 0 < passband_hz < stopband_hz <= f_lo: raise ValueError("need 0 < passband_hz < stopband_hz <= min(fs_in, fs_out)")
    if not 1 <= ntaps <= 64: raise ValueError("ntaps must be 1 .. 64")
    if beta is None: beta = _kaiser_beta(2.285 * 2 * np.pi * (stopband_hz - passband_hz) / fs_in * max(ntaps - 1, 1) + 8)
    fc = 0.5 * (passband_hz + stopband_hz) / fs_in                       # cycles per input sample
    c = (ntaps - 1) // 2; half = ntaps / 2.0
    d = np.arange(ntaps)[None, :] - c - (np.arange(256) / 256.0)[:, None]
    h = 2 * fc * np.sinc(2 * fc * d) * np.i0(beta * np.sqrt(np.clip(1 - (d / half) ** 2, 0, 1))) / np.i0(beta)
    q = np.rint(h / h.sum(1, keepdims=True) * 16384).astype(np.int64)
    q[np.arange(256), np.argmax(np.abs(q), 1)] += 16384 - q.sum(1)       # exact unity DC gain on every row
    if np.abs(q).max() > 32767 or (np.abs(q).sum(1) > 65535).any(): raise ValueError("a row of the table exceeds sum |H| <= 65535")
    return q.astype(np.int16)

class DdcChannel(C.Structure):
    _fields_ = [("phase_inc", C.c_uint32), ("phase0", C.c_uint32)]

class DucChannel(C.Structure):
    _fields_ = [("phase_inc", C.c_uint32), ("phase0", C.c_uint32), ("gain", C.c_uint32)]

class SimLink(C.Structure):
    """sb200_link: one link of sb200_channel_sim (include/sora_b200.h)."""
    _fields_ = [("tau0", C.c_uint64), ("step", C.c_uint64), ("phase_inc", C.c_uint32), ("phase0", C.c_uint32), ("noise_q8", C.c_uint32), ("reserved", C.c_uint32)]

LINK_DTYPE = np.dtype([("tau0", "<u8"), ("step", "<u8"), ("phase_inc", "<u4"), ("phase0", "<u4"), ("noise_q8", "<u4"), ("reserved", "<u4")])
assert LINK_DTYPE.itemsize == C.sizeof(SimLink)

def sim_links(records):
    """Link records for sb200_channel_sim: a LINK_DTYPE array, or tuples (tau0, step, phase_inc, phase0, noise_q8) -> LINK_DTYPE array.
    Increments and phases wrap mod 2^32, so a negative phase_inc stands for a negative frequency."""
    if isinstance(records, np.ndarray) and records.dtype == LINK_DTYPE:
        return np.ascontiguousarray(records)
    out = np.zeros(len(records), LINK_DTYPE)
    for i, (tau0, step, inc, ph, sig) in enumerate(records):
        out[i] = (int(tau0), int(step), int(inc) % 2 ** 32, int(ph) % 2 ** 32, int(sig), 0)
    return out

def clock_step(ppm):
    """Clock step of a link whose receiver's sample clock runs ppm parts per million fast: round(2^32 / (1 + ppm 1e-6)) input samples (Q32.32)
    per output sample, so the receiver takes (1 + ppm 1e-6) times as many samples of the same signal."""
    return int(round(2 ** 32 / (1 + ppm * 1e-6)))

def sim_taps(delays, gains, L):
    """Tapped-delay-line profile (delays in whole samples, complex gains, or 2x2 matrices g[r, t] for a MIMO link) -> Q14 int16 [R, T, L, 2]
    taps of sb200_channel_sim: g[r][t][d] = rint(16384 gain).  Raises ValueError when a delay is not below L or a row's sum of |re| + |im|
    exceeds 65535."""
    g0 = np.asarray(gains[0], np.complex128)
    R, T = (1, 1) if g0.ndim == 0 else g0.shape
    h = np.zeros((R, T, L), np.complex128)
    for d, g in zip(delays, gains):
        if not 0 <= int(d) < L: raise ValueError(f"delay {d} is not below L = {L}")
        h[:, :, int(d)] += np.asarray(g, np.complex128).reshape(R, T)
    q = np.stack([np.rint(h.real * 16384), np.rint(h.imag * 16384)], -1)
    if np.abs(q).max() > 32767 or (np.abs(q).sum((1, 2, 3)) > 65535).any():
        raise ValueError("taps out of range: every |g| below 2 and every row's sum of |re| + |im| at most 65535 / 16384")
    return q.astype(np.int16)

def spectrum_window(N, kind="hann"):
    """Q15 window of N taps for Engine.spectrum: rint(32767 w[n]) of the periodic (DFT-even) window, n = 0 .. N - 1.
    kind "hann":            w[n] = 0.5 - 0.5 cos(2 pi n / N)
    kind "blackman-harris": w[n] = 0.35875 - 0.48829 cos(2 pi n / N) + 0.14128 cos(4 pi n / N) - 0.01168 cos(6 pi n / N)  (4 terms)"""
    a = 2 * np.pi * np.arange(N) / N
    if kind == "hann": w = 0.5 - 0.5 * np.cos(a)
    elif kind in ("blackman-harris", "blackmanharris"): w = 0.35875 - 0.48829 * np.cos(a) + 0.14128 * np.cos(2 * a) - 0.01168 * np.cos(3 * a)
    else: raise ValueError("kind must be 'hann' or 'blackman-harris'")
    return np.clip(np.rint(32767 * w), 0, 32767).astype(np.int16)

def spectrum_frames(n_in, N, hop=None):
    """Frames of sb200_spectrum in a row of n_in samples: frame f covers [f hop, f hop + N); (n_in - N) // hop + 1 if n_in >= N, else 0."""
    hop = N if hop is None else hop
    return (n_in - N) // hop + 1 if n_in >= N else 0

def fftshift_bins(spec, fs_hz=1.0):
    """Display order of a spectrum (bins in natural FFT order along the last axis, bin k at k fs / N for k < N / 2 and (k - N) fs / N
    above): (the bins in centred order, from -fs / 2 up, and their frequencies in Hz)."""
    spec = np.asarray(spec); N = spec.shape[-1]
    return np.fft.fftshift(spec, axes=-1), np.fft.fftshift(np.fft.fftfreq(N, 1.0 / fs_hz))

_NDBPS_11A = {6000: 24, 9000: 36, 12000: 48, 18000: 72, 24000: 96, 36000: 144, 48000: 192, 54000: 216}   # 802.11a data bits per OFDM symbol
_NDBPS_11N = {8: 52, 9: 104, 10: 156}                   # 802.11n data bits per OFDM symbol over both streams, MCS 8 .. 10
_CHIPS_11B = {1000: 88, 2000: 44, 5500: 16, 11000: 8}   # 802.11b chips per PSDU byte

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

def _rows4(k, n, rows=None):
    """k zeroed int16 rows of n samples, a stride of n rounded up to 4 apart, with `rows` ([k, n, 2]) copied in -> (int16 [k, stride, 2], stride)."""
    stride = (n + 3) // 4 * 4
    x = np.zeros((k, stride, 2), np.int16)
    if rows is not None: x[:, :n] = rows
    return x, stride

def _out_samples(out, n):
    """The output of a combiner: zeros when out is None, else out itself once checked to be a writeable C-contiguous int16 [n, 2] array."""
    if out is None: return np.zeros((n, 2), np.int16)
    if not (isinstance(out, np.ndarray) and out.dtype == np.int16 and out.shape == (n, 2) and out.flags.c_contiguous and out.flags.writeable):
        raise ValueError("out must be a writeable C-contiguous int16 numpy array of shape [n_out, 2]")
    return out

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

    @staticmethod
    def tx11a_out_stride(length, rate_kbps, lead=0):
        """Default out_stride of tx11a_batch for MPDUs of up to `length` bytes (FCS not included): lead, the preamble, SIGNAL and the data
        symbols with two to spare, and 32 samples more.  KeyError for a rate that is not an 802.11a rate."""
        return lead + 640 + 160 * (2 + -(-(length + 7) * 8 // _NDBPS_11A[rate_kbps]) + 1) + 32

    def tx11a_batch(self, payloads, rate_kbps, seeds=None, lead=0, sample_bits=8, out_stride=None):
        """payloads: list of uint8 arrays (MPDUs without FCS) -> (samples [F, out_stride, 2] int8 or int16, nsamples [F])."""
        flat, offs, lens = _payload_table(payloads)
        if out_stride is None: out_stride = self.tx11a_out_stride(int(lens.max()), rate_kbps, lead)
        out = np.zeros((len(lens), out_stride, 2), np.int8 if sample_bits == 8 else np.int16); ns = np.zeros(len(lens), np.uint32)
        sd = None if seeds is None else np.ascontiguousarray(seeds, dtype=np.uint8)
        self.tx11a_raw(_ptr(flat), flat.size, _ptr(offs), _ptr(lens), 0 if sd is None else _ptr(sd), len(lens), rate_kbps, lead, sample_bits, _ptr(out), out_stride, _ptr(ns))
        return out, ns

    def tx11n_raw(self, pay_ptr, pay_total, off_ptr, len_ptr, seed_ptr, nframes, mcs, lead, out0_ptr, out1_ptr, out_stride, ns_ptr, stream=0):
        self._check(self._lib.sb200_tx11n_batch(self._h, C.c_void_p(pay_ptr), C.c_uint64(pay_total), C.c_void_p(off_ptr), C.c_void_p(len_ptr), C.c_void_p(seed_ptr), C.c_uint32(nframes),
                                                C.c_uint32(mcs), C.c_uint32(lead), C.c_void_p(out0_ptr), C.c_void_p(out1_ptr), C.c_uint64(out_stride), C.c_void_p(ns_ptr),
                                                C.c_void_p(stream)), "sb200_tx11n_batch")

    @staticmethod
    def tx11n_out_stride(length, mcs, lead=0):
        """Default out_stride of tx11n_batch for MPDUs of up to `length` bytes (FCS not included): lead, the preamble and SIG symbols, and the
        data symbols with one to spare.  MCS 11 .. 14 are sized as MCS 8, which needs the most symbols."""
        return lead + 1600 + 160 * (-(-((length + 4) * 8 + 22) // _NDBPS_11N.get(mcs, 52)) + 1)

    def tx11n_batch(self, payloads, mcs, seeds=None, lead=0, out_stride=None):
        """payloads: list of uint8 arrays (MPDUs without FCS) -> (stream 0 [F, out_stride, 2] int16, stream 1, nsamples [F]) at 40 Msps."""
        flat, offs, lens = _payload_table(payloads)
        if out_stride is None: out_stride = self.tx11n_out_stride(int(lens.max()), mcs, lead)
        o0 = np.zeros((len(lens), out_stride, 2), np.int16); o1 = np.zeros_like(o0); ns = np.zeros(len(lens), np.uint32)
        sd = None if seeds is None else np.ascontiguousarray(seeds, dtype=np.uint8)
        self.tx11n_raw(_ptr(flat), flat.size, _ptr(offs), _ptr(lens), 0 if sd is None else _ptr(sd), len(lens), mcs, lead, _ptr(o0), _ptr(o1), out_stride, _ptr(ns))
        return o0, o1, ns

    def tx11b_raw(self, pay_ptr, pay_total, off_ptr, len_ptr, nframes, rate_kbps, init_phase, lead, bits, out_ptr, out_stride, ns_ptr, stream=0, fp_ptr=0):
        self._check(self._lib.sb200_tx11b_batch(self._h, C.c_void_p(pay_ptr), C.c_uint64(pay_total), C.c_void_p(off_ptr), C.c_void_p(len_ptr), C.c_uint32(nframes),
                                                C.c_uint32(rate_kbps), C.c_uint32(init_phase), C.c_uint32(lead), C.c_uint32(bits), C.c_void_p(out_ptr),
                                                C.c_uint64(out_stride), C.c_void_p(ns_ptr), C.c_void_p(fp_ptr), C.c_void_p(stream)), "sb200_tx11b_batch")

    @staticmethod
    def tx11b_out_stride(length, rate_kbps, lead=0):
        """Default out_stride of tx11b_batch for MPDUs of up to `length` bytes (FCS not included): lead and four samples per chip of the PLCP
        and the PSDU and five more, rounded up to 8.  An unknown rate is the library's error to report."""
        return (lead + (24 * 88 + (length + 4) * _CHIPS_11B.get(rate_kbps, 8) + 5) * 4 + 15) // 8 * 8

    def tx11b_batch(self, payloads, rate_kbps, init_phase=0, lead=0, sample_bits=8, out_stride=None, return_phase=False):
        """payloads: list of uint8 arrays (MPDUs without FCS) -> (samples [F, out_stride, 2] int8 or int16 at 44 Msps, nsamples [F])."""
        flat, offs, lens = _payload_table(payloads)
        if out_stride is None: out_stride = self.tx11b_out_stride(int(lens.max()), rate_kbps, lead)
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

    def channelize_raw(self, in_ptr, n_in, channels, decim, taps, out_ptr, out_stride, stream=0, interp=1):
        """Pointer-level sb200_channelize (interp = 1) or sb200_channelize_rational: in_ptr / out_ptr host or device addresses; channels a
        list of (phase_inc, phase0); taps int16 Q15."""
        ch = (DdcChannel * max(len(channels), 1))(*[DdcChannel(int(a) % 2 ** 32, int(b) % 2 ** 32) for a, b in channels])
        t = np.ascontiguousarray(taps, dtype=np.int16)
        if interp == 1:
            self._check(self._lib.sb200_channelize(self._h, C.c_void_p(in_ptr), C.c_uint64(n_in), C.cast(ch, C.c_void_p), C.c_uint32(len(channels)), C.c_uint32(decim),
                                                   C.c_void_p(_ptr(t)), C.c_uint32(len(t)), C.c_void_p(out_ptr), C.c_uint64(out_stride), C.c_void_p(stream)), "sb200_channelize")
        else:
            self._check(self._lib.sb200_channelize_rational(self._h, C.c_void_p(in_ptr), C.c_uint64(n_in), C.cast(ch, C.c_void_p), C.c_uint32(len(channels)),
                                                            C.c_uint32(interp), C.c_uint32(decim), C.c_void_p(_ptr(t)), C.c_uint32(len(t)), C.c_void_p(out_ptr),
                                                            C.c_uint64(out_stride), C.c_void_p(stream)), "sb200_channelize_rational")

    def channelize(self, iq, channels, decim, taps, interp=1):
        """Wideband channelizer: int16 [n,2] and K channels (phase_inc, phase0) -> int16 [K, ceil(interp n / decim), 2], channel k shifted
        to 0 Hz, filtered by taps (int16 Q15, odd count; interp = 1: <= 255 taps, sum |t| <= 65535; else ceil(ntaps / interp) <= 255 and
        the same limit per branch) and resampled by interp / decim."""
        iq = np.ascontiguousarray(iq, dtype=np.int16).reshape(-1, 2)
        n_out = -(-interp * len(iq) // decim); out, stride = _rows4(len(channels), n_out)
        self.channelize_raw(_ptr(iq), len(iq), channels, decim, taps, _ptr(out), stride, interp=interp)
        return out[:, :n_out]

    def channelize_bank_raw(self, in_ptr, n_in, nchannels, decim, taps, out_ptr, out_stride, odd=False, stream=0):
        """Pointer-level sb200_channelize_bank: in_ptr / out_ptr host or device addresses, row k of the output at out_ptr + 4 k out_stride
        bytes; taps int16 Q15."""
        t = np.ascontiguousarray(taps, dtype=np.int16)
        self._check(self._lib.sb200_channelize_bank(self._h, C.c_void_p(in_ptr), C.c_uint64(n_in), C.c_uint32(nchannels), C.c_uint32(decim), C.c_uint32(int(bool(odd))),
                                                    C.c_void_p(_ptr(t)), C.c_uint32(len(t)), C.c_void_p(out_ptr), C.c_uint64(out_stride), C.c_void_p(stream)),
                    "sb200_channelize_bank")

    def channelize_bank(self, iq, nchannels, decim, taps, odd=False):
        """Polyphase filter-bank channelizer: int16 [n,2] -> int16 [M, ceil(n / decim), 2], every channel of the uniform grid of M =
        nchannels (a power of two, 2 .. 64) centred at bank_centres(M, fs, odd), shifted to 0 Hz, filtered by taps (int16 Q15, odd count
        <= 1023, sum |t| <= 65535) and decimated by decim (a divisor of M)."""
        iq = np.ascontiguousarray(iq, dtype=np.int16).reshape(-1, 2)
        n_out = -(-len(iq) // decim); out, stride = _rows4(nchannels, n_out)
        self.channelize_bank_raw(_ptr(iq), len(iq), nchannels, decim, taps, _ptr(out), stride, odd=odd)
        return out[:, :n_out]

    def channelize_arbitrary_raw(self, in_ptr, n_in, channels, tau0, step, taps, out_ptr, out_stride, n_out, stream=0):
        """Pointer-level sb200_channelize_arbitrary: in_ptr / out_ptr host or device addresses, row k of the output at out_ptr + 4 k out_stride
        bytes; channels a list of (phase_inc, phase0); taps int16 Q14 [256, ntaps]."""
        ch = (DdcChannel * max(len(channels), 1))(*[DdcChannel(int(a) % 2 ** 32, int(b) % 2 ** 32) for a, b in channels])
        t = np.ascontiguousarray(taps, dtype=np.int16)
        if t.ndim != 2 or t.shape[0] != 256: raise ValueError("taps must be int16 [256, ntaps]")
        self._check(self._lib.sb200_channelize_arbitrary(self._h, C.c_void_p(in_ptr), C.c_uint64(n_in), C.cast(ch, C.c_void_p), C.c_uint32(len(channels)),
                                                         C.c_uint64(tau0), C.c_uint64(step), C.c_void_p(_ptr(t)), C.c_uint32(t.shape[1]), C.c_void_p(out_ptr),
                                                         C.c_uint64(out_stride), C.c_uint64(n_out), C.c_void_p(stream)), "sb200_channelize_arbitrary")

    def channelize_arbitrary(self, iq, channels, step, taps, tau0=0, n_out=None):
        """Arbitrary-rate channelizer: int16 [n,2] and K channels (phase_inc, phase0) -> int16 [K, n_out, 2], channel k shifted to 0 Hz and
        resampled at input times (tau0 + m step) / 2^32 through the 256-phase Q14 table taps (int16 [256, ntaps], arbitrary_taps);
        step = arbitrary_step(fs_in, fs_out).  n_out defaults to the outputs whose time lies inside the input, tau0 + m step < n 2^32."""
        iq = np.ascontiguousarray(iq, dtype=np.int16).reshape(-1, 2)
        if n_out is None: n_out = max(0, -(-((len(iq) << 32) - tau0) // step))
        out, stride = _rows4(len(channels), n_out)
        self.channelize_arbitrary_raw(_ptr(iq), len(iq), channels, tau0, step, taps, _ptr(out), stride, n_out)
        return out[:, :n_out]

    def combine_raw(self, rows_ptr, row_stride, n_in, channels, interp, taps, out_ptr, stream=0, decim=1, n_out=None, accumulate=False):
        """Pointer-level sb200_combine (decim = 1, n_out None, accumulate False) or sb200_combine_rational: rows_ptr / out_ptr host or device
        addresses; channels a list of (phase_inc, phase0, gain); taps int16 Q15; n_out outputs (None: ceil(interp n_in / decim))."""
        ch = (DucChannel * max(len(channels), 1))(*[DucChannel(int(a) % 2 ** 32, int(b) % 2 ** 32, int(g)) for a, b, g in channels])
        t = np.ascontiguousarray(taps, dtype=np.int16)
        if decim == 1 and n_out is None and not accumulate:
            self._check(self._lib.sb200_combine(self._h, C.c_void_p(rows_ptr), C.c_uint64(row_stride), C.c_uint64(n_in), C.cast(ch, C.c_void_p), C.c_uint32(len(channels)),
                                                C.c_uint32(interp), C.c_void_p(_ptr(t)), C.c_uint32(len(t)), C.c_void_p(out_ptr), C.c_void_p(stream)), "sb200_combine")
        else:
            n_out = -(-interp * n_in // decim) if n_out is None else n_out
            self._check(self._lib.sb200_combine_rational(self._h, C.c_void_p(rows_ptr), C.c_uint64(row_stride), C.c_uint64(n_in), C.cast(ch, C.c_void_p),
                                                         C.c_uint32(len(channels)), C.c_uint32(interp), C.c_uint32(decim), C.c_void_p(_ptr(t)), C.c_uint32(len(t)),
                                                         C.c_void_p(out_ptr), C.c_uint64(n_out), C.c_uint32(int(accumulate)), C.c_void_p(stream)), "sb200_combine_rational")

    def combine(self, rows, channels, interp, taps, decim=1, n_out=None, accumulate=False, out=None):
        """Wideband combiner: int16 [K, n_in, 2] rows and K channels (phase_inc, phase0, gain Q12) -> int16 [n_out, 2], every row
        interpolated by interp through taps (int16 Q15, odd count <= 255, per-branch sum |t| <= 65535), moved to its centre, scaled and summed;
        n_out = interp * n_in.  With decim, n_out or accumulate it is sb200_combine_rational: the rate changes by interp / decim (ntaps <= 4095
        with ceil(ntaps / interp) <= 255), n_out defaults to ceil(interp n_in / decim), and accumulate adds the sum onto `out` (int16
        [n_out, 2], updated in place and returned) with one saturation."""
        rows = np.asarray(rows, dtype=np.int16).reshape(len(channels), -1, 2); n_in = rows.shape[1]; x, stride = _rows4(len(channels), n_in, rows)
        out = _out_samples(out, -(-interp * n_in // decim) if n_out is None else n_out)
        self.combine_raw(_ptr(x), stride, n_in, channels, interp, taps, _ptr(out), decim=decim, n_out=n_out, accumulate=accumulate)
        return out

    def combine_bank_raw(self, rows_ptr, row_stride, n_in, nchannels, interp, taps, out_ptr, n_out, odd=False, accumulate=False, stream=0):
        """Pointer-level sb200_combine_bank: rows_ptr / out_ptr host or device addresses, row k at rows_ptr + 4 k row_stride bytes; taps
        int16 Q15; n_out outputs."""
        t = np.ascontiguousarray(taps, dtype=np.int16)
        self._check(self._lib.sb200_combine_bank(self._h, C.c_void_p(rows_ptr), C.c_uint64(row_stride), C.c_uint64(n_in), C.c_uint32(nchannels), C.c_uint32(interp),
                                                 C.c_uint32(int(bool(odd))), C.c_void_p(_ptr(t)), C.c_uint32(len(t)), C.c_void_p(out_ptr), C.c_uint64(n_out),
                                                 C.c_uint32(int(bool(accumulate))), C.c_void_p(stream)), "sb200_combine_bank")

    def combine_bank(self, rows, interp, taps, odd=False, n_out=None, accumulate=False, out=None):
        """Polyphase filter-bank combiner: int16 [M, n_in, 2] rows -> int16 [n_out, 2], row k interpolated by interp (a divisor of M, a
        power of two 2 .. 64) through taps (int16 Q15, odd count <= 1023 and <= 2048 interp / M) and moved to bank_centres(M, fs, odd)[k];
        n_out defaults to interp * n_in.  accumulate adds the sum onto `out` (int16 [n_out, 2], updated in place and returned) with one
        saturation."""
        rows = np.asarray(rows, dtype=np.int16)
        if rows.ndim != 3 or rows.shape[2] != 2: raise ValueError("rows must be int16 [M, n_in, 2]")
        M, n_in = rows.shape[:2]; x, stride = _rows4(M, n_in, rows)
        out = _out_samples(out, interp * n_in if n_out is None else n_out)
        self.combine_bank_raw(_ptr(x), stride, n_in, M, interp, taps, _ptr(out), len(out), odd=odd, accumulate=accumulate)
        return out

    def combine_arbitrary_raw(self, rows_ptr, row_stride, n_in, channels, tau0, step, taps, out_ptr, n_out, accumulate=False, stream=0):
        """Pointer-level sb200_combine_arbitrary: rows_ptr / out_ptr host or device addresses, row k at rows_ptr + 4 k row_stride bytes;
        channels a list of (phase_inc, phase0, gain); taps int16 Q14 [256, ntaps]; n_out outputs."""
        ch = (DucChannel * max(len(channels), 1))(*[DucChannel(int(a) % 2 ** 32, int(b) % 2 ** 32, int(g)) for a, b, g in channels])
        t = np.ascontiguousarray(taps, dtype=np.int16)
        if t.ndim != 2 or t.shape[0] != 256: raise ValueError("taps must be int16 [256, ntaps]")
        self._check(self._lib.sb200_combine_arbitrary(self._h, C.c_void_p(rows_ptr), C.c_uint64(row_stride), C.c_uint64(n_in), C.cast(ch, C.c_void_p),
                                                      C.c_uint32(len(channels)), C.c_uint64(tau0), C.c_uint64(step), C.c_void_p(_ptr(t)), C.c_uint32(t.shape[1]),
                                                      C.c_void_p(out_ptr), C.c_uint64(n_out), C.c_uint32(int(bool(accumulate))), C.c_void_p(stream)),
                    "sb200_combine_arbitrary")

    def combine_arbitrary(self, rows, channels, step, taps, tau0=0, n_out=None, accumulate=False, out=None):
        """Arbitrary-rate combiner: int16 [K, n_in, 2] rows and K channels (phase_inc, phase0, gain Q12) -> int16 [n_out, 2], every row
        resampled at row times (tau0 + n step) / 2^32 through the 256-phase Q14 table taps (int16 [256, ntaps], arbitrary_taps), moved to
        its centre, scaled and summed; step = arbitrary_step(fs_rows, fs_capture).  n_out defaults to the outputs whose time lies inside
        the rows, tau0 + n step < n_in 2^32.  accumulate adds the sum onto `out` (int16 [n_out, 2], updated in place and returned) with one
        saturation."""
        rows = np.asarray(rows, dtype=np.int16).reshape(len(channels), -1, 2); n_in = rows.shape[1]; x, stride = _rows4(len(channels), n_in, rows)
        if n_out is None: n_out = max(0, -(-((n_in << 32) - tau0) // step))
        out = _out_samples(out, n_out)
        self.combine_arbitrary_raw(_ptr(x), stride, n_in, channels, tau0, step, taps, _ptr(out), n_out, accumulate=accumulate)
        return out

    def channel_sim_raw(self, x_ptr, in_link_stride, in_row_stride, ntx, n_in, links, taps, ntaps, nlinks, seed, y_ptr, out_link_stride, out_row_stride,
                        nrx, n_out, stream=0):
        """Pointer-level sb200_channel_sim: x / y / links / taps each a host or device address (links and taps may also be numpy arrays)."""
        self._check(self._lib.sb200_channel_sim(self._h, C.c_void_p(x_ptr), C.c_uint64(in_link_stride), C.c_uint64(in_row_stride), C.c_uint32(ntx), C.c_uint64(n_in),
                                                C.c_void_p(_ptr(links)), C.c_void_p(_ptr(taps)), C.c_uint32(ntaps), C.c_uint32(nlinks), C.c_uint64(seed % 2 ** 64),
                                                C.c_void_p(y_ptr), C.c_uint64(out_link_stride), C.c_uint64(out_row_stride), C.c_uint32(nrx), C.c_uint64(n_out),
                                                C.c_void_p(stream)), "sb200_channel_sim")

    def channel_sim(self, x, links, taps, n_out, seed=0):
        """Radio channel simulator: int16 x [nlinks, T, n_in, 2], link records (sim_links), Q14 taps int16 [nlinks, R, T, L, 2] (or [R, T, L, 2]
        for every link), n_out -> int16 y [nlinks, R, n_out, 2].  See sb200_channel_sim in include/sora_b200.h for the arithmetic."""
        x = np.asarray(x, np.int16); nl, T, n_in = x.shape[:3]
        lk = sim_links(links); assert len(lk) == nl
        t = np.asarray(taps, np.int16)
        if t.ndim == 4: t = np.broadcast_to(t, (nl,) + t.shape)
        t = np.ascontiguousarray(t); R, L = t.shape[1], t.shape[3]; assert t.shape[2] == T
        si = (n_in + 3) // 4 * 4; xs = np.zeros((nl, T, si, 2), np.int16); xs[:, :, :n_in] = x
        so = (n_out + 3) // 4 * 4; y = np.zeros((nl, R, so, 2), np.int16)
        self.channel_sim_raw(_ptr(xs), T * si, si, T, n_in, lk, t, L, nl, seed, _ptr(y), R * so, so, R, n_out)
        return y[:, :, :n_out]

    def spectrum_raw(self, in_ptr, row_stride, nrows, n_in, fft_len, hop, avg, window, out_ptr, stream=0):
        """Pointer-level sb200_spectrum: in_ptr / out_ptr host or device addresses, row r at in_ptr + 4 r row_stride bytes; window None or
        int16 Q15 [fft_len] (host); out int64 [nrows, ngroups, fft_len]."""
        w = None if window is None else np.ascontiguousarray(window, dtype=np.int16)
        self._check(self._lib.sb200_spectrum(self._h, C.c_void_p(in_ptr), C.c_uint64(row_stride), C.c_uint32(nrows), C.c_uint64(n_in), C.c_uint32(fft_len),
                                             C.c_uint64(hop), C.c_uint32(avg), C.c_void_p(_ptr(w)), C.c_void_p(out_ptr), C.c_void_p(stream)), "sb200_spectrum")

    def spectrum(self, iq_rows, fft_len, hop=None, avg=1, window=None):
        """Spectrum meter (TSpecMeter<N> of the reference spectrum analyser, generalised): int16 [n_in, 2] or [R, n_in, 2] -> int64
        [R, ngroups, N].  Frames of N = fft_len samples every hop (default N) samples, windowed by `window` (None, int16 Q15 [N], or a
        spectrum_window kind such as "hann"), through FFT<N>; |X[k]|^2 per bin in natural FFT order (bin k at k fs / N, see fftshift_bins),
        bin 0 cleared, summed over groups of avg frames; ngroups = spectrum_frames(n_in, N, hop) // avg."""
        x = np.asarray(iq_rows, dtype=np.int16)
        if x.ndim == 2: x = x[None]
        if x.ndim != 3 or x.shape[2] != 2: raise ValueError("iq_rows must be int16 [n_in, 2] or [R, n_in, 2]")
        R, n_in = x.shape[:2]; xs, stride = _rows4(R, n_in, x)
        hop = fft_len if hop is None else hop
        if isinstance(window, str): window = spectrum_window(fft_len, window)
        out = np.zeros((R, spectrum_frames(n_in, fft_len, hop) // avg, fft_len), np.int64)
        self.spectrum_raw(_ptr(xs), stride, R, n_in, fft_len, hop, avg, window, _ptr(out))
        return out

    def power_meter_raw(self, in_ptr, row_stride, nrows, n_in, block_len, out_ptr, stream=0):
        """Pointer-level sb200_power_meter: in_ptr / out_ptr host or device addresses; out uint32 [nrows, n_in // block_len]."""
        self._check(self._lib.sb200_power_meter(self._h, C.c_void_p(in_ptr), C.c_uint64(row_stride), C.c_uint32(nrows), C.c_uint64(n_in),
                                                C.c_uint32(block_len), C.c_void_p(out_ptr), C.c_void_p(stream)), "sb200_power_meter")

    def power_meter(self, iq_rows, block_len):
        """Power meter (TPowerMeter<N> of the reference spectrum analyser): int16 [n_in, 2] or [R, n_in, 2] -> uint32 [R, n_in // N], the
        mean |x|^2 of each block of N = block_len samples with the reference's per-vector division order (include/sora_b200.h)."""
        x = np.asarray(iq_rows, dtype=np.int16)
        if x.ndim == 2: x = x[None]
        if x.ndim != 3 or x.shape[2] != 2: raise ValueError("iq_rows must be int16 [n_in, 2] or [R, n_in, 2]")
        R, n_in = x.shape[:2]; xs, stride = _rows4(R, n_in, x)
        out = np.zeros((R, n_in // block_len), np.uint32)
        self.power_meter_raw(_ptr(xs), stride, R, n_in, block_len, _ptr(out))
        return out

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

    @staticmethod
    def tx11b_legacy_nsamples(psdu_len, rate_kbps, short_preamble=False):
        """Samples BB11BPMDBufferTx4X* writes for a PSDU of psdu_len bytes (FCS included): four per chip and TX_FIR_DEPTH zeros, rounded up
        to 128.  The short preamble sends no data chips at 1 Mbps."""
        cpb = 0 if short_preamble and rate_kbps == 1000 else _CHIPS_11B.get(rate_kbps, 8)     # an unknown rate is the library's error to report
        return (4 * ((1056 if short_preamble else 2112) + psdu_len * cpb) + 37 + 127) // 128 * 128

    def tx11b_legacy_batch(self, payloads, rate_kbps, short_preamble=False, filter=1, fcs_in_payload=False, out_stride=None):
        """The legacy 802.11b transmitter (BB11BPMDBufferTx4X* and, filter 1 / 2, the SSE / ASM 37-tap filter).  payloads: list of uint8 arrays,
        MPDUs without FCS (or with it, fcs_in_payload=True) -> (COMPLEX8 samples int8 [F, out_stride, 2] at 44 Msps, nsamples [F])."""
        flat, offs, lens = _payload_table(payloads)
        if out_stride is None: out_stride = self.tx11b_legacy_nsamples(int(lens.max()) + (0 if fcs_in_payload else 4), rate_kbps, short_preamble)
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
