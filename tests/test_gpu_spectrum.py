"""GPU tests of the spectrum and power meters (sb200_spectrum, sb200_power_meter; pytest -m gpu): bit for bit against the reference's own
compiled TSpecMeter<N> and TPowerMeter<N> (oracle/_ref/libmeter_ref.so, built by oracle/build_ref_meter.sh) and against the numpy model
of tests/spectrum_model.py where the call goes beyond them (overlap, windows, group sums); shapes, pointer residency, caller streams,
argument checks; and a functional loop through the filter-bank combiner and channelizer."""
import ctypes as C
import numpy as np, pytest
import torch
import spectrum_model as SM
import wideband_inputs as W
from sora_b200 import api
from test_gpu_abi_residency import _matrix, _each, _fill
from test_cpu_spectrum_reference import SIZES, POWER_SIZES, METER, inputs, ref_spec, ref_power
import os

pytestmark = pytest.mark.gpu
V, U32, U64 = C.c_void_p, C.c_uint32, C.c_uint64
need_ref = pytest.mark.skipif(not os.path.exists(METER), reason="oracle/_ref/libmeter_ref.so not built")

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

def _noise(shape, seed, amp=32768):
    return np.random.default_rng(seed).integers(-amp, amp, shape).astype(np.int16)

# ---- bit-exactness ------------------------------------------------------------------------------------------------------------------
@need_ref
@pytest.mark.parametrize("N", SIZES)
def test_spectrum_equals_compiled_spec_meter(eng, N):
    """window = NULL, hop = N, avg = 1: every output row is TSpecMeter<N>'s row, on the structured and random frames of the CPU test."""
    x = inputs(N, 7)
    got = eng.spectrum(x.reshape(-1, 2), N)
    assert got.shape == (1, len(x), N) and (got[0] == ref_spec(x)).all()

@pytest.mark.parametrize("N", [4, 8, 16, 64, 256, 1024, 4096, 32768])
@pytest.mark.parametrize("hop_of", ["quarter", "minus1", "plus3", "double"])
def test_spectrum_hops_windows_avg(eng, N, hop_of):
    hop = {"quarter": max(1, N // 4), "minus1": max(1, N - 1), "plus3": N + 3, "double": 2 * N}[hop_of]
    n_in = max(40 * N, 3 * N + 5 * hop) + 7
    x = _noise((n_in, 2), N + hop)
    for avg, win in ((1, None), (3, "hann"), (64, "blackman-harris")):
        w = None if win is None else api.spectrum_window(N, win)
        got = eng.spectrum(x, N, hop=hop, avg=avg, window=w)
        want = SM.spectrum(x, N, hop, avg, w)
        assert got.shape == want.shape and (got == want).all(), (N, hop, avg, win)

@need_ref
@pytest.mark.parametrize("N", POWER_SIZES)
def test_power_meter_equals_compiled(eng, N):
    rng = np.random.default_rng(N); B = max(4, 131072 // N)
    x = np.concatenate([rng.integers(-32768, 32768, (B, N, 2)), np.full((1, N, 2), -32768), rng.integers(-300, 300, (B, N, 2)),
                        np.where(rng.integers(0, 2, (B, N, 2)) == 1, 32767, -32768)]).astype(np.int16)
    got = eng.power_meter(x.reshape(-1, 2), N)
    assert got.shape == (1, len(x)) and (got[0] == ref_power(x)).all()

def test_power_meter_negative_vector_sums(eng):
    for N in (4, 5, 128, 840, 4096):
        x = np.full((3, N, 2), -32768, np.int16); x[1, 3::4] = (16384, 0); x[2, 3::4] = (0, 1)
        assert (eng.power_meter(x.reshape(-1, 2), N)[0] == SM.power_meter_blocks(x)).all()

# ---- shapes ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,hop,avg", [(64, 64, 1), (256, 100, 3), (1024, 1024, 5), (16384, 8000, 2)])
def test_many_rows_and_partial_frames(eng, N, hop, avg):
    """Up to 64 rows a stride above n_in apart; n_in not a whole number of frames; trailing frames that do not fill a group unused."""
    R = 64 if N <= 1024 else 5
    n_in = 7 * hop + N + 13; stride = (n_in + 3) // 4 * 4 + 8
    x = np.full((R, stride, 2), 0x3C3C, np.int16); x[:, :n_in] = _noise((R, n_in, 2), N)
    ng = SM.frames_of(n_in, N, hop) // avg
    out = np.zeros((R, ng, N), np.int64)
    eng.spectrum_raw(x.ctypes.data, stride, R, n_in, N, hop, avg, None, out.ctypes.data)
    assert (out == SM.spectrum(x[:, :n_in], N, hop, avg)).all()
    pm = np.zeros((R, n_in // 840), np.uint32)
    eng.power_meter_raw(x.ctypes.data, stride, R, n_in, 840, pm.ctypes.data)
    assert (pm == SM.power_meter(x[:, :n_in], 840)).all()

def test_nothing_to_do_launches_nothing(eng):
    x = _noise((1000, 2), 1); n0 = eng.launches
    assert eng.spectrum(x, 1024).shape == (1, 0, 1024) and eng.spectrum(x, 256, avg=4).shape == (1, 0, 256)
    assert eng.power_meter(x, 1001).shape == (1, 0)
    assert eng.launches == n0

# ---- the C ABI ----------------------------------------------------------------------------------------------------------------------
def test_residency(eng):
    """iq and out each host or device; the bytes after out untouched."""
    R, n, stride, N, hop, avg = 3, 5000, 5004, 256, 200, 2
    x = np.full((R, stride, 2), 0x5A5A, np.int16); x[:, :n] = _noise((R, n, 2), 40)
    w = api.spectrum_window(N, "hann"); ng = SM.frames_of(n, N, hop) // avg; nb = R * ng * N * 8
    args = dict(iq=x, out=_fill(nb + 16))
    ref = _matrix(lambda p: eng.spectrum_raw(p["iq"], stride, R, n, N, hop, avg, w, p["out"]), args, _each(*args))
    assert (ref["out"][:nb].view(np.int64).reshape(R, ng, N) == SM.spectrum(x[:, :n], N, hop, avg, w)).all() and (ref["out"][nb:] == 0xA5).all()
    nb2 = R * (n // 840) * 4; args = dict(iq=x, out=_fill(nb2 + 16))
    ref2 = _matrix(lambda p: eng.power_meter_raw(p["iq"], stride, R, n, 840, p["out"]), args, _each(*args))
    assert (ref2["out"][:nb2].view(np.uint32).reshape(R, -1) == SM.power_meter(x[:, :n], 840)).all() and (ref2["out"][nb2:] == 0xA5).all()

def test_caller_stream_pinned_back_to_back():
    """Device and page-locked host buffers on a caller stream, two calls back to back, one launch each, timed."""
    e = api.Engine(0)
    try:
        N, n = 1024, 1 << 18; x = _noise((2, n, 2), 77); w = api.spectrum_window(N, "hann")
        want = [SM.spectrum(x[r], N, N // 2, 8, w)[0] for r in range(2)]
        s = torch.cuda.Stream(); s.wait_stream(torch.cuda.current_stream())
        d_in = torch.from_numpy(x).cuda(); h_in = torch.from_numpy(x).pin_memory()
        ng = SM.frames_of(n, N, N // 2) // 8
        with torch.cuda.stream(s):
            d_out = torch.zeros((2, ng, N), dtype=torch.int64, device="cuda"); h_out = torch.zeros((2, ng, N), dtype=torch.int64).pin_memory()
            n0 = e.launches
            e.spectrum_raw(d_in[0].data_ptr(), n, 1, n, N, N // 2, 8, w, d_out[0].data_ptr(), stream=s.cuda_stream)
            e.spectrum_raw(h_in[1].data_ptr(), n, 1, n, N, N // 2, 8, w, d_out[1].data_ptr(), stream=s.cuda_stream)
            e.spectrum_raw(d_in.data_ptr(), n, 2, n, N, N // 2, 8, w, h_out.data_ptr(), stream=s.cuda_stream)
            assert e.launches - n0 == 3
            p_out = torch.zeros((2, n // 4096), dtype=torch.int32, device="cuda")
            e.power_meter_raw(d_in.data_ptr(), n, 2, n, 4096, p_out.data_ptr(), stream=s.cuda_stream)
            e.power_meter_raw(h_in.data_ptr(), n, 2, n, 4096, p_out.data_ptr(), stream=s.cuda_stream)
        s.synchronize()
        assert e.last_kernel_ms() > 0
        for r in range(2):
            assert (d_out[r].cpu().numpy() == want[r]).all() and (h_out[r].numpy() == want[r]).all()
        assert (p_out.cpu().numpy().view(np.uint32) == SM.power_meter(x, 4096)).all()
    finally:
        e.close()

def _spec(eng, iq, stride, R, n, N, hop, avg, win, out):
    return eng._lib.sb200_spectrum(eng._h, V(iq), U64(stride), U32(R), U64(n), U32(N), U64(hop), U32(avg), V(win), V(out), V(0))

def _pwr(eng, iq, stride, R, n, N, out):
    return eng._lib.sb200_power_meter(eng._h, V(iq), U64(stride), U32(R), U64(n), U32(N), V(out), V(0))

def test_invalid_arguments_are_rejected(eng):
    x = _noise((4096, 2), 3); out = np.full(1 << 16, 0x1234, np.int64); before = out.copy()
    xp, op = x.ctypes.data, out.ctypes.data
    w = api.spectrum_window(256, "hann"); wbad = w.copy(); wbad[17] = -1
    n0 = eng.launches
    bad = {"N 0": (xp, 4096, 1, 4096, 0, 256, 1, 0), "N 2": (xp, 4096, 1, 4096, 2, 2, 1, 0), "N 96": (xp, 4096, 1, 4096, 96, 96, 1, 0),
           "N 65536": (xp, 4096, 1, 4096, 65536, 65536, 1, 0), "hop 0": (xp, 4096, 1, 4096, 256, 0, 1, 0),
           "hop > 2^32": (xp, 4096, 1, 4096, 256, (1 << 32) + 1, 1, 0), "avg 0": (xp, 4096, 1, 4096, 256, 256, 0, 0),
           "avg > 2^31": (xp, 4096, 1, 4096, 256, 256, (1 << 31) + 1, 0), "nrows 0": (xp, 4096, 0, 4096, 256, 256, 1, 0),
           "nrows 65": (xp, 4096, 65, 4096, 256, 256, 1, 0), "stride < n_in": (xp, 4092, 1, 4096, 256, 256, 1, 0),
           "stride % 4": (xp, 4098, 1, 4096, 256, 256, 1, 0), "stride > 2^40": (xp, (1 << 40) + 4, 1, 4096, 256, 256, 1, 0),
           "n_in > 2^40": (xp, (1 << 40) + 4, 1, (1 << 40) + 1, 256, 256, 1, 0), "window < 0": (xp, 4096, 1, 4096, 256, 256, 1, wbad.ctypes.data),
           "null iq": (0, 4096, 1, 4096, 256, 256, 1, 0)}
    for name, a in bad.items():
        assert _spec(eng, *a, op) == -1, name
    assert _spec(eng, xp, 4096, 1, 4096, 256, 256, 1, 0, 0) == -1, "null out"
    pbad = {"N 0": (xp, 4096, 1, 4096, 0), "N 65537": (xp, 4096, 1, 4096, 65537), "nrows 0": (xp, 4096, 0, 4096, 128),
            "nrows 65": (xp, 4096, 65, 4096, 128), "stride < n_in": (xp, 4092, 1, 4096, 128), "stride % 4": (xp, 4098, 1, 4096, 128),
            "stride > 2^40": (xp, (1 << 40) + 4, 1, 4096, 128), "n_in > 2^40": (xp, (1 << 40) + 4, 1, (1 << 40) + 1, 128), "null iq": (0, 4096, 1, 4096, 128)}
    for name, a in pbad.items():
        assert _pwr(eng, *a, op) == -1, name
    assert _pwr(eng, xp, 4096, 1, 4096, 128, 0) == -1, "null out"
    d = torch.zeros(4096 * 2 + 8, dtype=torch.int16, device="cuda")
    assert _spec(eng, d.data_ptr() + 4, 4096, 1, 4094, 256, 256, 1, 0, op) == -1, "misaligned device input"
    dout = torch.zeros(1 << 12, dtype=torch.int64, device="cuda")
    assert _spec(eng, xp, 4096, 1, 4096, 256, 256, 1, 0, dout.data_ptr() + 8) == -1, "misaligned device output"
    assert _pwr(eng, d.data_ptr() + 4, 4096, 1, 4094, 128, op) == -1, "misaligned device input"
    assert eng.launches == n0, "a refused call launched"
    assert (out == before).all(), "a refused call wrote out"
    assert _spec(eng, xp, 4096, 1, 4096, 256, 1 << 32, 1 << 31, w.ctypes.data, op) == 0 and eng.launches == n0   # at the limits: no group

# ---- functional loop ------------------------------------------------------------------------------------------------------------------
OCCUPIED = {1: 6000, 4: 3000, 6: 1500}     # channel -> noise amplitude of its 40 Msps row (the other five rows are zero)
# The empty channels hold the fixed-point floor of FFT<1024> (a >> 2 per stage) and the filters' leakage from an occupied neighbour: on
# the H100 about 21 dB below the weakest occupied channel here, so 15 dB leaves room.
MARGIN_DB = 15.0

def test_occupied_channels_found_and_ranked(eng):
    """Three 40 Msps rows at known levels go into an eight-channel odd-stacked grid (sb200_combine_bank, U = 4); sb200_spectrum of the
    160 Msps capture (N = 1024, Hann, avg 16) puts at least MARGIN_DB more energy in each occupied channel than in any empty one, and
    sb200_channelize_bank of the capture, then sb200_power_meter per row, ranks the channels as the spectrum does."""
    M, U, n_in, fs = 8, 4, 40960, 160e6
    rows = np.zeros((M, n_in, 2), np.int16)
    for k, a in OCCUPIED.items(): rows[k] = _noise((n_in, 2), 100 + k, a)
    y = eng.combine_bank(rows, U, W.lowpass(255, 10e6 / 160e6, gain=4), odd=True)
    spec = eng.spectrum(y, 1024, avg=16, window="hann").sum((0, 1)).astype(np.float64)
    _, f = api.fftshift_bins(spec, fs); f = np.fft.ifftshift(f)          # frequency of each bin in natural order
    centres = api.bank_centres(M, fs, odd=True)
    centres = (np.asarray(centres) + fs / 2) % fs - fs / 2
    energy = np.array([spec[np.abs(f - c) <= 8e6].sum() for c in centres])
    occ = sorted(OCCUPIED); empty = [k for k in range(M) if k not in OCCUPIED]
    assert 10 * np.log10(energy[occ].min() / max(energy[empty].max(), 1.0)) >= MARGIN_DB, energy
    ch = eng.channelize_bank(y, M, U, W.lowpass(255, 10e6 / 160e6), odd=True)
    pw = eng.power_meter(ch, 4096).astype(np.float64).mean(1)
    assert list(np.argsort(pw)[::-1][:3]) == list(np.argsort(energy)[::-1][:3]) == sorted(OCCUPIED, key=lambda k: -OCCUPIED[k])
