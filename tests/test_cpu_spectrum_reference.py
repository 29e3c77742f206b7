"""The spectrum and power meters' model (tests/spectrum_model.py) against the reference's OWN code, compiled from its headers where they lie
(oracle/build_ref_meter.sh): FFT<N> of kernel/core/inc/fft_r4dif.h at every N = 4 .. 32768 with its twiddle and bit-reversal tables
(oracle/_ref/libfftn_ref.so, with the debug tap of oracle/build_ref_fft.sh), and TSpecMeter<N> / TPowerMeter<N> of
kernel/sdl/inc/sdlmeasure.hpp (oracle/_ref/libmeter_ref.so).  The model is what tests/test_gpu_spectrum.py holds the device to where the
compiled meters cannot be used directly (overlap, windows, group sums).  Skipped where oracle/_ref was not built."""
import ctypes as C, os
import numpy as np, pytest
import oracle_py
import spectrum_model as SM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FFTN = os.path.join(ROOT, "oracle", "_ref", "libfftn_ref.so")
METER = os.path.join(ROOT, "oracle", "_ref", "libmeter_ref.so")
SIZES = [1 << k for k in range(2, 16)]
POWER_SIZES = [1, 3, 4, 5, 128, 840, 4096, 65536]

pytestmark = pytest.mark.skipif(not (os.path.exists(FFTN) and os.path.exists(METER)), reason="oracle/_ref/libfftn_ref.so / libmeter_ref.so not built (needs the reference tree)")

def _p(a): return a.ctypes.data_as(C.c_void_p)

def ref_fft(x):
    """Compiled FFT<N> of int16 [F, N, 2] -> (int16 [F, N, 2], tap counts [clip add, clip sub, pack drop, madd wrap])."""
    lib = C.CDLL(FFTN); x = np.ascontiguousarray(x, np.int16); out = np.zeros_like(x)
    assert lib.ref_fftn(C.c_uint32(x.shape[1]), C.c_size_t(x.shape[0]), _p(x), _p(out)) == 0
    d = (C.c_uint64 * 4)(); lib.ref_fftn_debug(d)
    return out, list(d)

def ref_spec(x):
    lib = C.CDLL(METER); x = np.ascontiguousarray(x, np.int16); out = np.zeros(x.shape[:2], np.int32)
    assert lib.ref_spec_meter(C.c_uint32(x.shape[1]), C.c_size_t(x.shape[0]), _p(x), _p(out)) == 0
    return out

def ref_power(x):
    lib = C.CDLL(METER); x = np.ascontiguousarray(x, np.int16); out = np.zeros(x.shape[0], np.int32)
    assert lib.ref_power_meter(C.c_uint32(x.shape[1]), C.c_size_t(x.shape[0]), _p(x), _p(out)) == 0
    return out.view(np.uint32)

def inputs(N, seed=0):
    """Impulses (at 0, 1, N/2 and N-1), full-scale tones at bins 0, 1, N/4, N/2 and N-1, random int16, all -32768, alternating rails, and
    random rails: int16 [F, N, 2]."""
    rng = np.random.default_rng(seed + N)
    n = np.arange(N); fr = []
    for p in (0, 1, N // 2, N - 1):
        for v in ((32767, 0), (-32768, -32768), (1, -1)):
            f = np.zeros((N, 2), np.int64); f[p] = v; fr.append(f)
    for k in (0, 1, N // 4, N // 2, N - 1):
        a = 2 * np.pi * k * n / N
        fr.append(np.stack([np.rint(32767 * np.cos(a)), np.rint(32767 * np.sin(a))], 1))
        fr.append(np.stack([np.where(np.cos(a) >= 0, 32767, -32768), np.where(np.sin(a) >= 0, 32767, -32768)], 1))
    fr.append(np.full((N, 2), -32768)); fr.append(np.full((N, 2), 32767))
    fr.append(np.where((n % 2 == 0)[:, None], 32767, -32768) * np.ones((1, 2), np.int64))
    fr.append(np.where((n % 2 == 0)[:, None], np.array([32767, -32768]), np.array([-32768, 32767])))
    F = max(8, 8192 // N)
    rnd = rng.integers(-32768, 32768, (F, N, 2)); rails = np.where(rng.integers(0, 2, (F, N, 2)) == 1, 32767, -32768)
    return np.concatenate([np.stack(fr), rnd, rails]).astype(np.int16)

@pytest.mark.parametrize("N", SIZES)
def test_fft_equals_compiled(N):
    x = inputs(N)
    got, taps = ref_fft(x)
    assert (SM.fft(x) == got).all()
    assert taps[3] == 0                    # no pmaddwd wraps: a twiddle half is never -32768 (and ~w.im <= 32766), so no lane is -32768 twice

@pytest.mark.parametrize("N", SIZES)
def test_spec_meter_equals_compiled(N):
    x = inputs(N, 1)
    assert (SM.spec_meter(x) == ref_spec(x)).all()

def test_fft8_rails_reach_the_clips():
    """Every rail vector of FFT<8> (2^16 of them): FFTSSEEx<8>'s last saturating adds clip (m0 + m1 reaches 16382 + 23165), the model
    still equals the compiled transform, and TSpecMeter<8> too."""
    b = (np.arange(65536)[:, None] >> np.arange(16)) & 1
    x = np.where(b == 1, 32767, -32768).astype(np.int16).reshape(65536, 8, 2)
    got, taps = ref_fft(x)
    assert taps[0] > 0 and taps[3] == 0, taps
    assert (SM.fft(x) == got).all() and (SM.spec_meter(x) == ref_spec(x)).all()

@pytest.mark.parametrize("N", [16, 32, 64, 1024, 32768])
def test_fft_pack_drops(N):
    """Random full-scale frames reach mul_shift's wrapping pack (significant bits dropped) at every stage size tried."""
    x = np.random.default_rng(N).integers(-32768, 32768, (max(4, 65536 // N), N, 2)).astype(np.int16)
    got, taps = ref_fft(x)
    assert taps[2] > 0, taps
    assert (SM.fft(x) == got).all()

def test_fft64_equals_the_fft_oracle():
    """At N = 64 the model also equals oracle/_ref/libfft_ref.so's FFT<64>, the transform the receivers' tests hold the device to."""
    if not oracle_py.ref_fft_available(): pytest.skip("oracle/_ref/libfft_ref.so not built")
    x = inputs(64, 2)
    assert (SM.fft(x) == oracle_py.ref_fft64(x)).all()

@pytest.mark.parametrize("N", SIZES)
def test_tables_equal_compiled(N):
    """gen_twiddle(N, M) is FFT_GetTwiddleConst<N, M> for M = 1, 2, 3 and bitrev(N) is FFTLUTMapTable<N>; at N = 8 the one table is
    wFFTLUT8 = (W^0, W^1, W^0, W^3), which the device and the model state as constants."""
    lib = C.CDLL(FFTN); tw = np.zeros((3, max(N // 4, 4), 2), np.int16); mp = np.zeros(N, np.int16)
    assert lib.ref_fftn_tables(C.c_uint32(N), _p(tw), _p(mp)) == 0
    assert (mp == SM.bitrev(N)).all()
    if N == 8:
        assert (tw[0] == [[32767, 0], [23169, -23169], [32767, 0], [-23169, -23169]]).all()
    elif N >= 16:
        for M in (1, 2, 3): assert (tw[M - 1] == SM.gen_twiddle(N, M)).all(), M

@pytest.mark.parametrize("N", POWER_SIZES)
def test_power_meter_equals_compiled(N):
    rng = np.random.default_rng(N)
    B = max(4, 65536 // N)
    x = [rng.integers(-32768, 32768, (B, N, 2)), np.full((1, N, 2), -32768), np.full((1, N, 2), 32767), rng.integers(-300, 300, (B, N, 2)),
         np.where(rng.integers(0, 2, (B, N, 2)) == 1, 32767, -32768)]
    x = np.concatenate(x).astype(np.int16)
    assert (SM.power_meter_blocks(x) == ref_power(x)).all()

def test_power_meter_negative_vector_sum():
    """A 4-sample vector whose wrapping SquaredNorm sum is negative divides as 2^64 + v (size_t N): all -32768 gives four INT32_MIN lanes
    (sum 0), three -32768 samples and one (16384, 0) give 3 INT32_MIN + 2^28, negative; the compiled meter agrees with the model."""
    for N in (4, 5, 128, 840):
        x = np.full((3, N, 2), -32768, np.int64); x[1, 3::4] = (16384, 0); x[2, 3::4] = (0, 1)
        x = x.astype(np.int16)
        e = SM.squared_norm(x.astype(np.int64))
        s = SM._w32(e[1, :4].sum())
        assert s < 0
        assert (SM.power_meter_blocks(x) == ref_power(x)).all()

def test_spectrum_model_groups_and_hops():
    """spectrum() with hop = N, avg = 1 and no window is TSpecMeter<N> frame by frame; with overlap and avg it sums the same frames."""
    rng = np.random.default_rng(3)
    for N in (4, 64, 1024):
        x = rng.integers(-32768, 32768, (5 * N + 3, 2)).astype(np.int16)
        assert (SM.spectrum(x, N)[0] == ref_spec(x[:5 * N].reshape(5, N, 2))).all()
        hop = max(1, N // 3); fr = SM.frames_of(len(x), N, hop)
        idx = (np.arange(fr) * hop)[:, None] + np.arange(N)
        p = ref_spec(x[idx]).astype(np.int64)
        assert (SM.spectrum(x, N, hop, avg=2)[0] == p[:fr // 2 * 2].reshape(-1, 2, N).sum(1)).all()
