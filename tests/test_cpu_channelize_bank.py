"""The filter-bank channelizer's model (tests/bank_model.py, the arithmetic of sb200_channelize_bank in include/sora_b200.h) without a
GPU: the direct and polyphase forms against each other, the table identities the kernel relies on, the relation to sb200_channelize's
model, tones, windows, and 802.11a / n captures taken apart by the model and decoded by the CPU oracle's continuous-capture receivers.
test_gpu_channelize_bank.py runs the same captures through the device."""
import ctypes as C
import numpy as np, pytest
import oracle_py
import wideband_inputs as W
import bank_model as B
from sora_b200 import api
from test_cpu_channelize import CCA_WIDE, _full_scale, _decoded, decode_11a

GRID = [(M, D) for M in (2, 4, 8, 16, 32, 64) for D in (1, 2, 4, 8, 16, 32, 64) if M % D == 0]

@pytest.mark.parametrize("M,D", GRID)
def test_direct_equals_polyphase(M, D):
    rng = np.random.default_rng(M * 100 + D)
    x = _full_scale(300 + 7 * M, M + D)
    for odd in (0, 1):
        taps = rng.integers(-400, 400, [1, 3, 2 * M + 1, 4 * M + 3][(M + D + odd) % 4]).astype(np.int16)
        assert (B.direct(x, M, D, odd, taps) == B.bank(x, M, D, odd, taps)).all(), (M, D, odd)

def test_nco_identities():
    """NCO[i + 2048] = -NCO[i] and NCO[i + 1024] = (-S, C), exactly, for all 4096 entries: the pairs p, p + M/2 of the DFT are +-1 / +-j."""
    i = np.arange(4096); C_, S_ = W.NCO[i, 0], W.NCO[i, 1]
    assert (W.NCO[(i + 2048) % 4096] == -W.NCO[i]).all()
    assert (W.NCO[(i + 1024) % 4096, 0] == -S_).all() and (W.NCO[(i + 1024) % 4096, 1] == C_).all()

@pytest.mark.parametrize("M", [2, 4, 8, 16, 32, 64])
def test_within_2_lsb_of_the_channelizer(M):
    """Where neither side saturates (|x| <= 23170, |rotated x| <= 32767), channel k is sb200_channelize at phase_inc = (2k + o) 2^31 / M
    within its two roundings."""
    rng = np.random.default_rng(M)
    x = rng.integers(-23170, 23171, (1500, 2)).astype(np.int16); taps = W.lowpass(63, 0.4 / M)
    for odd in (0, 1):
        for D in sorted({1, M // 2, M}):
            ch = W.channelize(x, B.phase_incs(M, odd), D, taps).astype(np.int64)
            assert np.abs(ch - B.bank(x, M, D, odd, taps)).max() <= 2, (M, odd, D)

@pytest.mark.parametrize("odd", [0, 1])
def test_a_tone_comes_out_of_its_channel(odd):
    """A tone at channel k's centre plus delta comes out of channel k at delta of the output rate, and more than 50 dB lower elsewhere."""
    M, D, fs = 8, 4, 160e6; n = 20000; A = 12000; taps = B.TAPS_BANK
    for k, delta in ((1, 1.5e6), (6, -2e6), (4, 0.7e6)):
        f = api.bank_centres(M, fs, odd)[k] + delta
        z = A * np.exp(2j * np.pi * f / fs * np.arange(n))
        y = B.bank(np.stack([np.round(z.real), np.round(z.imag)], 1).astype(np.int16), M, D, odd, taps)[:, 200:-200].astype(np.float64)
        v = y[..., 0] + 1j * y[..., 1]
        ph = np.unwrap(np.angle(v[k]))
        assert abs((ph[-1] - ph[0]) / (len(ph) - 1) / (2 * np.pi) * fs / D - delta) < 1e3, (odd, k)
        assert abs(np.abs(v[k]).mean() - A * taps.sum() / 32768) < 0.02 * A
        assert all(np.abs(v[j]).max() < A * 10 ** (-50 / 20) for j in range(M) if j != k), (odd, k)

def test_bank_centres():
    assert list(api.bank_centres(8, 160e6)) == [0, 20e6, 40e6, 60e6, -80e6, -60e6, -40e6, -20e6]
    assert list(api.bank_centres(8, 160e6, odd=True)) == [10e6, 30e6, 50e6, 70e6, -70e6, -50e6, -30e6, -10e6]

def test_a_window_of_outputs_needs_only_its_inputs():
    x = _full_scale(3001, 6); taps = W.lowpass(511, 0.02)
    for M, D, odd in ((8, 4, 1), (16, 1, 0), (64, 64, 1)):
        full = B.bank(x, M, D, odd, taps); n_out = full.shape[1]
        for m0, m1 in ((0, 7), (0, n_out), (n_out // 2 - 5, n_out // 2 + 9), (n_out - 3, n_out)):
            assert (B.window(x, M, D, odd, taps, m0, m1) == full[:, m0:m1]).all(), (M, D, m0, m1)


# ---- end to end through the CPU oracle --------------------------------------------------------------------------------------------------
def bank_rows_11a():
    """capture_11a (channels at -60 / -20 / +20 / +60 MHz) by the even-stacked bank of M = 8, D = 4: channels 5 / 7 / 1 / 3 carry
    them, 0 / 2 / 4 / 6 nothing.  -> (rows [8, n_out, 2], {row: psdus})."""
    iq, fcs, ps = W.capture_11a()
    k = [int(round(f / 20e6)) % 8 for f in fcs]
    return B.bank(iq, 8, 4, 0, B.TAPS_BANK), {k[c]: ps[c] for c in range(len(fcs))}

def bank_rows_11n():
    (a0, a1), fcs, ps = W.capture_11n()
    k = [int(round(f / 20e6)) % 8 for f in fcs]
    return B.bank(a0, 8, 4, 0, B.TAPS_BANK), B.bank(a1, 8, 4, 0, B.TAPS_BANK), {k[c]: ps[c] for c in range(len(fcs))}

def bank_rows_octet():
    iq, fcs, ps = B.capture_11a_octet()
    k = [int(np.argmin(np.abs(api.bank_centres(8, W.FS_11A_WIDE, True) - f))) for f in fcs]
    return B.bank(iq, 8, 4, 1, B.TAPS_BANK), {k[c]: ps[c] for c in range(len(fcs))}

def _check_11a(rows, want):
    for c, (r, o) in enumerate(decode_11a(rows)):
        assert _decoded(r, o, lambda L: L) == [bytes(p) for p in want.get(c, [])], c

def test_bank_11a():
    """Even stacking on capture_11a: every PSDU out of its own channel, no frame out of the four empty ones."""
    _check_11a(*bank_rows_11a())

def test_bank_11a_odd_stacking():
    """Eight adjacent channels, one 10 dB above its neighbours, odd stacking: every PSDU delivered on its own channel."""
    rows, want = bank_rows_octet()
    assert sorted(want) == list(range(8))
    _check_11a(rows, want)

def test_bank_11n():
    """One bank per antenna of capture_11n (2x2 channels at -20 / +20 MHz): channels 7 and 1 decode, the others yield no frame."""
    r0, r1, want = bank_rows_11n()
    for c in range(8):
        r, o = oracle_py.rx11n_run(r0[c], r1[c], max_frames=16, out_stride=2048)
        assert _decoded(r, o, lambda L: L) == [bytes(p) for p in want.get(c, [])], c
