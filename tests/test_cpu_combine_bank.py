"""The filter-bank combiner's model (tests/combine_bank_model.py, the arithmetic of sb200_combine_bank in include/sora_b200.h) without a
GPU: the direct and vectorised forms against each other over every M and U | M, the bound against sb200_combine's model, tones and
leakage, windows, n_out and accumulate, then the oracle transmitters' frames sent through the model bank, taken apart again and decoded by
the CPU oracle.  test_gpu_combine_bank.py runs the device against the same model."""
import numpy as np, pytest
import oracle_py
import wideband_inputs as W
import bank_model as B
import combine_model as CM
import combine_bank_model as CB
import combine_rational_model as CR
import rational_model as R
from sora_b200 import api
from test_cpu_channelize import _full_scale, _decoded, decode_11a
from test_cpu_channelize_rational import TAPS_160_44
from test_cpu_combine import _mpdu, _psdus, rows_of
from test_cpu_combine_rational import TAPS_44_160

GRID = [(M, U) for M in (2, 4, 8, 16, 32, 64) for U in (1, 2, 4, 8, 16, 32, 64) if M % U == 0]
TAPS_TX = W.lowpass(255, 10e6 / 160e6, gain=4)          # 40 -> 160 Msps, M = 8, U = 4: each branch near unity, -6 dB at 10 MHz

def max_taps(M, U):
    """The largest ntaps the call accepts: odd, <= 1023 and <= 2048 U / M."""
    return min(1023, 2048 * U // M - 1)

def combine_taps(M, U):
    """A low-pass within both calls' limits (ntaps <= 255 and <= 2048 U / M, every branch sum <= 65535), for comparing with sb200_combine."""
    nt = min(255, max_taps(M, U)); t = W.lowpass(nt, 0.45 / M, gain=U)
    s = max(int(np.abs(t[r::U].astype(np.int64)).sum()) for r in range(U))
    return t if s <= 65535 else W.lowpass(nt, 0.45 / M, gain=U * 0.98 * 65535 / s)

def _rows(M, n, seed, amp=32768):
    return np.random.default_rng(seed).integers(-amp, amp, (M, n, 2)).astype(np.int16)

@pytest.mark.parametrize("M,U", GRID)
def test_direct_equals_window(M, U):
    rng = np.random.default_rng(M * 100 + U)
    n_in = 9 + 96 // U
    for odd in (0, 1):
        for nt in sorted({1, 3, 2 * U + 1, max_taps(M, U)}):
            x = _rows(M, n_in, M + U + nt + odd)
            taps = rng.integers(-32768, 32768, nt).astype(np.int16)
            n_out = U * n_in + nt // 2 + 3                                   # past the rows' support: the filter's tail
            assert (CB.direct(x, U, odd, taps, n_out) == CB.combine_bank(x, U, odd, taps, n_out)).all(), (M, U, odd, nt)

@pytest.mark.parametrize("M", [2, 4, 8, 16])
def test_within_the_bound_of_the_combiner(M):
    """Where nothing saturates, the bank is sb200_combine at channels {(2k + o) 2^31 / M, 0, 4096} within the header's bound."""
    rng = np.random.default_rng(M)
    for U in sorted({1, M // 2, M}):
        for odd in (0, 1):
            taps = combine_taps(M, U)
            x = _rows(M, 700, 7 * M + U + odd, 6000 // M)
            x[rng.integers(M)] = 0                                           # K < M: a zero row adds no rounding
            assert max(int(np.abs(taps[r::U].astype(np.int64)).sum()) for r in range(U)) <= 65535
            bank = CB.combine_bank(x, U, odd, taps).astype(np.int64)
            comb = CM.combine(x, CB.channels(M, odd), U, taps).astype(np.int64)
            assert np.abs(bank).max() < 32767 and np.abs(comb).max() < 32767
            assert np.abs(bank - comb).max() <= CB.combine_bound(x, taps, U), (M, U, odd)

@pytest.mark.parametrize("odd", [0, 1])
def test_a_row_comes_out_at_its_centre(odd):
    """A constant row k comes out as a tone at bank_centres(M, fs, o)[k]; a tone at delta of the row rate at that centre + delta, with its
    leakage into every other channel's band (taken apart by the bank channelizer's model) more than 50 dB down."""
    M, U, fs = 8, 4, 160e6; n = 6000; A = 12000
    for k, delta in ((1, 0.0), (6, 1.5e6), (3, -2e6), (4, 0.7e6)):
        z = A * np.exp(2j * np.pi * delta / (fs / U) * np.arange(n))
        x = np.zeros((M, n, 2), np.int16); x[k] = np.stack([np.round(z.real), np.round(z.imag)], 1)
        y = CB.combine_bank(x, U, odd, TAPS_TX)
        v = (y[:, 0] + 1j * y[:, 1].astype(np.float64))[600:-600]
        ph = np.unwrap(np.angle(v))
        f = (ph[-1] - ph[0]) / (len(ph) - 1) / (2 * np.pi) * fs
        assert abs(f - (api.bank_centres(M, fs, odd)[k] + delta)) < 1e3, (odd, k, f)
        assert abs(np.abs(v).mean() - A) < 0.02 * A
        back = B.bank(y, M, U, odd, B.TAPS_BANK)[:, 300:-300].astype(np.float64)
        mag = np.abs(back[..., 0] + 1j * back[..., 1])
        assert all(mag[j].max() < mag[k].mean() * 10 ** (-50 / 20) for j in range(M) if j != k), (odd, k)

def test_a_window_of_outputs_needs_only_its_inputs():
    for M, U, odd, nt in ((8, 4, 1, 255), (16, 1, 0, 127), (64, 64, 1, 1023), (2, 2, 0, 1023)):
        x = _rows(M, 900 // U + 7, M + U); taps = W.lowpass(nt, 0.4 / M, gain=U)
        n_out = U * x.shape[1] + 40; full = CB.combine_bank(x, U, odd, taps, n_out)
        for n0, n1 in ((0, 7), (0, n_out), (n_out // 2 - 5, n_out // 2 + 9), (n_out - 3, n_out), (5, 5)):
            assert (CB.window(x, M, U, odd, taps, n0, n1) == full[n0:n1]).all(), (M, U, n0, n1)

def test_n_out_cuts_or_extends():
    """n_out shorter than U n_in cuts the capture, equal is the default, longer adds the filter's tail and then zeros."""
    M, U = 8, 4; x = _rows(M, 300, 3, 3000)
    full = CB.combine_bank(x, U, 1, TAPS_TX); n = len(full); assert n == U * 300
    assert (CB.combine_bank(x, U, 1, TAPS_TX, n - 101) == full[:n - 101]).all()
    long = CB.combine_bank(x, U, 1, TAPS_TX, n + 400)
    assert (long[:n] == full).all() and long[n:n + 100].any() and not long[n + len(TAPS_TX) // 2 + 1:].any()

def test_accumulate_is_one_saturation():
    """With accumulate, y = sat16(a + the call's rounded sum): one saturation, on random and on rail contents of out."""
    M, U = 16, 2; x = _rows(M, 500, 5, 1500); taps = W.lowpass(127, 0.4 / M, gain=U)
    plain = CB.combine_bank(x, U, 1, taps).astype(np.int64); n = len(plain)
    assert np.abs(plain).max() < 32767
    rng = np.random.default_rng(6)
    for a in (rng.integers(-32768, 32768, (n, 2)), np.full((n, 2), 32767), np.full((n, 2), -32768),
              np.where(rng.random((n, 2)) < 0.5, 32767, -32768)):
        a = a.astype(np.int16)
        got = CB.combine_bank(x, U, 1, taps, acc=a)
        assert (got == np.clip(a.astype(np.int64) + plain, -32768, 32767)).all()


# ---- transmit -> bank combiner -> bank channelizer -> receive, through the CPU oracle ----------------------------------------------------
RATES_OCTET = (6000, 9000, 12000, 18000, 24000, 36000, 48000, 54000)

def frames_octet(channels=range(8)):
    """The oracle transmitter's 802.11a frames (COMPLEX8 x 20) in the rows of the M = 8 grid, one per channel at its own rate and start
    -> (rows int16 [8, n, 2], {row: [mpdu]}, {row: (start, rate, seed)})."""
    chans, mpdus, plan = [[] for _ in range(8)], {}, {}
    for ci in channels:
        rate = RATES_OCTET[ci]; t = 300 + 350 * ci; seed = 1 + 9 * ci
        m = _mpdu(120 + 40 * ci, 0x3E8B0000 + ci)
        chans[ci].append((t, oracle_py.tx11a_modulate(m, rate, seed).astype(np.int16) * 20))
        mpdus[ci] = [m]; plan[ci] = (t, rate, seed)
    n = max(s + len(f) for fr in chans for s, f in fr) + 400
    return rows_of(chans, n), mpdus, plan

def test_octet_through_both_banks():
    """Eight 802.11a frames at eight rates on the odd-stacked grid of M = 8 (+-10 / 30 / 50 / 70 MHz of 160 Msps), combined by the bank
    (U = 4) and taken apart by the bank channelizer (D = 4): every PSDU arrives on its own channel, with a good FCS, and nothing else."""
    rows, mpdus, _ = frames_octet()
    y = CB.combine_bank(rows, 4, 1, TAPS_TX)
    assert np.abs(y.astype(np.int64)).max() < 32767
    back = B.bank(y, 8, 4, 1, B.TAPS_BANK)
    for c, (r, o) in enumerate(decode_11a(back)):
        assert _decoded(r, o, lambda L: L) == _psdus(mpdus[c]), c

# The mixed capture: OFDM on bank channels 0, 3, 4, 7 (+10, +70, -70, -10 MHz), rows 1 and 2 (+30, +50 MHz) zero, and one 802.11b row at
# 44 Msps added over those two empty channels, centred at +40 MHz, by the rational combiner (U / D = 40 / 11) with accumulate.
OFDM_ROWS = (0, 3, 4, 7)
F_11B, GAIN_11B = 40e6, 2048
FRAMES_11B = ((2000, 70), (11000, 120))

def frames_11b_row():
    """The oracle's 802.11b frames (COMPLEX8 << 6, 44 Msps) in one row -> (int16 [n, 2], [mpdu, ...])."""
    fr, ms, t = [], [], 500
    for j, (rate, nb) in enumerate(FRAMES_11B):
        m = _mpdu(nb, 0x3E8C0000 + j); f = oracle_py.tx11b_modulate(m, rate).astype(np.int16) << 6
        fr.append((t, f)); ms.append(m); t += len(f) + 900
    return rows_of([fr])[0], ms

def mixed_capture():
    """-> (capture int16 [n_out, 2], the bank's output alone, OFDM rows, {row: [mpdu]}, the 802.11b row, its mpdus)."""
    rows, mpdus, _ = frames_octet(OFDM_ROWS)
    rb, mb = frames_11b_row()
    n_out = max(4 * rows.shape[1], -(-40 * len(rb) // 11)) + 400; n_out += (-n_out) % 4
    first = CB.combine_bank(rows, 4, 1, TAPS_TX, n_out)
    y = CR.combine_rational(rb[None], [(W.phase_inc(F_11B, 160e6), 0, GAIN_11B)], 40, 11, TAPS_44_160, n_out, acc=first)
    return y, first, rows, mpdus, rb, mb

def test_mixed_capture():
    """OFDM rows through the bank and an 802.11b row over two empty channels through the rational combiner, in one capture: the bank
    channelizer returns every OFDM PSDU on its own channel, the rational channelizer every 802.11b PSDU (without its last FCS byte)."""
    y, _, _, mpdus, _, mb = mixed_capture()
    assert np.abs(y.astype(np.int64)).max() < 32767
    back = B.bank(y, 8, 4, 1, B.TAPS_BANK)
    for c, (r, o) in zip(OFDM_ROWS, decode_11a(back[list(OFDM_ROWS)])):
        assert _decoded(r, o, lambda L: L) == _psdus(mpdus[c]), c
    row_b = R.channelize_rational(y, [(W.phase_inc(F_11B, 160e6), 0)], 11, 40, TAPS_160_44)[0]
    r, o = oracle_py.rx11b_run(row_b, max_frames=16, out_stride=4096)
    assert _decoded(r, o, lambda L: L - 1) == [p[:-1] for p in _psdus(mb)]
    assert (r["status"] == oracle_py.E_FRAME_OK).all()
