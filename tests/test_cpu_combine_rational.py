"""The rational-rate combiner's model (tests/combine_rational_model.py, the arithmetic of sb200_combine_rational in include/sora_b200.h)
and what it is for, without a GPU: its properties, then the oracle transmitters' 802.11b frames (44 Msps) and OFDM frames (40 Msps) combined
into one 2.4 GHz capture with two calls into one buffer, at 160 and at 176 Msps, passed through the channel simulator's model with noise,
channelized again by the rational channelizer's model and decoded by the CPU oracle, every channel on its own.  test_gpu_combine_rational.py
runs the same chain on the device."""
import numpy as np, pytest
import oracle_py
import wideband_inputs as W
import combine_model as CM
import combine_rational_model as CR
import rational_model as R
import sim_model as SM
from test_cpu_channelize import _full_scale
from test_cpu_channelize_rational import PLANS, decode_24ghz
from test_cpu_combine import TAPS_UP, TAPS_UP_11B, _mpdu, _psdus, rows_of

def test_decim_1_is_the_combiner():
    rows = np.stack([_full_scale(1001, 20 + k) for k in range(3)]); taps = W.lowpass(127, 0.1, gain=4)
    ch = [(0, 0, 4096), (2 ** 29, 0, 65535), (0x9E3779B9, 0xDEADBEEF, 1234)]
    for u in range(1, 17):
        assert (CR.combine_rational(rows, ch, u, 1, taps) == CM.combine(rows, ch, u, taps)).all(), u

def test_an_impulse_returns_the_branch_taps():
    """x = -32768 at i0 through channel (0, 0, 4096): y(n) = -taps[U i0 - D n + c] wherever that index is a tap, zero elsewhere."""
    for U, D in ((40, 11), (22, 5), (4, 3), (64, 15), (17, 16)):
        taps = np.random.default_rng(U).integers(-3000, 3000, 10 * U + 1).astype(np.int16); c = len(taps) // 2; i0 = 57
        x = np.zeros((1, 120, 2), np.int16); x[0, i0, 0] = -32768
        y = CR.combine_rational(x, [(0, 0, 4096)], U, D, taps)
        k = U * i0 - D * np.arange(len(y)) + c; at = (k >= 0) & (k < len(taps))
        assert at.sum() > 0 and (y[at, 0] == -taps[k[at]]).all() and (y[~at] == 0).all() and (y[:, 1] == 0).all(), (U, D)

TAPS_44_160 = W.lowpass(1761, 12e6 / 1.76e9, gain=40)          # 44 -> 160 Msps, (40, 11): 45 taps per branch
TAPS_40_176 = W.lowpass(1321, 11.3e6 / 880e6, gain=22)         # 40 -> 176 Msps, (22, 5): 61 taps per branch

def test_a_constant_becomes_a_tone_and_a_tone_moves_by_fc():
    """A constant row comes out at f_c with branch r's gain on the outputs of that branch; a tone at delta of the row rate comes out at
    f_c + delta of the capture rate."""
    fs, f, U, D, A = 160e6, -25e6, 40, 11, 8000; taps = TAPS_44_160; c = len(taps) // 2; inc = W.phase_inc(f, fs); fr = fs * D / U
    x = np.zeros((1, 4000, 2), np.int16); x[0, :, 0] = A
    y = CR.combine_rational(x, [(inc, 0, 4096)], U, D, taps)[400:-400].astype(np.float64); n = np.arange(400, 400 + len(y))
    base = (y[:, 0] + 1j * y[:, 1]) * np.exp(-2j * np.pi * inc / 2 ** 32 * n)
    bsum = np.array([taps[(c - D * m) % U::U].astype(np.int64).sum() for m in n])   # branch of output n: taps j = c - D n (mod U)
    assert np.abs(base - A * bsum / 32768).max() < 0.01 * A
    delta = 3e6
    z = A * np.exp(2j * np.pi * delta / fr * np.arange(4000) + 0.4j); x = np.stack([np.round(z.real), np.round(z.imag)], 1)[None].astype(np.int16)
    y = CR.combine_rational(x, [(inc, 0, 4096)], U, D, taps)[400:-400].astype(np.float64)
    v = (y[:, 0] + 1j * y[:, 1]) * np.exp(-2j * np.pi * (f + delta) / fs * n)
    assert abs(abs(v.mean()) - A) < 0.02 * A and np.abs(v - v.mean()).max() < 0.02 * A

def test_a_window_of_outputs_needs_only_its_inputs():
    rows = np.stack([_full_scale(701, 6 + k) for k in range(3)]); ch = [(0, 0, 4096), (2 ** 29, 0, 65535), (0x9E3779B9, 0xDEADBEEF, 1234)]
    for U, D, taps in ((4, 1, TAPS_UP), (40, 11, TAPS_44_160), (22, 5, TAPS_40_176), (17, 16, W.lowpass(255, 0.02, gain=17))):
        n_out = -(-U * 701 // D) + 50; full = CR.combine_rational(rows, ch, U, D, taps, n_out)
        for n0, n1 in ((0, 7), (0, n_out), (n_out // 2 - 5, n_out // 2 + 90), (n_out - 3, n_out), (3, 5)):
            assert (CR.combine_rational_window(rows, ch, U, D, taps, n0, n1) == full[n0:n1]).all(), (U, D, n0, n1)

def test_n_out_cuts_or_extends():
    """n_out shorter than ceil(U n_in / D) is a prefix; longer adds the filter's tail and then zeros."""
    rows = np.stack([_full_scale(300, 9)]) // 4; ch = [(W.phase_inc(10e6, 160e6), 7, 4096)]; U, D, taps = 40, 11, TAPS_44_160
    full = CR.combine_rational(rows, ch, U, D, taps); n = len(full)
    assert n == -(-U * 300 // D)
    assert (CR.combine_rational(rows, ch, U, D, taps, n - 100) == full[:n - 100]).all()
    long = CR.combine_rational(rows, ch, U, D, taps, n + 400)
    assert (long[:n] == full).all() and np.abs(long[n:n + 50].astype(np.int64)).max() > 0 and (long[n + 300:] == 0).all()

def test_accumulate_is_one_saturation():
    """accumulate: y = sat16(a + sum) exactly, on random and rail contents; two calls equal one joint call wherever no partial sum
    leaves int16."""
    rng = np.random.default_rng(12); U, D, taps = 22, 5, TAPS_40_176
    rows = rng.integers(-6000, 6000, (3, 500, 2)).astype(np.int16)
    ch = [(W.phase_inc(-30e6, 176e6), 0, 4096), (W.phase_inc(25e6, 176e6), 0x12345678, 9000), (0, 0, 3000)]
    n_out = -(-U * 500 // D)
    plain = CR.combine_rational(rows, ch, U, D, taps, n_out).astype(np.int64)
    assert np.abs(plain).max() < 32767                                                 # the sum is not clipped, so sat16(a + sum) is exact here
    for a in (rng.integers(-32768, 32768, (n_out, 2)), np.where(rng.random((n_out, 2)) < 0.5, -32768, 32767)):
        a = a.astype(np.int16)
        got = CR.combine_rational(rows, ch, U, D, taps, n_out, acc=a)
        assert (got == np.clip(a.astype(np.int64) + plain, -32768, 32767)).all()
    first = CR.combine_rational(rows[:1], ch[:1], U, D, taps, n_out)
    two = CR.combine_rational(rows[1:], ch[1:], U, D, taps, n_out, acc=first)
    assert (two == plain).all()

def test_the_rational_channelizer_undoes_it():
    """A tone sent with (U, D) and received with (D, U) and the same NCO pair comes back at its amplitude within 2 %."""
    A = 6000
    for fs, U, D, taps, tb, f in ((160e6, 40, 11, TAPS_44_160, PLANS[160e6][1], -25e6), (176e6, 22, 5, TAPS_40_176, PLANS[176e6][3], 0.0)):
        fr = fs * D / U; z = A * np.exp(2j * np.pi * 1.5e6 / fr * np.arange(3000) + 1.1j)
        x = np.stack([np.round(z.real), np.round(z.imag)], 1).astype(np.int16)
        inc = W.phase_inc(f, fs)
        y = CR.combine_rational(x[None], [(inc, 0, 4096)], U, D, taps)
        back = R.channelize_rational(y, [(inc, 0)], D, U, tb)[0][300:-300].astype(np.float64)
        m = np.arange(300, 300 + len(back)); v = (back[:, 0] + 1j * back[:, 1]) * np.exp(-2j * np.pi * 1.5e6 / fr * m)
        assert abs(abs(v.mean()) - A) < 0.02 * A and np.abs(v - v.mean()).max() < 0.02 * A, fs


# ---- transmit -> combine (two calls into one buffer) -> channelize -> receive, through the CPU oracle ------------------------------------
# fs -> ((U, D) of the 802.11b rows at 44 Msps, their taps, (U, D) of the OFDM row at 40 Msps, its taps).  The channel centres and kinds
# are capture_24ghz's: 802.11b at -25 and +25 MHz, OFDM at 0 Hz.
TX_PLANS = {160e6: ((40, 11), TAPS_44_160, (4, 1), TAPS_UP), 176e6: ((4, 1), TAPS_UP_11B, (22, 5), TAPS_40_176)}
GAIN_B, GAIN_A = 2048, 8192                             # the OFDM row 12 dB above each 802.11b row: its 36 Mbps frame decodes beside them
FRAMES_24 = (((2000, 70), (11000, 40)), ((24000, 150), (6000, 90), (36000, 200)), ((5500, 60), (11000, 50)))   # (rate kbps, bytes) per channel

def frames_24ghz():
    """The oracle transmitters' frames in rows: 802.11b (COMPLEX8 << 6, 44 Msps) on channels 0 and 2, OFDM (x 20, 40 Msps) on channel 1,
    staggered starts -> ({channel: rows int16 [n, 2]}, [[mpdu, ...] per channel], [[(start, rate, seed), ...] per channel])."""
    rows, mpdus, plan = {}, [], []
    for ci, kind in enumerate(R.KIND_24):
        t, fr, ms, pl = 300 + 500 * ci, [], [], []
        for j, (rate, nb) in enumerate(FRAMES_24[ci]):
            m = _mpdu(nb, 0x3E240000 + 16 * ci + j); seed = 3 + 5 * j
            f = oracle_py.tx11b_modulate(m, rate).astype(np.int16) << 6 if kind == "11b" else oracle_py.tx11a_modulate(m, rate, seed).astype(np.int16) * 20
            fr.append((t, f)); ms.append(m); pl.append((t, rate, seed)); t += len(f) + 900
        rows[ci] = rows_of([fr])[0]; mpdus.append(ms); plan.append(pl)
    return rows, mpdus, plan

def capture_of(fs, rows):
    """Two calls into one buffer: the 802.11b rows, then the OFDM row added onto them -> (int16 [n_out, 2], the first call's output)."""
    (ub, db), tb, (ua, da), ta = TX_PLANS[fs]
    n_out = max(-(-ub * len(rows[0]) // db), -(-ub * len(rows[2]) // db), -(-ua * len(rows[1]) // da)) + 400
    n_out += (-n_out) % 4
    n_b = max(len(rows[0]), len(rows[2])); rb = np.zeros((2, n_b, 2), np.int16); rb[0, :len(rows[0])] = rows[0]; rb[1, :len(rows[2])] = rows[2]
    chb = [(W.phase_inc(R.CH_24[c], fs), 0, GAIN_B) for c in (0, 2)]
    first = CR.combine_rational(rb, chb, ub, db, tb, n_out)
    y = CR.combine_rational(rows[1][None], [(0, 0, GAIN_A)], ua, da, ta, n_out, acc=first)
    return y, first

# The radio between the combiner and the channelizers: sb200_channel_sim as one link with one tap of 16384 (Q14 unity), no clock or carrier
# offset, and Gaussian noise of sigma = 20 LSB per real component (noise_q8 = 20 x 256), the level of rational_model.capture_24ghz.
SIM_LINK_24 = (0, 2 ** 32, 0, 0, 20 * 256)
SIM_TAPS_24 = np.array([16384, 0], np.int16).reshape(1, 1, 1, 2)
SIM_SEED_24 = 0x24C0

def through_the_air(y):
    """The capture y through the channel simulator's model (SIM_LINK_24): the same samples plus the seeded noise."""
    return SM.sim(y[None, None], [SIM_LINK_24], SIM_TAPS_24, len(y), SIM_SEED_24)[0, 0]

def test_tx_tap_plans_fit_the_limits():
    for (ub, db), tb, (ua, da), ta in TX_PLANS.values():
        for u, d, t in ((ub, db, tb), (ua, da, ta)):
            assert np.gcd(u, d) == 1 and 1 <= d <= 16 and d <= u <= 64
            assert len(t) % 2 == 1 and len(t) <= 4095 and -(-len(t) // u) <= 255
            assert max(int(np.abs(t[r::u].astype(np.int64)).sum()) for r in range(u)) <= 65535
    assert -(-len(TAPS_44_160) // 40) == 45 and max(int(np.abs(TAPS_44_160[r::40].astype(np.int64)).sum()) for r in range(40)) == 59150
    assert -(-len(TAPS_40_176) // 22) == 61 and max(int(np.abs(TAPS_40_176[r::22].astype(np.int64)).sum()) for r in range(22)) == 64398

@pytest.mark.parametrize("fs", [160e6, 176e6])
def test_mixed_24ghz_transmit(fs):
    """802.11b on channels 1 and 11 and OFDM on channel 6 sent into one capture, through the channel simulator's noise: every channel
    returns exactly its own PSDUs (802.11b without the last FCS byte), every one with a good FCS, and nothing of its neighbours; the capture
    does not clip."""
    rows, mpdus, _ = frames_24ghz()
    clean, _ = capture_of(fs, rows)
    assert np.abs(clean.astype(np.int64)).max() < 32767
    y = through_the_air(clean)
    assert 18 < np.std((y.astype(np.int64) - clean)) < 22                               # the noise is there, at sigma = 20
    (ub, db), tb, (ua, da), ta = PLANS[fs]
    back = {c: R.channelize_rational(y, [(W.phase_inc(f, fs), 0)], *((ub, db, tb) if kind == "11b" else (ua, da, ta)))[0]
            for c, (f, kind) in enumerate(zip(R.CH_24, R.KIND_24))}
    for c, (r, o, got) in decode_24ghz(back).items():
        own = [p[:-1] if R.KIND_24[c] == "11b" else p for p in _psdus(mpdus[c])]
        assert got == own, (fs, c, len(got), len(own))
        assert (r["status"] == oracle_py.E_FRAME_OK).all(), (fs, c, r["status"])
