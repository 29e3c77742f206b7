"""The 802.11a front end between the carrier sense and the Viterbi against the reference's OWN bricks, compiled from its headers where
they lie (oracle/build_ref_rx11a.sh -> oracle/_ref/librx11a_ref.so): T11aLTS, TFreqCompensation, TFFT64, TChannelEqualization,
TPhaseCompensate, TPilotTrack, T11aDemap<1,2,4,6>, the four de-interleavers and TDownSample44_40.  The oracle (oracle/rx11a.cpp) restates
them; here every intermediate it taps must equal the compiled bricks byte for byte when they are handed the same blocks: the 144
samples on_lts is handed (lts_in) and the 80-sample blocks on_symbol is handed (sym_in), both tapped from the oracle on each capture.

Compared: CFO_est, FreqCoeffs, ChannelCoeffs, and per symbol fft_in, fft_out, the equalised and the tracked symbol and the de-interleaved
soft values.  Not compared, because the reference leaves them undefined: the tracked symbol's bin 0 and bins 27-37.  TPilotTrack's
_build_coeff (pilot.hpp:143-166) never writes the rotation coefficients of bins 0, 27 .. 37, and _rotate (pilot.hpp:137-140) skips vectors
7 and 8 (bins 28-35), which keep whatever the output queue held.  The oracle zeroes those bins.  The demapper reads none of them.

Inputs, each placed in a valid 40 Msps frame (the 20 Msps block samples each repeated twice) so that the oracle's framing hands it over:
  - LTS blocks: random full-scale, random at every power-of-two amplitude (|Y|^2 >> 8 of 0, 1 and 2, the wrapping pack of the channel
    inverse, and the ranges where uatan2's bit_scope shift changes), the adversarial symbol families on both LTS copies (bins at
    +-32768), and the frame's own LTS rotated through every int16 CFO;
  - data symbols: the adversarial families of test_gpu_fft_reference, random symbols at every amplitude (equalised values past the
    demap clamp and rotations whose pack wraps), all eight rates (SIGNAL included), frames of more than 127 data symbols (PilotSgn and the
    CFO_comp / SFO_comp accumulators wrap);
  - whole captures: synth frames at all 8 rates and channel_inputs' multipath / SCO cases.
The 44 -> 40 resampler: random and full-scale streams whose lengths are not multiples of 28 or 11, sample for sample.
The debug tap's counters show which edges the corpus reaches; test_counters_reached asserts each one is."""
import numpy as np, pytest
import oracle_py as O, channel_inputs as CI
from sora_b200 import synth
import test_gpu_fft_reference as G

pytestmark = pytest.mark.skipif(not O.ref_rx11a_available(), reason="oracle/_ref/librx11a_ref.so not built (needs the reference tree)")
RATES = (6000, 9000, 12000, 18000, 24000, 36000, 48000, 54000)
DEFINED = np.ones(64, bool); DEFINED[0] = False; DEFINED[27:38] = False        # bins the reference defines in the tracked symbol
COUNTS = {}


def _frame(rate, psdu_len=300, seed=0):
    iq, _ = synth.make_frames(1, psdu_len=psdu_len, rate_kbps=rate, snr_db=30, lead=400, trail=228, seed0=0xF11A0000 + rate + seed)
    return iq[0][: len(iq[0]) // 28 * 28]


def _blocks_at(frame):
    """20 Msps index of the LTS block the oracle takes from this frame (its symbols follow every 80 samples)."""
    t = O.rx11a_taps(frame); h = frame[::2]
    j = [k for k in range(len(h) - 144) if (h[k:k + 144] == t["lts_in"]).all()]
    assert len(j) == 1, j
    return j[0]


def _place(frame, j, lts=None, syms=(), first=1):
    """frame with the 20 Msps LTS block at j replaced by lts [144, 2] and the symbol blocks from index `first` by syms [.., 80, 2]."""
    out = frame.copy()
    if lts is not None: out[2 * j:2 * (j + 144)] = np.repeat(lts, 2, axis=0)
    for k, s in enumerate(syms):
        a = 2 * (j + 144 + 80 * (first + k))
        if a + 160 > len(out): break
        out[a:a + 160] = np.repeat(s, 2, axis=0)
    return out


def _sym80(s64):
    return np.concatenate([s64[-16:], s64]).astype(np.int16)


def check(cap, name):
    """The oracle's taps on cap equal the compiled bricks on the oracle's own lts_in / sym_in.  Returns the number of symbols compared."""
    o = O.rx11a_taps(cap, max_sym=600)
    if o["res"]["status"] == O.E_NO_FRAME and o["nsym"] == 0 and not o["lts_in"].any(): return 0
    ncbps = int(o["soft_off"][2] - o["soft_off"][1]) if o["nsym"] > 1 else 48     # res is only filled on an event: the modulation from
    rate = {48: 6000, 96: 12000, 192: 24000, 288: 54000}[ncbps]                    # the soft values per DATA symbol
    cfo, fc, cc = O.ref_rx11a_lts(o["lts_in"])
    if o["res"]["status"] != O.E_NO_FRAME: assert cfo == o["res"]["cfo_est"], (name, cfo, o["res"]["cfo_est"])   # res is only filled on an event
    assert (fc == o["freq_coeffs"]).all() and (cc == o["chan_coeffs"]).all(), (name, "lts", np.argwhere(cc != o["chan_coeffs"])[:4])
    ns = o["nsym"]
    if ns == 0: return 0
    r = O.ref_rx11a_symbols(o["lts_in"], o["sym_in"], rate)
    for k, v in O.ref_rx11a_debug().items(): COUNTS[k] = COUNTS.get(k, 0) + v
    assert r["cfo_est"] == cfo and (r["chan_coeffs"] == cc).all(), name
    for k in ("fft_in", "fft_out", "equalized"):
        bad = np.argwhere((r[k] != o[k]).any(-1))
        assert not len(bad), (name, k, bad[:4])
    bad = np.argwhere((r["tracked"][:, DEFINED] != o["tracked"][:, DEFINED]).any(-1))
    assert not len(bad), (name, "tracked", bad[:4])
    for i in range(ns):
        got = o["soft"][o["soft_off"][i]:o["soft_off"][i + 1]]
        assert (got == r["soft"][i]).all(), (name, "soft", i, np.argwhere(got != r["soft"][i])[:4])
    return ns


@pytest.fixture(scope="module")
def base():
    f = _frame(6000, psdu_len=800)
    return f, _blocks_at(f)


def test_lts_random_and_scaled(base):
    f, j = base; rng = np.random.default_rng(11)
    for k in range(16):
        for seed in range(6):
            lts = rng.integers(-32768, 32768, (144, 2)) >> (15 - k) if k < 15 else rng.integers(-32768, 32768, (144, 2))
            check(_place(f, j, lts=lts.astype(np.int16)), ("scale", k, seed))
    for s in G.adversarial_symbols(5):
        check(_place(f, j, lts=np.concatenate([s[-16:], s, s]).astype(np.int16)), "family")


def test_lts_every_cfo(base):
    f, j = base
    lts = f[2 * j:2 * (j + 144):2].astype(np.float64); z = lts[:, 0] + 1j * lts[:, 1]; n = np.arange(144)
    for c in range(-32768, 32768):
        y = z * np.exp(1j * np.pi * c / 32768 * n) * 0.9
        b = np.clip(np.round(np.stack([y.real, y.imag], 1)), -32768, 32767).astype(np.int16)
        check(_place(f, j, lts=b), ("cfo", c))


@pytest.mark.parametrize("rate", RATES)
def test_symbol_families(base, rate):
    f = _frame(rate, psdu_len=400); j = _blocks_at(f)
    syms = [_sym80(s) for s in G.adversarial_symbols(rate)]
    rng = np.random.default_rng(rate)
    for k in range(16):
        syms.append(_sym80((rng.integers(-32768, 32768, (64, 2)) >> (15 - k)).astype(np.int16)))
    for r in range(0, len(syms), 7):                      # every family in front in one capture, the rest behind it
        assert check(_place(f, j, syms=np.roll(np.array(syms), -r, axis=0)), (rate, r)) >= 2


def test_long_frames_wrap_pilot_polarity(base):
    f, j = base
    n = check(f, "long")
    assert n > 127 + 40, n                                 # symbol_count passes 126 -> 0 and PilotSgn wraps
    rng = np.random.default_rng(3)
    noisy = np.clip(f + rng.integers(-3000, 3000, f.shape), -32768, 32767).astype(np.int16)
    check(noisy, "long noisy")


@pytest.mark.parametrize("rate", RATES)
def test_whole_captures(rate):
    assert check(_frame(rate), rate) >= 2
    for name, c in (CI.cases_11a(rate)[:4] if rate in CI.RATES_11A else ()):
        check(c, (rate, name))


def test_resample_44_40():
    rng = np.random.default_rng(44)
    for n in (1, 27, 28, 29, 11 * 28 + 5, 28 * 113 + 17, 50011):
        for x in (rng.integers(-32768, 32768, (n, 2)), np.full((n, 2), -32768), np.full((n, 2), 32767),
                  np.where(rng.random((n, 2)) < 0.5, -32768, 32767)):
            x = x.astype(np.int16)
            a, b = O.ref_resample_44_40(x), O.resample_44_40(x)
            assert a.shape == b.shape and (a == b).all(), n


def test_counters_reached(base):
    """What the corpus above reached in the reference's bricks (see ref_rx11a_debug); run alone, it runs the LTS and 54 Mbps corpus first."""
    if not COUNTS:
        test_lts_random_and_scaled(base); test_symbol_families(base, 54000)
    print("front11a reference counters:", COUNTS)
    for k in ("lts_e0", "lts_pack", "demap_clamp", "mul_pack", "eq_pack"):
        assert COUNTS[k] > 0, (k, COUNTS)


# ---- carrier sense: TDownSample2 -> TDCRemoveEx<4> -> TCCA11a -> TDCEstimator -------------------------------------------------------------
def check_cs(cap, name):
    """The oracle's carrier-sense trace equals the compiled bricks', vector for vector, up to the detection.  cca_peak_index is compared
    once TCCA11a has first set it (with cca_pwr_reading, cca.hpp:335-341): CF_11CCA's constructor leaves it unset (ieee80211facade.hpp:33-36)."""
    a, da = O.rx11a_cs_trace(cap); b, db = O.ref_rx11a_carrier_sense(cap)
    assert a.shape == b.shape and da == db, (name, a.shape, b.shape, da, db)
    set_ = np.cumsum(a[:, 11] != 0) > 0
    keep = np.ones(13, bool); keep[10] = False
    bad = np.argwhere((a[:, keep] != b[:, keep]).any(1))
    assert not len(bad), (name, bad[:4], a[bad[0, 0]], b[bad[0, 0]])
    assert (a[set_, 10] == b[set_, 10]).all(), (name, "peak_index")
    return a, da


def _sts_capture(shift, dc=(0, 0), gain=1.0, lead=2000):
    f = _frame(6000, psdu_len=60, seed=shift)
    x = np.concatenate([np.zeros((lead + 2 * shift, 2)), f.astype(np.float64) * gain]) + np.array(dc)
    return np.clip(np.round(x), -32768, 32767).astype(np.int16)[: (lead + 2 * shift + len(f)) // 28 * 28]


def test_carrier_sense_sts_every_peak_index():
    peaks = set()
    for shift in range(32):                                 # the STS period is 16 samples at 20 Msps: every alignment, twice
        a, d = check_cs(_sts_capture(shift), ("shift", shift))
        assert d >= 0, shift
        peaks.add(int(a[-1, 10]))
    assert peaks == {0, 1, 2, 3}, peaks


def test_carrier_sense_noise_threshold_and_timeouts():
    rng = np.random.default_rng(7)
    nt = 0
    for amp in (200, 700, 1000, 1100, 1200, 1300, 1500, 2000, 4000):   # energy of x >> 2 summed over 16 samples >> 4 around 10^6
        x = rng.normal(0, amp, (30000, 2))
        tone = np.exp(1j * 2 * np.pi * np.arange(30000) / 32) * amp       # a periodic signal: the autocorrelation test passes as well
        for y in (x, x + np.stack([tone.real, tone.imag], 1)):
            a, _ = check_cs(np.clip(np.round(y), -32768, 32767).astype(np.int16), ("noise", amp))
            nt += int((a[:, 1] == np.int32(np.uint32(0x80000007).view(np.int32))).sum())
    assert nt > 0                                                        # timeouts fired and the carrier sense re-armed
    # a constant (4000, 0): x >> 2 = 1000, each lane's |.|^2 >> 4 = 62 500, four lanes and four vectors: an energy of exactly
    # cca_pwr_threshold = 10^6 (fb11ademod_config.hpp:107) until the DC estimate first moves; the energy test is strict (cca.hpp:316)
    for v in ((4000, 0), (0, -4000), (4004, 0), (3996, 0)):
        check_cs(np.tile(np.array(v, np.int16), (6000, 1)), ("at threshold", v))


def test_carrier_sense_dc_on_the_rails():
    for dc in ((32767, 32767), (-32768, -32768), (32767, -32768), (-20000, 12000)):
        check_cs(_sts_capture(3, dc=dc, gain=0.3), ("dc", dc))
        check_cs(np.tile(np.array(dc, np.int16), (20000, 1)), ("dc only", dc))
    for gain in (0.01, 0.05, 4.0):                                          # below the threshold, and clipped at the rails
        check_cs(_sts_capture(5, gain=gain), ("gain", gain))


def test_carrier_sense_whole_captures():
    for rate in RATES:
        check_cs(_frame(rate), rate)
        for name, c in (CI.cases_11a(rate)[:4] if rate in CI.RATES_11A else ()):
            check_cs(c, (rate, name))
