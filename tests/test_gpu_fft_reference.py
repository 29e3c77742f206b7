"""The device's OFDM transforms against the reference's OWN FFT<64> / IFFT<128> (oracle/_ref/libfft_ref.so, built by build(); see
tests/test_cpu_fft_reference.py), on the GPU (pytest -m gpu):
  - 802.11a: captures with a valid preamble and SIGNAL whose data symbols are adversarial (full-scale noise, DC on the rails, Nyquist,
    impulses, tones, the searched FFT<64> corpus), cyclic-prefixed so any FFT window sees a cyclic shift of them.  At 40 Msps the device's
    fft_out tap equals ref_fft64 of what the oracle handed its fft64, symbol for symbol; at 20, 40 and 44 Msps verdicts and bytes equal the
    oracle, whose own fft_out equals ref_fft64(fft_in).  Most of these frames end in CRC32_FAIL, as expected.
  - 802.11n: the same symbols on both antennas.  The device's 802.11n tap entry point has no FFT tap, so the link is made through the
    oracle: its fft_out equals ref_fft64(fft_in), and the device's equalised symbols, phase track and soft values equal the oracle's.
  - Transmitters: every rate and MCS, payloads long enough that every data bin takes as many distinct values as the constellation has
    points (checked on the logged symbols).  The device's
    tx11a_batch, tx11n_batch and tx11a_legacy_batch (40 and 44 Msps) equal the oracle, and the oracle's ifft128 equals ref_ifft128 on exactly
    the symbols it transformed, so warp_ifft128 is tied to the reference through that one pinned link."""
import numpy as np, pytest
import oracle_py, oracle_tx11a_legacy, rail_inputs as R
import test_cpu_fft_reference as T
from sora_b200 import api, synth

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not oracle_py.ref_fft_available(), reason="oracle/_ref/libfft_ref.so not built")]
F11A = ("status", "rate_kbps", "length", "crc32", "nsym", "detect_index", "cfo_est")
F11N = ("status", "mcs", "length", "crc32", "nsym", "detect_index", "cfo_est", "lsig_length")
BODY = (oracle_py.E_FRAME_OK, oracle_py.E_CRC32_FAIL)


@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)


def adversarial_symbols(seed):
    """64-sample (20 Msps) symbol bodies, int16 [n, 64, 2]."""
    rng = np.random.default_rng(seed); t = np.arange(64)
    s = [rng.integers(-32768, 32768, (64, 2)), np.full((64, 2), -32768), np.full((64, 2), 32767), np.tile([[32767, -32768]], (64, 1)),
         np.where((t % 2 == 0)[:, None], -32768, 32767).repeat(2, 1), np.where(rng.random((64, 2)) < 0.5, -32768, 32767)]
    for p in (0, 17, 63):
        x = np.zeros((64, 2)); x[p] = (-32768, 32767); s.append(x)
    for k in (1, 31, 32):
        z = 32768 * np.exp(2j * np.pi * k * t / 64); s.append(np.clip(np.round(np.stack([z.real, z.imag], 1)), -32768, 32767))
    s.append(T.corpus_vec(T.FFT64_PACK, 64))
    return np.array(s, np.int16)


def with_symbols(frame, start, syms, per_sym):
    """frame with its data symbols from `start` replaced by syms (GI = the last 16 samples), each 20 Msps sample repeated per_sym / 80 times."""
    out = frame.copy(); rep = per_sym // 80
    for k, s in enumerate(syms):
        a = start + k * per_sym
        if a + per_sym > len(out): break
        out[a:a + per_sym] = np.repeat(np.concatenate([s[-16:], s]), rep, axis=0)
    return out


def caps_11a(rate):
    iq, _ = synth.make_frames(1, psdu_len=300, rate_kbps=rate, snr_db=30, lead=400, trail=228, seed0=0xFF7A0000 + rate)
    f = iq[0][: len(iq[0]) // 28 * 28]
    syms = adversarial_symbols(rate)
    caps = []
    for k in range(len(syms)):                      # every family first in one capture, the others after it
        caps.append(("rot%d" % k, with_symbols(f, 1200, np.roll(syms, -k, axis=0), 160)))
    return caps


@pytest.mark.parametrize("rate", [6000, 54000])
def test_rx11a_fft_equals_reference(eng, rate):
    names, caps = zip(*caps_11a(rate))
    flat, off, ln = R.slots(caps)
    M = 80
    t = eng.rx11a_taps(flat, off, ln, max_sym=M)
    nsym = 0
    for i, (n, c) in enumerate(zip(names, caps)):
        o = oracle_py.rx11a_taps(c, max_sym=M)
        assert t["res"]["status"][i] == o["res"]["status"], n
        ns = o["nsym"]; assert ns >= 2, (n, ns)
        ref = oracle_py.ref_fft64(o["fft_in"])
        assert (o["fft_out"] == ref).all(), (n, "oracle")
        assert (t["fft_out"][i, :ns] == ref).all(), (n, "device", np.argwhere(t["fft_out"][i, :ns] != ref)[:4])
        nsym += ns
    assert nsym >= 100
    res, out = eng.rx11a_batch(flat, off, ln)                                        # 40 Msps
    ores, oout = oracle_py.rx11a_batch(flat, off, ln, out_stride=out.shape[1])
    _check(names, res, out, ores, oout)
    h, hoff, hln = R.slots([c[::2] for c in caps])                                  # 20 Msps: the oracle gets each sample twice
    res, out = eng.rx11a_batch(h, hoff, hln, sample_rate_mhz=20)
    rep = np.repeat(h, 2, axis=0)
    ores, oout = oracle_py.rx11a_batch(rep, 2 * hoff, 2 * hln, out_stride=out.shape[1])
    _check(names, res, out, ores, oout)
    for i in range(len(caps)):
        o = oracle_py.rx11a_taps(rep[2 * int(hoff[i]):2 * (int(hoff[i]) + int(hln[i]))], max_sym=M)
        assert (oracle_py.ref_fft64(o["fft_in"]) == o["fft_out"]).all(), names[i]
    res, out = eng.rx11a_batch(flat, off, ln, sample_rate_mhz=44)                   # 44 Msps: the oracle sees the 44 -> 40 resampled capture
    for i, (n, c) in enumerate(zip(names, caps)):
        r40 = oracle_py.resample_44_40(c)
        o, ob = oracle_py.rx11a_run(r40, max_frames=1, out_stride=out.shape[1])
        if len(o) == 0:
            assert res["status"][i] == oracle_py.E_NO_FRAME, n; continue
        _check([n], res[i:i + 1], out[i:i + 1], o, ob)
        tp = oracle_py.rx11a_taps(r40, max_sym=M)
        assert (oracle_py.ref_fft64(tp["fft_in"]) == tp["fft_out"]).all(), n


def _check(names, res, out, ores, oout, fields=F11A):
    for i, n in enumerate(names):
        for k in fields:
            if k == "status" or ores["status"][i] != oracle_py.E_NO_FRAME:
                assert res[k][i] == ores[k][i], (n, k, res[i], ores[i])
        if ores["status"][i] in BODY:
            L = int(ores["length"][i]); assert (out[i, :L] == oout[i, :L]).all(), (n, "bytes")


@pytest.mark.parametrize("mcs", [8, 14])
def test_rx11n_fft_inputs_through_the_chain(eng, mcs):
    eng.set_option("ht_mcs_limit", 15); oracle_py.set_ht_mcs_limit(15)
    try:
        a, b, _ = synth.make_frames_11n(1, psdu_len=300, mcs=mcs, snr_db=30, lead=400, trail=228, seed0=0xFF7B0000 + mcs)
        n = len(a[0]) // 28 * 28; f0, f1 = a[0][:n], b[0][:n]
        start = 400 + 640 + 480 + 160 + 320                                         # lead, legacy preamble, L-SIG + HT-SIG, HT-STF, 2 HT-LTFs
        syms = adversarial_symbols(mcs)
        caps = [("rot%d" % k, (with_symbols(f0, start, np.roll(syms, -k, axis=0), 160), with_symbols(f1, start, np.roll(syms, -k - 1, axis=0), 160)))
                for k in range(len(syms))]
        names = [c for c, _ in caps]
        x0, off, ln = R.slots([c[0] for _, c in caps]); x1, _, _ = R.slots([c[1] for _, c in caps])
        o = [oracle_py.rx11n_taps(p, q) for _, (p, q) in caps]
        M = max(1, max(t["ndata"] for t in o))
        g = eng.rx11n_taps(x0, x1, off, ln, max_sym=M)
        nfft = 0
        for i, (n, t) in enumerate(zip(names, o)):
            assert t["fft_in"].shape[1] >= 4, n
            assert (oracle_py.ref_fft64(t["fft_in"]) == t["fft_out"]).all(), (n, "oracle")
            nfft += t["fft_in"].shape[1]
            st = t["res"]["status"]
            assert g["res"]["status"][i] == st, n
            assert (g["siso"][i] == t["siso"]).all() and (g["sig"][i] == t["sig"]).all(), n
            if st == oracle_py.E_PLCP_FAIL: continue
            nd = t["ndata"]
            assert (g["hinv"][i] == t["hinv"]).all(), (n, "hinv")
            assert (g["theta"][i, :nd] == t["theta"]).all() and (g["eq"][i][:, :nd] == t["eq"]).all(), (n, "eq")
            ns = len(t["soft"]); assert (g["soft"][i, :ns] == t["soft"]).all(), (n, "soft")
        assert nfft >= 100
        res, out = eng.rx11n_batch(x0, x1, off, ln)
        ores, oout = oracle_py.rx11n_batch(x0, x1, off, ln, out_stride=out.shape[1])
        _check(names, res, out, ores, oout, F11N)
    finally:
        eng.set_option("ht_mcs_limit", 11); oracle_py.set_ht_mcs_limit(11)


NPOINTS = {6000: 2, 9000: 2, 12000: 4, 18000: 4, 24000: 16, 36000: 16, 48000: 64, 54000: 64}
NPOINTS_HT = {8: 2, 9: 4, 10: 4, 11: 16, 12: 16, 13: 64, 14: 64}
PILOTS = (7, 21, 128 - 21, 128 - 7)                                                 # subcarriers +-7, +-21 in the zero-stuffed 128


def _covers_every_point(x, npoints):
    """Every used bin other than the pilots takes at least npoints distinct values over the symbols x (the data constellation's points,
    next to the few training and SIGNAL values); returns (ok, the fewest any such bin took)."""
    used = [b for b in np.flatnonzero((x != 0).any(axis=(0, 2))) if b not in PILOTS]
    fewest = min(len(np.unique(x[:, b], axis=0)) for b in used)
    return len(used) >= 48 and fewest >= npoints, fewest


def _payloads(seed, n=8, L=4000):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, L).astype(np.uint8) for _ in range(n)]


@pytest.mark.parametrize("rate", [6000, 9000, 12000, 18000, 24000, 36000, 48000, 54000])
def test_tx11a_symbols(eng, rate):
    pay = _payloads(rate)
    td, ns = eng.tx11a_batch(pay, rate)
    xs = []
    for i, p in enumerate(pay):
        want, x = oracle_py.ifft128_inputs(oracle_py.tx11a_modulate, p, rate, 0xFF, 0)
        assert ns[i] == len(want) and (td[i, :len(want)] == want).all(), i
        xs.append(x)
    x = np.concatenate(xs)
    ok, npts = _covers_every_point(x, NPOINTS[rate]); assert ok, (rate, npts)
    assert (oracle_py.ifft128(x) == oracle_py.ref_ifft128(x)).all()


@pytest.mark.parametrize("sr", [40, 44])
@pytest.mark.parametrize("rate", [6000, 9000, 12000, 18000, 24000, 36000, 48000, 54000])
def test_tx11a_legacy_symbols(eng, rate, sr):
    pay = _payloads(rate + 1, n=8, L=4000)
    out, ns = eng.tx11a_legacy_batch(pay, rate, oracle_tx11a_legacy.preamble(), sample_rate_mhz=sr)
    xs = []
    for i, p in enumerate(pay):
        want = oracle_tx11a_legacy.modulate(p, rate, sr)
        assert ns[i] == len(want) and (out[i, :ns[i]] == want).all(), i
        xs.append(oracle_py.ifft128_inputs(oracle_py.tx11a_legacy_modulate, p, rate)[1])   # the same symbols: 44 Msps resamples after the IFFT
    x = np.concatenate(xs)
    ok, npts = _covers_every_point(x, NPOINTS[rate]); assert ok, (rate, npts)
    assert (oracle_py.ifft128(x) == oracle_py.ref_ifft128(x)).all()


@pytest.mark.parametrize("mcs", range(8, 15))
def test_tx11n_symbols(eng, mcs):
    pay = _payloads(100 + mcs, n=16)                                                 # two streams: half the symbols per stream of one
    t0, t1, ns = eng.tx11n_batch(pay, mcs)
    xs = []
    for i, p in enumerate(pay):
        (w0, w1), x = oracle_py.ifft128_inputs(oracle_py.tx11n_modulate, p, mcs)
        assert ns[i] == len(w0) and (t0[i, :len(w0)] == w0).all() and (t1[i, :len(w1)] == w1).all(), i
        xs.append(x)
    x = np.concatenate(xs)
    ok, npts = _covers_every_point(x, NPOINTS_HT[mcs]); assert ok, (mcs, npts)
    assert (oracle_py.ifft128(x) == oracle_py.ref_ifft128(x)).all()
