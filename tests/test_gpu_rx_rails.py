"""GPU parity at the int16 rails (pytest -m gpu): clipped, DC-offset and full-scale captures (rail_inputs.py) through every receive chain,
CUDA through the C ABI against the CPU oracle on the same IQ.  Every result field and the delivered bytes must agree; frames need only
decode where the oracle decodes them (most of these inputs do not, as in the reference)."""
import numpy as np, pytest
import oracle_py, rail_inputs as R
from sora_b200 import api

pytestmark = pytest.mark.gpu

F11A = ("status", "rate_kbps", "length", "crc32", "nsym", "detect_index", "cfo_est")
F11B = ("status", "rate_kbps", "length", "crc32", "sample_index", "detect_vec")
F11N = ("status", "mcs", "length", "crc32", "nsym", "detect_index", "cfo_est", "lsig_length")
BODY = (oracle_py.E_FRAME_OK, oracle_py.E_CRC32_FAIL)


@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)


def _check(names, fields, res, out, ores, oout, body_short=0):
    """Field by field, slot by slot; fields other than status only where the oracle saw an event; the bytes of OK / CRC-fail frames
    (802.11b: the sink stops one byte short of the FCS end, body_short = 1)."""
    for i, n in enumerate(names):
        ev = ores["status"][i] != oracle_py.E_NO_FRAME
        for k in fields:
            if k == "status" or ev:
                assert res[k][i] == ores[k][i], (n, k, res[i], ores[i])
        if ores["status"][i] in BODY:
            L = int(ores["length"][i]) - body_short
            assert (out[i, :L] == oout[i, :L]).all(), (n, "bytes")


def _unzip(cases):
    return [n for n, _ in cases], [c for _, c in cases]


@pytest.mark.parametrize("rate", [6000, 24000, 54000])
def test_rx11a_rails(eng, rate):
    names, caps = _unzip(R.cases_11a(rate))
    flat, off, ln = R.slots(caps)
    res, out = eng.rx11a_batch(flat, off, ln)                                       # 40 Msps
    ores, oout = oracle_py.rx11a_batch(flat, off, ln, out_stride=out.shape[1])
    _check(names, F11A, res, out, ores, oout)
    assert (ores["status"] == 1).sum() >= 1                                          # gain 2 still decodes
    h, hoff, hln = R.slots([c[::2] for c in caps])                                  # 20 Msps: the even samples; the oracle gets each one twice and
    res, out = eng.rx11a_batch(h, hoff, hln, sample_rate_mhz=20)                    # TDownSample2 keeps one of the two
    ores, oout = oracle_py.rx11a_batch(np.repeat(h, 2, axis=0), 2 * hoff, 2 * hln, out_stride=out.shape[1])
    _check(names, F11A, res, out, ores, oout)
    assert (ores["status"] == 1).sum() >= 1
    res, out = eng.rx11a_batch(flat, off, ln, sample_rate_mhz=44)                   # 44 Msps: the 11:10 resampler at full scale
    for i, (n, c) in enumerate(zip(names, caps)):
        o, ob = oracle_py.rx11a_run(oracle_py.resample_44_40(c), max_frames=1, out_stride=out.shape[1])
        if len(o) == 0:
            assert res["status"][i] == oracle_py.E_NO_FRAME, (n, res[i]); continue
        _check([n], F11A, res[i:i + 1], out[i:i + 1], o, ob)
    # stage taps on the slots that detect (40 Msps): FFT, channel, equaliser, pilot tracking, soft values
    M = 80
    t = eng.rx11a_taps(flat, off, ln, max_sym=M)
    used = [b for b in range(64) if (1 <= b <= 26) or (38 <= b <= 63)]
    ndet = 0
    for i, (n, c) in enumerate(zip(names, caps)):
        o = oracle_py.rx11a_taps(c, max_sym=M)
        if o["res"]["status"] == oracle_py.E_NO_FRAME: continue
        ndet += 1; ns = o["nsym"]
        assert t["res"]["status"][i] == o["res"]["status"], n
        assert (t["freq_coeffs"][i] == o["freq_coeffs"]).all() and (t["chan_coeffs"][i] == o["chan_coeffs"]).all(), n
        assert (t["fft_out"][i, :ns] == o["fft_out"]).all() and (t["equalized"][i, :ns] == o["equalized"]).all(), n
        assert (t["tracked"][i, :ns][:, used] == o["tracked"][:, used]).all(), n
        nsoft = max(len(o["soft"]) - 48, 0)                                         # the oracle's soft values start with the SIGNAL's 48
        assert (t["soft"][i, :nsoft] == o["soft"][48:48 + nsoft]).all(), n
    assert ndet >= 6


@pytest.mark.parametrize("rate", [1000, 2000, 5500, 11000])
def test_rx11b_rails(eng, rate):
    names, caps = _unzip(R.cases_11b(rate))
    flat, off, ln = R.slots(caps)
    res, out = eng.rx11b_batch(flat, off, ln)
    ores, oout = oracle_py.rx11b_batch(flat, off, ln, out_stride=out.shape[1])
    _check(names, F11B, res, out, ores, oout, body_short=1)
    assert ores["status"][names.index("gain2")] == 1 and ores["status"][names.index("tail")] == oracle_py.E_CRC32_FAIL   # the data path ran at full scale


def _streams_11b(eng, caps):
    flat, off, ln = R.slots(caps)
    res, out, cnt = eng.rx11b_streams(flat, off, ln, max_frames=64, out_stride=2048)
    nev = 0
    for s, c in enumerate(caps):
        o, ob = oracle_py.rx11b_run(c, max_frames=64, out_stride=2048)
        assert len(o) < 64
        assert cnt[s] == len(o), (s, cnt[s], res[s, :cnt[s]], o)
        _check([f"stream {s} event {k}" for k in range(len(o))], F11B, res[s, :len(o)], out[s, :len(o)], o, ob, body_short=1)
        nev += len(o)
    return nev


def test_rx11b_streams_across_clipped_bursts(eng):
    """Continuous captures in which the DC estimate, the energy window and the descrambler carry across clipped bursts, DC steps and
    full-scale stretches."""
    caps = []
    for rate in (1000, 2000, 5500, 11000):
        cs = dict(R.cases_11b(rate)); f = cs["gain2"]
        caps.append(np.concatenate([cs["burst"], f, R.scaled(f, 1.0, (20000, -20000)), f, R.pattern("tone", 2800), f, cs["tail"], f]))
        caps.append(np.concatenate([R.pattern("min", 5600), f, R.pattern("rails", 2800), R.scaled(f, 1.0, (-7000, 13000)), f]))
    assert _streams_11b(eng, caps) >= 3 * len(caps)


def _with_mcs_limit(eng, limit):
    eng.set_option("ht_mcs_limit", limit); oracle_py.set_ht_mcs_limit(limit)

@pytest.fixture
def mcs_limit(eng):
    yield lambda limit: _with_mcs_limit(eng, limit)
    _with_mcs_limit(eng, 11)


@pytest.mark.parametrize("mcs,limit", [(8, 11), (10, 11), (14, 15)])
def test_rx11n_rails(eng, mcs_limit, mcs, limit):
    """Batch parity and the stage taps (SISO channel, H^-1, equaliser, pilot phase, soft values).  Includes two rank-deficient channels,
    ((1, 1), (1, 1)) and ((1, 0), (0, 0)): det H = 0 sends the inverse through NaN / out-of-range conversions.  MCS 14 (64-QAM) with
    the HT-SIG gate opened reaches the QAM demap clamp."""
    mcs_limit(limit)
    cs = R.cases_11n(mcs)
    names = [n for n, _ in cs]; a = [c[0] for _, c in cs]; b = [c[1] for _, c in cs]
    f0, off, ln = R.slots(a); f1, _, _ = R.slots(b)
    res, out = eng.rx11n_batch(f0, f1, off, ln)
    ores, oout = oracle_py.rx11n_batch(f0, f1, off, ln, out_stride=out.shape[1])
    _check(names, F11N, res, out, ores, oout)
    assert (ores["status"] == 1).sum() >= 2 and (ores["status"][[names.index("rank1"), names.index("single")]] == oracle_py.E_CRC32_FAIL).all()
    o = [oracle_py.rx11n_taps(x, y) for x, y in zip(a, b)]
    M = max(1, max(t["ndata"] for t in o))
    g = eng.rx11n_taps(f0, f1, off, ln, max_sym=M)
    for i, (n, t) in enumerate(zip(names, o)):
        st = t["res"]["status"]
        assert g["res"]["status"][i] == st, n
        if st == oracle_py.E_NO_FRAME: continue
        assert (g["siso"][i] == t["siso"]).all() and (g["sig"][i] == t["sig"]).all(), n
        if st == oracle_py.E_PLCP_FAIL: continue
        nd = t["ndata"]
        assert (g["hinv"][i] == t["hinv"]).all(), (n, "hinv")
        assert (g["theta"][i, :nd] == t["theta"]).all() and (g["eq"][i][:, :nd] == t["eq"]).all(), (n, "eq")
        ns = len(t["soft"]); assert (g["soft"][i, :ns] == t["soft"]).all(), (n, "soft")


@pytest.mark.parametrize("mcs,limit", [(8, 11), (10, 11), (14, 15)])
def test_rx11n_streams_across_clipped_bursts(eng, mcs_limit, mcs, limit):
    """Continuous two-antenna captures: TCCA11n / MimoAutoCorr history carried across clipped bursts, full-scale stretches and DC steps."""
    mcs_limit(limit)
    cs = dict(R.cases_11n(mcs, chans=False)); f = cs["gain2"]
    pat = lambda k, n: (R.pattern(k, n, 1), R.pattern(k, n, 2))
    parts = [[cs["burst"], f, pat("min", 2800), f, cs["tail"], f], [pat("nyquist", 2800), cs["dc+20000-20000"], f, pat("rails", 1400), cs["gain0.125"], f]]
    caps = [(np.concatenate([p[0] for p in ps]), np.concatenate([p[1] for p in ps])) for ps in parts]
    f0, off, ln = R.slots([c[0] for c in caps]); f1, _, _ = R.slots([c[1] for c in caps])
    res, out, sidx, cnt = eng.rx11n_streams(f0, f1, off, ln, max_frames=8)
    nok = 0
    for s, (c0, c1) in enumerate(caps):
        o, ob = oracle_py.rx11n_run(c0, c1, max_frames=8, out_stride=1536)
        assert cnt[s] == len(o), (s, cnt[s], res[s, :cnt[s]], o)
        vec_base = 0; prev = 0
        for k in range(len(o)):
            for fld in ("status", "mcs", "length", "nsym", "cfo_est", "lsig_length"):
                assert res[s, k][fld] == o[k][fld], (s, k, fld, res[s, k], o[k])
            assert sidx[s, k] == o[k]["sample_index"], (s, k)
            assert vec_base + res[s, k]["detect_index"] == o[k]["detect_index"], (s, k)    # the oracle counts 20 Msps vectors since the capture began
            vec_base += 4 * ((int(sidx[s, k]) - prev) // 8); prev = int(sidx[s, k])
            if o[k]["status"] in BODY:
                L = int(o[k]["length"]); assert res[s, k]["crc32"] == o[k]["crc32"] and (out[s, k, :L] == ob[k, :L]).all(), (s, k)
            nok += int(o[k]["status"] == 1)
    assert nok >= 3
