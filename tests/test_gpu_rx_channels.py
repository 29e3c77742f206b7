"""GPU parity through frequency-selective channels and a sampling-clock offset (pytest -m gpu): the captures of channel_inputs.py
(exponential delay profiles, echoes beyond the guard interval, pre-echoes, spectral nulls on data / pilot / near-DC bins, per-tap 2x2
channels, SCO up to +-100 ppm) through every receive chain, CUDA through the C ABI against the CPU oracle on the same IQ.

Every result field where the oracle saw an event and the delivered bytes must agree, and where a chain has stage taps, every stage of
every slot that detects: 802.11a frequency-offset and channel-inverse coefficients, FFT, equaliser, pilot tracking and soft values at
6 / 12 / 24 / 54 Mbps (so the BPSK, QPSK, 16-QAM and 64-QAM demap all sit under the taps); 802.11n SISO channel, per-bin 2x2 inverse,
equaliser, pilot phase, HT-SIG and soft values."""
import numpy as np, pytest
import oracle_py, channel_inputs as CI, rail_inputs as R
from sora_b200 import api
from test_gpu_rx_rails import _check, _streams_11b, F11A, F11B, F11N, BODY

pytestmark = pytest.mark.gpu

OUT = 4096                                             # row of delivered bytes: the longest 802.11a PSDU here is 2500 B
LANE_MIN_DEFAULT = 16384                               # the library's own choice: the lane Viterbi kernel from 16 384 code blocks on
USED = [b for b in range(64) if (1 <= b <= 26) or (38 <= b <= 63)]
# FRAME_OK per rate the oracle reaches on the 40 / 20 / 44 Msps renderings (of 17 cases each); the test asserts no fewer
MIN_OK_11A = {6000: 13, 12000: 11, 24000: 11, 54000: 7}


@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)


def _unzip(cases):
    return [n for n, _ in cases], [c for _, c in cases]


def _first_diff(name, stages):
    """The first stage (in pipeline order) whose device and oracle arrays differ, with the first differing index and both values."""
    for stage, dev, ora in stages:
        dev = np.asarray(dev); ora = np.asarray(ora)
        if dev.shape != ora.shape:
            return f"{name}: {stage} shape {dev.shape} != {ora.shape}"
        bad = np.argwhere(dev != ora)
        if len(bad):
            i = tuple(bad[0])
            return f"{name}: {stage} first differs at {i}: device {dev[i]} oracle {ora[i]} ({len(bad)} values differ)"
    return None


@pytest.mark.parametrize("rate", CI.RATES_11A)
def test_rx11a_channels_batch(eng, rate):
    """40, 20 and 44 Msps, and the 40 Msps batch once more through the lane Viterbi kernel."""
    names, caps = _unzip(CI.cases_11a(rate))
    flat, off, ln = R.slots(caps)
    res, out = eng.rx11a_batch(flat, off, ln, out_stride=OUT)
    ores, oout = oracle_py.rx11a_batch(flat, off, ln, out_stride=OUT)
    _check(names, F11A, res, out, ores, oout)
    assert (ores["status"] == oracle_py.E_FRAME_OK).sum() >= MIN_OK_11A[rate] and (ores["status"] != oracle_py.E_FRAME_OK).any()
    try:
        eng.set_option("viterbi_lane_min", 0)
        res2, out2 = eng.rx11a_batch(flat, off, ln, out_stride=OUT)
        assert eng.last_viterbi_kernel() == "k_viterbi_lane"
    finally:
        eng.set_option("viterbi_lane_min", LANE_MIN_DEFAULT)
    assert (res2 == res).all() and (out2 == out).all()
    h, hoff, hln = R.slots([c[::2] for c in caps])                                  # 20 Msps: the even samples; the oracle gets each one twice and
    res, out = eng.rx11a_batch(h, hoff, hln, out_stride=OUT, sample_rate_mhz=20)    # TDownSample2 keeps one of the two
    ores, oout = oracle_py.rx11a_batch(np.repeat(h, 2, axis=0), 2 * hoff, 2 * hln, out_stride=OUT)
    _check(names, F11A, res, out, ores, oout)
    assert (ores["status"] == oracle_py.E_FRAME_OK).sum() >= MIN_OK_11A[rate]
    names44, caps44 = _unzip(CI.cases_11a(rate, 44))                               # 44 Msps: the same channels rendered at 44 Msps
    f44, off44, ln44 = R.slots(caps44)
    res, out = eng.rx11a_batch(f44, off44, ln44, out_stride=OUT, sample_rate_mhz=44)
    nok = 0
    for i, (n, c) in enumerate(zip(names44, caps44)):
        o, ob = oracle_py.rx11a_run(oracle_py.resample_44_40(c), max_frames=1, out_stride=OUT)
        if len(o) == 0:
            assert res["status"][i] == oracle_py.E_NO_FRAME, (n, res[i]); continue
        _check([n], F11A, res[i:i + 1], out[i:i + 1], o, ob)
        nok += int(o["status"][0] == oracle_py.E_FRAME_OK)
    assert nok >= MIN_OK_11A[rate]


@pytest.mark.parametrize("rate", CI.RATES_11A)
def test_rx11a_channels_taps(eng, rate):
    names, caps = _unzip(CI.cases_11a(rate))
    flat, off, ln = R.slots(caps)
    o = [oracle_py.rx11a_taps(c, max_sym=900) for c in caps]
    M = max(t["nsym"] for t in o) + 1
    t = eng.rx11a_taps(flat, off, ln, max_sym=M)
    bad = []; ndet = 0
    for i, (n, ot) in enumerate(zip(names, o)):
        if ot["res"]["status"] == oracle_py.E_NO_FRAME:
            assert t["res"]["status"][i] == oracle_py.E_NO_FRAME, n; continue
        ndet += 1; ns = ot["nsym"]; nsoft = max(len(ot["soft"]) - 48, 0)            # the oracle's soft values start with the SIGNAL's 48
        d = _first_diff(n, [("status", t["res"]["status"][i], ot["res"]["status"]),
                            ("freq_coeffs", t["freq_coeffs"][i], ot["freq_coeffs"]), ("chan_coeffs", t["chan_coeffs"][i], ot["chan_coeffs"]),
                            ("fft_out", t["fft_out"][i, :ns], ot["fft_out"]), ("equalized", t["equalized"][i, :ns], ot["equalized"]),
                            ("tracked", t["tracked"][i, :ns][:, USED], ot["tracked"][:, USED]),
                            ("soft", t["soft"][i, :nsoft], ot["soft"][48:48 + nsoft])])
        if d: bad.append(d)
    assert not bad, bad
    assert ndet == len(caps)


def _with_mcs_limit(eng, limit):
    eng.set_option("ht_mcs_limit", limit); oracle_py.set_ht_mcs_limit(limit)

@pytest.fixture
def mcs_limit(eng):
    yield lambda limit: _with_mcs_limit(eng, limit)
    _with_mcs_limit(eng, 11)


@pytest.mark.parametrize("mcs,limit", CI.MCS_11N)
def test_rx11n_channels(eng, mcs_limit, mcs, limit):
    """Batch parity and the stage taps on per-tap 2x2 channels, near-singular bins, a faded antenna and SCO."""
    mcs_limit(limit)
    cs = CI.cases_11n(mcs)
    names = [n for n, _ in cs]; a = [c[0] for _, c in cs]; b = [c[1] for _, c in cs]
    f0, off, ln = R.slots(a); f1, _, _ = R.slots(b)
    res, out = eng.rx11n_batch(f0, f1, off, ln)
    ores, oout = oracle_py.rx11n_batch(f0, f1, off, ln, out_stride=out.shape[1])
    _check(names, F11N, res, out, ores, oout)
    assert (ores["status"] == oracle_py.E_FRAME_OK).sum() >= 3
    o = [oracle_py.rx11n_taps(x, y) for x, y in zip(a, b)]
    M = max(1, max(t["ndata"] for t in o))
    g = eng.rx11n_taps(f0, f1, off, ln, max_sym=M)
    bad = []
    for i, (n, t) in enumerate(zip(names, o)):
        st = t["res"]["status"]
        assert g["res"]["status"][i] == st, n
        if st == oracle_py.E_NO_FRAME: continue
        stages = [("siso", g["siso"][i], t["siso"]), ("sig", g["sig"][i], t["sig"])]
        if st != oracle_py.E_PLCP_FAIL:
            nd = t["ndata"]
            stages += [("hinv", g["hinv"][i], t["hinv"]), ("theta", g["theta"][i, :nd], t["theta"]), ("eq", g["eq"][i][:, :nd], t["eq"]),
                       ("soft", g["soft"][i, :len(t["soft"])], t["soft"])]
        d = _first_diff(n, stages)
        if d: bad.append(d)
    assert not bad, bad


@pytest.mark.parametrize("rate", CI.RATES_11B)
def test_rx11b_channels(eng, rate):
    names, caps = _unzip(CI.cases_11b(rate))
    flat, off, ln = R.slots(caps)
    res, out = eng.rx11b_batch(flat, off, ln, out_stride=OUT)
    ores, oout = oracle_py.rx11b_batch(flat, off, ln, out_stride=OUT)
    _check(names, F11B, res, out, ores, oout, body_short=1)
    assert (ores["status"] == oracle_py.E_FRAME_OK).sum() >= 2 and (ores["status"] != oracle_py.E_FRAME_OK).any()


def test_rx11a_stream_through_channels(eng):
    """One continuous capture of frames at four rates through different channels: the streams entry point against the oracle's RxThread."""
    iq = CI.stream_11a()
    ores, oout = oracle_py.rx11a_run(iq, max_frames=16, out_stride=OUT)
    res, out, sidx, cnt = eng.rx11a_streams(iq, [0], [len(iq)], max_frames=16, out_stride=OUT)
    assert len(ores) < 16 and cnt[0] == len(ores), (cnt[0], ores, res[0, :cnt[0]])
    r = res[0, :cnt[0]]
    for k in ("status", "rate_kbps", "length", "crc32", "nsym", "cfo_est"):
        assert (r[k] == ores[k]).all(), (k, r[k], ores[k])
    assert (sidx[0, :cnt[0]] == ores["sample_index"]).all()
    # the oracle counts 20 Msps vectors since the start of the capture, the library since the restart after each event
    seg = np.diff(np.concatenate([[0], ores["sample_index"].astype(np.int64)]))
    assert (r["detect_index"] + np.concatenate([[0], np.cumsum(4 * (seg // 8))[:-1]]) == ores["detect_index"]).all()
    for i in range(len(ores)):
        if ores["status"][i] in BODY:
            L = int(ores["length"][i]); assert (out[0, i, :L] == oout[i, :L]).all(), i
    assert (ores["status"] == oracle_py.E_FRAME_OK).sum() >= 4


def test_rx11b_stream_through_channels(eng):
    assert _streams_11b(eng, [CI.stream_11b()]) >= 8


@pytest.mark.parametrize("mcs,limit", CI.MCS_11N)
def test_rx11n_stream_through_channels(eng, mcs_limit, mcs, limit):
    mcs_limit(limit)
    c0, c1 = CI.stream_11n(mcs)
    res, out, sidx, cnt = eng.rx11n_streams(c0, c1, [0], [len(c0)], max_frames=16)
    o, ob = oracle_py.rx11n_run(c0, c1, max_frames=16, out_stride=out.shape[2])
    assert len(o) < 16 and cnt[0] == len(o), (cnt[0], res[0, :cnt[0]], o)
    vec_base = 0; prev = 0
    for k in range(len(o)):
        for fld in ("status", "mcs", "length", "nsym", "cfo_est", "lsig_length"):
            assert res[0, k][fld] == o[k][fld], (k, fld, res[0, k], o[k])
        assert sidx[0, k] == o[k]["sample_index"], k
        assert vec_base + res[0, k]["detect_index"] == o[k]["detect_index"], k      # the oracle counts 20 Msps vectors since the capture began
        vec_base += 4 * ((int(sidx[0, k]) - prev) // 8); prev = int(sidx[0, k])
        if o[k]["status"] in BODY:
            L = int(o[k]["length"]); assert res[0, k]["crc32"] == o[k]["crc32"] and (out[0, k, :L] == ob[k, :L]).all(), k
    assert (o["status"] == oracle_py.E_FRAME_OK).sum() >= 2
