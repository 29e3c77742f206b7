"""k_rx11b (sb200_rx11b_batch / sb200_rx11b_streams) against the reference's own compiled 802.11b graph (oracle/_ref/librx11b_ref.so,
built by oracle/build_ref_rx11b.sh): status, rate, length, CRC-32, the event sample and detection vector, and the delivered bytes up to
length - 1 (the sink never delivers the last FCS byte, PHY_11b.hpp:721-739)."""
import numpy as np, pytest
import oracle_py, rail_inputs
from sora_b200 import api, synth
from test_cpu_oracle_11b import _fixture
from test_gpu_rx11b import _capture_11b

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not oracle_py.ref_rx11b_available(), reason="oracle/_ref/librx11b_ref.so not built (oracle/build_ref_rx11b.sh)")]

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

def _same(res, out, rres, rout, ev_rows=None):
    for k in ("status", "rate_kbps", "length", "crc32", "sample_index", "detect_vec"):
        assert (res[k] == rres[k]).all(), (k, np.nonzero(res[k] != rres[k])[0][:8], res[k][:8], rres[k][:8])
    for i in np.nonzero(np.isin(rres["status"], (1, oracle_py.E_CRC32_FAIL)))[0]:
        L = min(int(rres["length"][i]) - 1, out.shape[-1])
        assert (out[i, :L] == rout[i, :L]).all(), f"slot {i}"

def _slots(frames):
    slot = max(len(f) for f in frames); slot += (-slot) % 28
    iq = np.zeros((len(frames), slot, 2), np.int16); ln = np.zeros(len(frames), np.uint32)
    for i, f in enumerate(frames): iq[i, :len(f)] = f; ln[i] = len(f)
    return iq.reshape(-1, 2), np.arange(len(frames), dtype=np.uint64) * slot, ln

def _batch(eng, frames):
    iq, off, ln = _slots(frames)
    res, out = eng.rx11b_batch(iq, off, ln, out_stride=2048)
    rres, rout = oracle_py.ref_rx11b_batch(iq, off, ln, out_stride=2048)
    _same(res, out, rres, rout)
    return res

def test_full_scale_11m_equals_the_reference(eng):
    """The clean 11 Mbps frames at gain 1.0 (peak 32512): the reference's own chain decodes all but frame 2, which fails its FCS, and the
    device must do exactly what it does."""
    iq, _ = synth.make_frames_11b(5, psdu_len=96, rate_kbps=11000, snr_db=None, gain=1.0, seed0=11000 + 7)
    res = _batch(eng, list(iq))
    assert (res["status"] == np.array([1, 1, oracle_py.E_CRC32_FAIL, 1, 1])).all(), res["status"]

def test_cck_rail_chips_equal_the_reference(eng):
    """5.5 and 11 Mbps PSDUs of rectangular chips on the rails (rail_inputs.cck_rail_frames_11b): the CCK decoders' phase decision must
    halve re and im before re + im, as soradsp.h:190-199 does; the unhalved form wraps there and changes the bytes and the CRC."""
    _batch(eng, [x for rate in (5500, 11000) for x in rail_inputs.cck_rail_frames_11b(rate, n=8)])

def test_rates_fixtures_rails_and_edges_equal_the_reference(eng):
    frames = [_fixture("1long44.mf.bin"), _fixture("2long44.mf.bin")]
    for rate in (1000, 2000, 5500, 11000):
        for snr, gain in ((None, 1.0), (40, 0.3), (28, 0.25), (18, 0.2)):
            frames += list(synth.make_frames_11b(5, psdu_len=96, rate_kbps=rate, snr_db=snr, gain=gain, seed0=rate + 7)[0])
        frames += [x for _, x in rail_inputs.cases_11b(rate)]
        frames += list(synth.make_frames_11b(2, psdu_len=120, rate_kbps=rate, snr_db=30, gain=0.3, seed0=rate + 99, cfo_hz=60e3)[0])
    f = synth.make_frames_11b(1, psdu_len=200, rate_kbps=11000, snr_db=40, gain=0.3)[0][0]
    frames += [f[:n] for n in (len(f) // 2, 3001, 3000, 29, 28, 27)]
    rng = np.random.default_rng(4)
    frames += [rng.normal(0, 2500, (28 * 300, 2)).astype(np.int16), np.zeros((5600, 2), np.int16)]
    _batch(eng, frames)

def test_large_batch_equals_the_reference(eng):
    """3 000 slots of mixed rates, gains and noise: more than one wave of 64-thread blocks."""
    rng = np.random.default_rng(21); frames = []
    for k in range(30):
        rate = (1000, 2000, 5500, 11000)[k % 4]
        iq, _ = synth.make_frames_11b(100, psdu_len=int(rng.integers(20, 60)), rate_kbps=rate, snr_db=float(rng.choice([12, 20, 30, 45])),
                                      gain=float(rng.choice([0.2, 0.5, 1.0])), seed0=5000 + k)
        frames += list(iq)
    res = _batch(eng, frames)
    assert len(frames) == 3000 and (res["status"] == 1).sum() > 1000

def test_streams_equal_the_reference(eng):
    caps = [_capture_11b(1, [(11000, 300, False), (2000, 60, False), (5500, 200, True), (11000, 1000, False), (1000, 40, False)], noise=60.0)[0],
            _capture_11b(2, [(5500, 500, False), (11000, 77, False)])[0],
            _capture_11b(3, [(2000, 100, True), (1000, 30, False), (11000, 1496, False)], noise=120.0)[0],
            np.zeros((5000, 2), np.int16)]
    off = np.cumsum([0] + [(len(c) + 3) // 4 * 4 for c in caps[:-1]]).astype(np.uint64)
    iq = np.zeros((int(off[-1]) + len(caps[-1]), 2), np.int16)
    for o, c in zip(off, caps): iq[int(o):int(o) + len(c)] = c
    ln = np.array([len(c) for c in caps], np.uint32)
    res, out, cnt = eng.rx11b_streams(iq, off, ln, max_frames=8, out_stride=2048)
    for s, c in enumerate(caps):
        rres, rout = oracle_py.ref_rx11b_run(c, max_frames=8, out_stride=2048)
        assert cnt[s] == len(rres), (s, cnt[s], rres)
        _same(res[s, :cnt[s]], out[s, :cnt[s]], rres, rout)
