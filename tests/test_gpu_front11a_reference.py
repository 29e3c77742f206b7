"""k_front11a against the reference's OWN 802.11a front-end bricks (oracle/_ref/librx11a_ref.so, built by build(); see
tests/test_cpu_front11a_reference.py), on the GPU (pytest -m gpu).  Captures from that file's families (adversarial data symbols and
scaled random symbols at every rate, random and full-scale LTS blocks, channel_inputs' multipath / SCO cases) go through
sb200_rx11a_taps at 40 Msps in one launch.  Per slot the device's freq_coeffs, chan_coeffs, equalized, tracked (the bins the reference
defines) and soft values, and cfo_est in res, must equal the compiled bricks run on the oracle's lts_in / sym_in of the same slot, and
detect_index and peak_index must equal the reference's compiled carrier sense.  At 44 Msps (channel_inputs' captures made at 44 MHz)
the device's verdicts and bytes must equal the oracle run on ref_resample_44_40 of the capture, the reference's own resampler, and at
20 Msps the oracle fed each sample twice; most of those frames decode, so their bytes are compared."""
import numpy as np, pytest
import oracle_py as O, channel_inputs as CI, rail_inputs as R
import test_cpu_front11a_reference as T
import test_gpu_fft_reference as G
from sora_b200 import api

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not O.ref_rx11a_available(), reason="oracle/_ref/librx11a_ref.so not built")]


@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)


def _caps(rate):
    f = T._frame(rate, psdu_len=400); j = T._blocks_at(f)
    syms = [T._sym80(s) for s in G.adversarial_symbols(rate)]
    rng = np.random.default_rng(rate)
    syms += [T._sym80((rng.integers(-32768, 32768, (64, 2)) >> (15 - k)).astype(np.int16)) for k in range(16)]
    caps = [("rot%d" % r, T._place(f, j, syms=np.roll(np.array(syms), -r, axis=0))) for r in range(0, len(syms), 7)]
    caps += [("lts%d" % k, T._place(f, j, lts=(rng.integers(-32768, 32768, (144, 2)) >> (15 - k)).astype(np.int16))) for k in (4, 8, 15)]
    caps += [(n, c) for n, c in (CI.cases_11a(rate)[:3] if rate in CI.RATES_11A else ())]
    return caps


@pytest.mark.parametrize("rate", [6000, 18000, 36000, 54000])
def test_rx11a_front_equals_reference(eng, rate):
    names, caps = zip(*_caps(rate))
    flat, off, ln = R.slots(caps)
    o = [O.rx11a_taps(c, max_sym=600) for c in caps]
    M = max(t["nsym"] for t in o) + 1
    t = eng.rx11a_taps(flat, off, ln, max_sym=M)
    nsym = 0
    for i, (n, ot) in enumerate(zip(names, o)):
        assert t["res"]["status"][i] == ot["res"]["status"], n
        if ot["nsym"] == 0: continue
        T.check(caps[i], n)                                                   # the oracle equals the compiled bricks on this slot
        ns = ot["nsym"]; ncbps = int(ot["soft_off"][2] - ot["soft_off"][1]) if ns > 1 else 48
        r = O.ref_rx11a_symbols(ot["lts_in"], ot["sym_in"], {48: 6000, 96: 12000, 192: 24000, 288: 54000}[ncbps])
        if ot["res"]["status"] != O.E_NO_FRAME:
            assert t["res"]["cfo_est"][i] == r["cfo_est"], n
            cs, det = O.ref_rx11a_carrier_sense(caps[i])                      # the reference's own carrier sense on the slot
            assert t["res"]["detect_index"][i] == 4 * det and t["res"]["peak_index"][i] == cs[-1, 10], (n, "carrier sense")
        assert (t["freq_coeffs"][i] == r["freq_coeffs"]).all() and (t["chan_coeffs"][i] == r["chan_coeffs"]).all(), (n, "lts")
        assert (t["equalized"][i, :ns] == r["equalized"]).all(), (n, "equalized")
        assert (t["tracked"][i, :ns][:, T.DEFINED] == r["tracked"][:, T.DEFINED]).all(), (n, "tracked")
        soft = np.concatenate(r["soft"][1:]) if ns > 1 else np.zeros(0, np.uint8)     # the device's soft values start after SIGNAL
        assert (t["soft"][i, :len(soft)] == soft).all(), (n, "soft", np.argwhere(t["soft"][i, :len(soft)] != soft)[:4])
        nsym += ns
    assert nsym >= 50


@pytest.mark.parametrize("rate", CI.RATES_11A)
def test_rx11a_44_and_20msps(eng, rate):
    """44 Msps captures (channel_inputs at fs = 44 MHz) against the oracle run on the reference resampler's output, and the 40 Msps
    cases taken at 20 Msps against the oracle fed each sample twice: verdicts and bytes."""
    names, caps = zip(*CI.cases_11a(rate, 44))
    flat, off, ln = R.slots(caps)
    res, out = eng.rx11a_batch(flat, off, ln, sample_rate_mhz=44)
    ok = 0
    for i, (n, c) in enumerate(zip(names, caps)):
        o, ob = O.rx11a_run(O.ref_resample_44_40(c), max_frames=1, out_stride=out.shape[1])
        if len(o) == 0:
            assert res["status"][i] == O.E_NO_FRAME, n; continue
        G._check([n], res[i:i + 1], out[i:i + 1], o, ob); ok += int(o["status"][0] == O.E_FRAME_OK)
    assert ok >= len(caps) // 2, (ok, len(caps))
    names, caps = zip(*CI.cases_11a(rate))
    h, hoff, hln = R.slots([c[::2] for c in caps])
    res, out = eng.rx11a_batch(h, hoff, hln, sample_rate_mhz=20)
    rep = np.repeat(h, 2, axis=0)
    ores, oout = O.rx11a_batch(rep, 2 * hoff, 2 * hln, out_stride=out.shape[1])
    G._check(names, res, out, ores, oout)
    assert (ores["status"] == O.E_FRAME_OK).sum() >= len(caps) // 2
