"""The 802.11a brick modulator on the device (k_tx11a behind sb200_tx11a_batch) against the reference's own compiled graphs
(oracle/build_ref_mod.sh: CreatePreamble11a_40M and CreateModGraph11a_40M driven as Test11A_FB_Mod drives them), directly rather than
through the oracle: every rate, the lengths and seeds of test_cpu_tx_reference.py, COMPLEX8 and COMPLEX16 output, a non-zero lead, and a
batch of 3000 mixed-length frames.  pytest -m gpu; skipped without the compiled library."""
import numpy as np, pytest
import oracle_py
from sora_b200 import api
from test_cpu_tx_reference import LENGTHS, RATES_11A, SEEDS, _std_nsym

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not oracle_py.ref_mod_available(), reason="oracle/_ref/libmod_ref.so not built (oracle/build_ref_mod.sh)")]

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

def _check(eng, pay, rate, seeds, lead=0, sample_bits=8):
    out, ns = eng.tx11a_batch(pay, rate, seeds=seeds, lead=lead, sample_bits=sample_bits)
    for i, p in enumerate(pay):
        want = oracle_py.ref_mod11a_frame(p, rate, int(seeds[i]))
        if sample_bits == 16: want = want.astype(np.int16) << 8
        assert ns[i] == lead + len(want), (rate, len(p), ns[i], lead + len(want))
        assert (out[i, :lead] == 0).all()
        bad = np.nonzero((out[i, lead:lead + len(want)] != want).any(1))[0]
        assert len(bad) == 0, (rate, len(p), int(seeds[i]), bad[:8])
        assert (out[i, lead + len(want):] == 0).all()

@pytest.mark.parametrize("rate", RATES_11A)
def test_device_equals_the_compiled_graph(eng, rate):
    rng = np.random.default_rng(rate + 7)
    edge = [n for n in range(2, 4092) if _std_nsym(n, rate) != _std_nsym(n - 1, rate)]
    lens = list(LENGTHS) + [m for n in edge[:3] + edge[-2:] for m in (n - 1, n)]
    pay = [rng.integers(0, 256, n).astype(np.uint8) for n in lens]
    seeds = np.array([SEEDS[i % len(SEEDS)] for i in range(len(lens))], np.uint8)
    _check(eng, pay, rate, seeds, lead=0, sample_bits=8)

@pytest.mark.parametrize("rate", (6000, 9000, 54000))
def test_device_complex16_and_lead_equal_the_compiled_graph(eng, rate):
    rng = np.random.default_rng(rate + 8)
    lens = [1, 5, 64, 333, 1500, 4091]
    pay = [rng.integers(0, 256, n).astype(np.uint8) for n in lens]
    seeds = rng.integers(1, 256, len(lens)).astype(np.uint8)
    _check(eng, pay, rate, seeds, lead=37, sample_bits=16)
    _check(eng, pay, rate, seeds, lead=400, sample_bits=8)

def test_device_equals_the_compiled_graph_on_a_mixed_batch(eng):
    """3000 frames of random lengths 1-1600 and random seeds in one call, at 54 and at 9 Mbps."""
    rng = np.random.default_rng(12)
    for rate in (54000, 9000):
        lens = rng.integers(1, 1601, 3000)
        pay = [rng.integers(0, 256, int(n)).astype(np.uint8) for n in lens]
        _check(eng, pay, rate, rng.integers(0, 256, len(lens)).astype(np.uint8))
