"""The three sample-staging variants of k_front11a (engine option front_stage) against the direct loads (0), whatever the library's
default is: identical FrameInfo and bytes on every rate, odd symbol counts, truncated slots and slots at every alignment mod 4 words."""
import numpy as np, pytest
from sora_b200 import api, synth

pytestmark = pytest.mark.gpu

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

def _captures():
    caps = []
    for i, rate in enumerate(sorted(synth.RATES)):
        iq, _ = synth.make_frames(2, psdu_len=53 + 101 * i, rate_kbps=rate, snr_db=25, seed0=0x5A00 + rate, lead=41 + 5 * i, trail=44 + i)
        caps += [iq[0], iq[1][: len(iq[1]) - 320 * (i % 3)]]
    off = np.concatenate([[0], np.cumsum([len(c) + 1 for c in caps])[:-1]]).astype(np.uint64)     # + 1: slot starts at every alignment mod 4 words
    flat = np.zeros((int(off[-1]) + len(caps[-1]) + 8, 2), np.int16)
    for o, c in zip(off, caps): flat[int(o): int(o) + len(c)] = c
    return flat, off, np.array([len(c) for c in caps], np.uint32)

def test_staging_variants_equal_direct_loads(eng):
    flat, off, ln = _captures()
    got = {}
    try:
        for stage in (0, 1, 2):
            eng.set_option("front_stage", stage)
            got[stage] = eng.rx11a_batch(flat, off, ln)
    finally:
        eng.set_option("front_stage", 1)
    ref, refo = got[0]
    assert (ref["status"] == 1).sum() >= 8
    for stage in (1, 2):
        res, out = got[stage]
        assert (res == ref).all() and (out == refo).all(), stage
