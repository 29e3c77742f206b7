"""GPU parity of every Viterbi kernel the library carries, on batches that mix rates and lengths inside one warp (pytest -m gpu).
Kept in its own file, sorted after the per-chain suites: it creates engines under different SB200_VITERBI settings."""
import os
import numpy as np, pytest
import oracle_py
from sora_b200 import api, synth

pytestmark = pytest.mark.gpu

def test_viterbi_variants_on_mixed_batches():
    """Every Viterbi kernel the library carries (SB200_VITERBI, read when an engine is created): v3 the four-lanes-per-code-block kernel, v4 two
    lanes, v8 the one-lane-per-code-block kernel (viterbi_k7_lane.cuh), v2 the round-1 quad.  One call holds frames of every rate and of many
    lengths, so that the code blocks sharing a warp reach their traceback triggers and their ends at different times; a damaged frame and an
    empty slot sit among them.  All must equal the CPU oracle, and the standalone decoder is run on wrap-around garbage at both windows."""
    rng = np.random.default_rng(0x8)
    parts = []; maxlen = 0
    for i, rate in enumerate(sorted(synth.RATES) * 5):                  # 40 frames: 8 rates x 5 lengths, interleaved -> mixed inside every warp
        L = (14, 61, 333, 700, 1201)[i // 8] + 3 * (i % 8)
        iq, _ = synth.make_frames(1, psdu_len=L, rate_kbps=rate, seed0=0x77000 + i, snr_db=28 if i % 3 else None, lead=40 + 4 * (i % 5), trail=64)
        parts.append(iq[0]); maxlen = max(maxlen, iq.shape[1])
    parts[5] = parts[5].copy(); parts[5][900:1100] = 0                  # a hole in the middle of frame 5: CRC failure
    parts.append(np.zeros((500, 2), np.int16))                          # nothing to find
    flat = np.zeros((len(parts), maxlen, 2), np.int16); ln = np.zeros(len(parts), np.uint32)
    for i, p in enumerate(parts): flat[i, :len(p)] = p; ln[i] = len(p)
    off = np.arange(len(parts), dtype=np.uint64) * maxlen
    ores, oout = oracle_py.rx11a_batch(flat.reshape(-1, 2), off, ln, out_stride=2560)
    assert (ores["status"] == 1).sum() >= 36
    soft = rng.integers(0, 8, (37, 4 * 451)).astype(np.uint8)           # 37 blocks: one full warp of the lane kernel plus five lanes of the next
    old = os.environ.get("SB200_VITERBI")
    try:
        for v, hb in (("v3", 0), ("v8", 6), ("v8", 8), ("v8", 9), ("v4", 0), ("v2", 0)):   # v8: the lane kernel with 6- / 8-column history blocks, 9 = 8 with the deferred walk
            os.environ["SB200_VITERBI"] = v
            e = api.Engine(0)
            if hb: e.set_option("vl_hist_block", min(hb, 8)); e.set_option("vl_defer_walk", 1 if hb == 9 else 0)
            res, out = e.rx11a_batch(flat.reshape(-1, 2), off, ln)
            assert e.last_viterbi_kernel() == ("k_viterbi_lane" if v == "v8" else "k_viterbi_re" if v != "v2" else e.last_viterbi_kernel())
            found = ores["status"] != oracle_py.E_NO_FRAME              # the fields of a slot without a frame are not defined
            assert (res["status"] == ores["status"]).all(), (v, hb, res["status"], ores["status"])
            for k in ("rate_kbps", "length", "crc32", "nsym"):
                assert (res[k][found] == ores[k][found]).all(), (v, hb, k, res[k], ores[k])
            for i in range(len(res)):
                if ores["status"][i] in (1, oracle_py.E_CRC32_FAIL):
                    assert (out[i, :ores["length"][i]] == oout[i, :ores["length"][i]]).all(), (v, hb, i)
            for cr, per in ((api.CR_12, 2), (api.CR_23, 3), (api.CR_34, 4)):
                ns = soft.shape[1] // per * per
                for depth, look, L in ((256, 24, 100), (192, 36, 61)):
                    g = e.viterbi_k7(soft[:, :ns], cr, L, depth, look)
                    assert (g == oracle_py.viterbi_blocks(soft[:, :ns], cr, L, depth, look)).all(), (v, hb, cr, depth)
            e.close()
    finally:
        if old is None: os.environ.pop("SB200_VITERBI", None)
        else: os.environ["SB200_VITERBI"] = old

@pytest.mark.parametrize("name, launches", [("rx11a_batch", 6), ("rx11n_batch", 5), ("rx11n_batch_mcs15", 5), ("viterbi_k7", 1)])
def test_v2_launch_counts(name, launches):
    """sb200_launch_count delta of a warm call under SB200_VITERBI=v2 (the quad kernel, one launch per code rate): the 802.11a receiver
    counts its three quads; the 802.11n receiver counts two, also when ht_mcs_limit 15 makes it launch the CR_23 one as well."""
    from test_gpu_abi_residency import BOOKKEEPING
    old = os.environ.get("SB200_VITERBI")
    os.environ["SB200_VITERBI"] = "v2"
    try:
        e = api.Engine(0)
        call = BOOKKEEPING[name][0](e)
        call(); n0 = e.launches; call()
        assert e.launches - n0 == launches
        e.close()
    finally:
        if old is None: os.environ.pop("SB200_VITERBI", None)
        else: os.environ["SB200_VITERBI"] = old
