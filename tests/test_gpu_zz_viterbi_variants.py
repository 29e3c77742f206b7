"""GPU parity of every Viterbi kernel the library carries, on batches that mix rates and lengths inside one warp (pytest -m gpu).
Kept in its own file, sorted after the per-chain suites: it forces each kernel with the options viterbi_lane_min / viterbi_lane_max."""
import numpy as np, pytest
import oracle_py
from sora_b200 import api, synth

pytestmark = pytest.mark.gpu

def test_viterbi_variants_on_mixed_batches():
    """Every Viterbi kernel the library carries, forced whatever the batch size: the four-lanes-per-code-block kernel (viterbi_lane_min
    0xFFFFFFFF) and the one-lane-per-code-block kernel (viterbi_k7_lane.cuh; viterbi_lane_min 0, viterbi_lane_max 0xFFFFFFFF) in its
    renderings.  One call holds frames of every rate and of many lengths, so that the code blocks sharing a warp reach their traceback
    triggers and their ends at different times; a damaged frame and an empty slot sit among them.  All must equal the CPU oracle, and the
    standalone decoder is run on wrap-around garbage at both windows."""
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
    # the lane kernel with 6- / 8-column history blocks, 9 = 8 with the deferred walk
    for v, hb in (("k_viterbi_re", 0), ("k_viterbi_lane", 6), ("k_viterbi_lane", 8), ("k_viterbi_lane", 9)):
        e = api.Engine(0)
        if v == "k_viterbi_lane": e.set_option("viterbi_lane_min", 0); e.set_option("viterbi_lane_max", 0xFFFFFFFF)
        else: e.set_option("viterbi_lane_min", 0xFFFFFFFF)
        if hb: e.set_option("vl_hist_block", min(hb, 8)); e.set_option("vl_defer_walk", 1 if hb == 9 else 0)
        res, out = e.rx11a_batch(flat.reshape(-1, 2), off, ln)
        assert e.last_viterbi_kernel() == v
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
