"""Both CUDA Viterbi kernels against the reference's OWN compiled T11aViterbi Filter (oracle/_ref/libviterbi_ref.so, built by
oracle/build_ref_viterbi.sh; tests/test_cpu_viterbi_reference.py holds the CPU side): sb200_viterbi_k7 row for row on the same input
families, rates and windows through k_viterbi_re (the default below 16 384 code blocks) and k_viterbi_lane (forced with viterbi_lane_min 0),
at the launch sizes where the lane kernel is picked by size and where the persistent k_viterbi_re CTAs loop, and one check that ties the
receive chains' Viterbi stage (802.11a and 802.11n, descrambled) to the reference."""
import numpy as np, pytest
import oracle_py
from sora_b200 import api, synth
from test_cpu_viterbi_reference import CR_12, CR_23, CR_34, INSTS, LENGTHS, FLUSH_LENGTHS, families, nsoft_for

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not oracle_py.ref_viterbi_available(), reason="oracle/_ref/libviterbi_ref.so not built")]

class _engine:
    def __enter__(self):
        self.e = api.Engine(0); return self.e
    def __exit__(self, *a):
        self.e.close()

def _decode(e, kernel, soft, cr, L, depth, look):
    e.set_option("viterbi_lane_min", 0 if kernel == "k_viterbi_lane" else 16384)
    g = e.viterbi_k7(soft, cr, L, depth, look)
    assert e.last_viterbi_kernel() == kernel
    e.set_option("viterbi_lane_min", 16384)
    return g

@pytest.mark.parametrize("kernel", ("k_viterbi_re", "k_viterbi_lane"))
@pytest.mark.parametrize("cr", (CR_12, CR_23, CR_34))
def test_kernels_equal_reference(kernel, cr):
    """Every input family at every frame length of the CPU file, all three instantiations' windows: every row == the compiled Filter."""
    rng = np.random.default_rng(300 + cr)
    with _engine() as e:
        for inst in sorted(INSTS):
            _, depth, look = INSTS[inst]
            for L in LENGTHS + FLUSH_LENGTHS:
                ns = nsoft_for(inst, cr, L, extra_groups=int(rng.integers(0, 9)))
                rows, _ = families(rng, cr, L, ns)
                soft = np.stack([r for _, r in rows])
                g = _decode(e, kernel, soft, cr, L, depth, look)
                for i, (name, r) in enumerate(rows):
                    ref = oracle_py.ref_viterbi_block(inst, r, cr, L)
                    assert (g[i] == ref).all(), (kernel, inst, cr, L, name, np.argwhere(g[i] != ref)[:4])

def _distinct_rows(rng, cr, L, ns, n=512):
    """About n distinct rows for one launch: the input families over several seeds, noisy code words at random flip rates, and rows that
    switch family part way, so that neighbouring code blocks in a warp disagree."""
    out = []
    while len(out) < n:
        rows, _ = families(rng, cr, L, ns, nflip=tuple(rng.uniform(0.0, 0.25, 3)))
        out += [r for _, r in rows]
        a, b = rows[int(rng.integers(len(rows)))][1], rows[int(rng.integers(len(rows)))][1]
        cut = int(rng.integers(0, ns)); out.append(np.concatenate([a[:cut], b[cut:]]))
    return np.stack(out[:n])

@pytest.mark.parametrize("nblocks, kernel", ((20000, "k_viterbi_lane"), (65536, "k_viterbi_re")))
def test_large_launches_equal_reference(nblocks, kernel):
    """Default options: 20 000 code blocks select the lane kernel by size; 65 536 (config #2's size) run the persistent k_viterbi_re, whose
    CTAs loop over several groups.  512 distinct rows tiled in a seeded order over the launch, one launch per code rate and frame length,
    each instantiation's window; every output row == the reference row of its distinct input."""
    import torch
    rng = np.random.default_rng(nblocks)
    cases = ((CR_12, 0, 200), (CR_23, 2, 57), (CR_34, 0, 300), (CR_34, 1, 131)) if nblocks == 65536 else \
            ((CR_12, 1, 61), (CR_23, 0, 250), (CR_34, 2, 300), (CR_34, 0, 1000))
    with _engine() as e:
        for cr, inst, L in cases:
            _, depth, look = INSTS[inst]
            ns = nsoft_for(inst, cr, L, extra_groups=int(rng.integers(0, 5)))
            uniq = _distinct_rows(rng, cr, L, ns)
            ref = torch.from_numpy(np.stack([oracle_py.ref_viterbi_block(inst, r, cr, L) for r in uniq])).cuda()
            idx = torch.from_numpy(rng.permutation(np.arange(nblocks) % len(uniq))).cuda()
            ds = torch.from_numpy(uniq).cuda()[idx].contiguous()
            dout = torch.zeros((nblocks, L + 2), dtype=torch.uint8, device="cuda")
            e.viterbi_raw(ds.data_ptr(), ns, ns, nblocks, cr, L, dout.data_ptr(), L + 2, depth, look)
            torch.cuda.synchronize()
            assert e.last_viterbi_kernel() == kernel, (nblocks, e.last_viterbi_kernel())
            bad = torch.nonzero((dout != ref[idx]).any(1)).flatten()
            assert bad.numel() == 0, (nblocks, cr, inst, L, bad.numel(), bad[:8].tolist(), idx[bad[:8]].tolist())
            del ds, dout

def test_rx11a_chain_equals_reference():
    """Noisy 54 and 36 Mbps frames through rx11a_batch (FrameInfo path, descrambled): the de-interleaved soft values of each frame
    (rx11a_taps), decoded by the reference's Filter <5000*8, 48, 256, 24> and descrambled, equal out_bytes up to length, CRC failures too."""
    checked = {api.FRAME_OK: 0, api.FRAME_CRC32_FAIL: 0}
    with _engine() as e:
        for rate, cr, snr in ((54000, CR_34, 17), (54000, CR_34, 21), (36000, CR_34, 12), (36000, CR_34, 15)):
            iq, _ = synth.make_frames(12, psdu_len=400, rate_kbps=rate, snr_db=snr, seed0=rate + snr)
            F, slot, _ = iq.shape
            off = np.arange(F, dtype=np.uint64) * slot; ln = np.full(F, slot, np.uint32)
            res, out = e.rx11a_batch(iq.reshape(-1, 2), off, ln)
            for i in range(F):
                if res["status"][i] not in checked: continue
                t = oracle_py.rx11a_taps(iq[i])
                L = int(res["length"][i]); assert int(t["res"]["length"]) == L
                soft = t["soft"][t["soft_off"][1]:]; assert len(soft) % 48 == 0          # the DATA symbols, after SIGNAL's 48
                dec = oracle_py.ref_viterbi_block(0, soft, cr, L)
                assert len(dec) == L + 2, (rate, snr, i, len(dec))
                assert (oracle_py.descramble(dec)[:L] == out[i, :L]).all(), (rate, snr, i, res["status"][i])
                checked[int(res["status"][i])] += 1
    assert checked[api.FRAME_OK] > 0 and checked[api.FRAME_CRC32_FAIL] > 0, checked

def test_rx11n_chain_equals_reference():
    """802.11n MCS 8 (rate 1/2) and MCS 12 (rate 3/4): the soft values of rx11n_taps, zero-padded to whole 312-value bursts as the
    oracle's brick queue does, decoded by the reference's Filter <5000*8, 312, 192, 36> and descrambled, equal rx11n_batch's bytes."""
    oracle_py.set_ht_mcs_limit(15)                                   # MCS 12 is past the HT-SIG parser as shipped (MCS 8 .. 10)
    try:
        with _engine() as e:
            e.set_option("ht_mcs_limit", 15)
            _rx11n_cases(e)
    finally:
        oracle_py.set_ht_mcs_limit(11)

def _rx11n_cases(e):
    n = 0
    for mcs, cr, snr in ((8, CR_12, 9), (8, CR_12, 30), (12, CR_34, 19), (12, CR_34, 30)):
        iq0, iq1, ps = synth.make_frames_11n(3, psdu_len=300, mcs=mcs, snr_db=snr, lead=400, trail=200)
        F, slot, _ = iq0.shape
        off = np.arange(F, dtype=np.uint64) * slot; ln = np.full(F, slot, np.uint32)
        res, out = e.rx11n_batch(iq0.reshape(-1, 2), iq1.reshape(-1, 2), off, ln)
        for i in range(F):
            if res["status"][i] not in (api.FRAME_OK, api.FRAME_CRC32_FAIL): continue
            t = oracle_py.rx11n_taps(iq0[i], iq1[i])
            L = int(res["length"][i])
            soft = np.zeros(-(-len(t["soft"]) // 312) * 312, np.uint8); soft[:len(t["soft"])] = t["soft"]
            dec = oracle_py.ref_viterbi_block(1, soft, cr, L)
            assert len(dec) == L + 2, (mcs, snr, i, len(dec))
            assert (oracle_py.descramble(dec)[:L] == out[i, :L]).all(), (mcs, snr, i, res["status"][i])
            n += 1
    assert n >= 8, n
