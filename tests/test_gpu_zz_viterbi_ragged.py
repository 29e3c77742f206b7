"""GPU parity of every Viterbi kernel (forced with the options viterbi_lane_min / viterbi_lane_max) where code blocks of one launch end at
different places in the trellis, and over the standalone decoder's whole envelope (pytest -m gpu).  Sorted after the per-chain suites, as
test_gpu_zz_viterbi_variants.py is.

  * 802.11n receive with mixed lengths in one call.  A frame's soft values are whole symbols of N_CBPS bytes; at MCS 8, 9, 11 (rate 1/2) and 13
    (rate 2/3) a symbol is not a whole number of 6-step chunks, so a frame can run out of whole chunks before its flush point while a
    neighbour in the warp still has chunks to step.  The lengths put the flush point at every offset of the last partial chunk, short and
    long frames alternate, and every frame must decode as the oracle decodes it.
  * sb200_viterbi_k7: every window the header accepts, short and empty frames, flush points next to a trigger, soft rows with extra groups,
    a trailing partial group or too few groups, wrap-inducing words, 1 to 37 blocks; staging from and to host and device memory; the
    selection of the kernel by batch size; config #5 (L = 2 500 at rate 3/4) at the batch sizes that select the lane and the four-lane kernel;
    and the arguments it refuses."""
import numpy as np, pytest
import oracle_py
from sora_b200 import api, synth
from test_gpu_rx11n import _capture_11n

pytestmark = pytest.mark.gpu

# (kernel, vl_hist_block, vl_defer_walk): four lanes per code block, one lane (6- or 8-column history blocks, walk at the trigger or spread
# over the step loop)
KERNELS = (("k_viterbi_re", 0, 0), ("k_viterbi_lane", 6, 0), ("k_viterbi_lane", 8, 0), ("k_viterbi_lane", 8, 1))

class _engine:
    """An engine that runs kernel v at every batch size, with the lane kernel's rendering options."""
    def __init__(self, v, hb=0, defer=0, mcs_limit=None):
        self.v, self.hb, self.defer, self.mcs_limit = v, hb, defer, mcs_limit
    def __enter__(self):
        self.e = api.Engine(0)
        if self.v == "k_viterbi_lane": self.e.set_option("viterbi_lane_min", 0); self.e.set_option("viterbi_lane_max", 0xFFFFFFFF)
        else: self.e.set_option("viterbi_lane_min", 0xFFFFFFFF)
        if self.hb: self.e.set_option("vl_hist_block", self.hb); self.e.set_option("vl_defer_walk", self.defer)
        if self.mcs_limit: self.e.set_option("ht_mcs_limit", self.mcs_limit)
        return self.e
    def __exit__(self, *a):
        self.e.close()

# ---- 802.11n receive: frames that run out of whole chunks before their flush point, beside longer ones ----
NDBPS = {8: 52, 9: 104, 10: 156, 11: 208, 12: 312, 13: 416, 14: 468}      # trellis steps per symbol, two streams
GSTEPS = {8: 1, 9: 1, 10: 3, 11: 1, 12: 3, 13: 2, 14: 3}                   # trellis steps per puncture group

def _lengths(mcs, n=44):
    """n PSDU lengths, short and long alternating.  The short ones put the flush point 8 L + 22 past the frame's last whole 6-step chunk, at
    every offset there a group boundary allows (rate 3/4 has no such frame: its symbols are whole chunks; plain short lengths then)."""
    nd = NDBPS[mcs]; by_off = {}
    for L in range(20, 400):
        S = -(-(8 * L + 22) // nd) * nd; whole = S // 6 * 6
        if 8 * L + 22 > whole: by_off.setdefault(8 * L + 22 - whole, []).append(L)
    short = [L for off in sorted(by_off) for L in by_off[off][:8]] or list(range(20, 400, 37))
    return [short[(i // 2) % len(short)] if i % 2 == 0 else 420 + 13 * (i % 7) for i in range(n)]

def _frames_11n(mcs, seed):
    lens = _lengths(mcs); parts0, parts1 = [], []
    for i, L in enumerate(lens):
        a, b, _ = synth.make_frames_11n(1, psdu_len=L, mcs=mcs, seed0=seed + i, snr_db=None if i % 3 or mcs >= 12 else 32, lead=200 + 8 * (i % 5), trail=120)
        parts0.append(a[0]); parts1.append(b[0])
    slot = max(len(p) for p in parts0)
    iq0 = np.zeros((len(lens), slot, 2), np.int16); iq1 = np.zeros_like(iq0)
    for i in range(len(lens)): iq0[i, :len(parts0[i])] = parts0[i]; iq1[i, :len(parts1[i])] = parts1[i]
    return iq0.reshape(-1, 2), iq1.reshape(-1, 2), np.arange(len(lens), dtype=np.uint64) * slot, np.full(len(lens), slot, np.uint32), lens

@pytest.fixture(scope="module")
def frames11n():
    """Frames and oracle answers of every MCS: batch form, and the same frames as continuous captures of four frames each."""
    out = {}
    for mcs in sorted(NDBPS):
        oracle_py.set_ht_mcs_limit(15 if mcs >= 11 else 11)
        try:
            iq0, iq1, off, ln, lens = _frames_11n(mcs, 0x11F00 + 100 * mcs)
            ores, oout = oracle_py.rx11n_batch(iq0, iq1, off, ln, out_stride=1536)
            assert (ores["status"] == 1).all() and (ores["length"] == lens).all(), (mcs, ores["status"])
            caps = [_capture_11n(mcs * 100 + c, [(mcs, L, None if mcs >= 12 else 32, 180 + 7 * k, 150, None) for k, L in enumerate(lens[4 * c:4 * c + 4])]) for c in range(len(lens) // 4)]
            orun = [oracle_py.rx11n_run(a, b, max_frames=8, out_stride=1536) for a, b in caps]
            out[mcs] = (iq0, iq1, off, ln, ores, oout, caps, orun)
        finally:
            oracle_py.set_ht_mcs_limit(11)
    return out

@pytest.mark.parametrize("v, hb, defer", KERNELS)
def test_rx11n_mixed_lengths_every_kernel(frames11n, v, hb, defer):
    """rx11n_batch and rx11n_streams with 44 frames per call whose flush points fall anywhere in their last partial chunk, short and long
    frames interleaved: every frame FRAME_OK with the oracle's fields and bytes, at MCS 8..10 and, under ht_mcs_limit 15, MCS 11..14."""
    for mcs, (iq0, iq1, off, ln, ores, oout, caps, orun) in frames11n.items():
        with _engine(v, hb, defer, 15 if mcs >= 11 else None) as e:
            res, out = e.rx11n_batch(iq0, iq1, off, ln)
            assert e.last_viterbi_kernel() == v
            bad = [(i, int(ores["length"][i]), hex(int(res["status"][i]))) for i in range(len(res)) if res["status"][i] != ores["status"][i]]
            assert not bad, (v, hb, defer, mcs, "frames (slot, length, status) differ from the oracle's FRAME_OK:", bad)
            for k in ("mcs", "length", "crc32", "nsym", "detect_index", "cfo_est", "lsig_length"):
                assert (res[k] == ores[k]).all(), (v, mcs, k)
            for i in range(len(res)):
                L = int(ores["length"][i]); assert (out[i, :L] == oout[i, :L]).all(), (v, mcs, i)
            # the same frames as continuous captures: the second phase decodes every event of every capture in one batch
            off_s = np.cumsum([0] + [(len(c[0]) + 3) // 4 * 4 for c in caps[:-1]]).astype(np.uint64)
            total = int(off_s[-1]) + len(caps[-1][0]); a = np.zeros((total, 2), np.int16); b = np.zeros((total, 2), np.int16)
            for o, c in zip(off_s, caps): a[int(o):int(o) + len(c[0])] = c[0]; b[int(o):int(o) + len(c[1])] = c[1]
            rs, os_, _, cnt = e.rx11n_streams(a, b, off_s, [len(c[0]) for c in caps], max_frames=8)
            for s, (ro, oo) in enumerate(orun):
                assert cnt[s] == len(ro) == 4, (v, mcs, s, cnt[s], len(ro))
                for k in range(len(ro)):
                    assert ro[k]["status"] == 1 and rs[s, k]["status"] == 1, (v, mcs, s, k, hex(int(rs[s, k]["status"])), int(ro[k]["length"]))
                    L = int(ro[k]["length"])
                    assert rs[s, k]["crc32"] == ro[k]["crc32"] and (os_[s, k, :L] == oo[k, :L]).all(), (v, mcs, s, k)

# ---- the standalone decoder ----
PER = {api.CR_12: (2, 1), api.CR_23: (3, 2), api.CR_34: (4, 3)}             # soft bytes and trellis steps per puncture group

def _words(rng, nblocks, ns, cr, L):
    """nblocks soft rows of ns bytes: clean and noisy code words, all 7, all 0, alternating extremes, uniform noise, in turn."""
    per, gst = PER[cr]
    nbits = -(-ns // per) * gst
    bits = rng.integers(0, 2, (nblocks, nbits)).astype(np.uint8); bits[:, 8 * L + 16:] = 0
    A, B = synth.conv_encode(bits)
    coded = synth.puncture(A, B, {api.CR_12: (1, 2), api.CR_23: (2, 3), api.CR_34: (3, 4)}[cr])[:, :ns]
    soft = np.where(coded > 0, rng.integers(5, 8, coded.shape), rng.integers(0, 3, coded.shape))
    for i in range(nblocks):
        k = i % 6
        if k == 1: soft[i] = np.where(rng.random(ns) < 0.08, rng.integers(0, 8, ns), soft[i])
        elif k == 2: soft[i] = 7
        elif k == 3: soft[i] = 0
        elif k == 4: soft[i] = np.tile([0, 7, 7, 0, 7], ns)[:ns]
        elif k == 5: soft[i] = rng.integers(0, 8, ns)
    return soft.astype(np.uint8)

def _triggers(depth, look, gst, upto):
    t, ob, out = 0, 0, []
    while t < upto:
        t += gst
        if t >= ob + depth + look + 6: out.append(t); ob += depth
    return out

def _cases():
    """(code rate, L, depth, lookahead, soft [nblocks, nsoft]): the envelope of sb200_viterbi_k7."""
    rng = np.random.default_rng(0xE7)
    cases = []
    for cr, (per, gst) in PER.items():
        full = lambda L, extra=0: (-(-(8 * L + 22) // gst) + extra) * per
        for depth in (8, 16, 64, 136, 192, 256):                              # every window shape at L = 61, 9 blocks
            for look in sorted({0, 1, 7, 8, 24, 36, 280 - depth}):
                if depth + look <= 280: cases.append((cr, 61, depth, look, _words(rng, 9, full(61, 2), cr, 61)))
        for depth, look in ((256, 24), (192, 36)):
            Ls = [0, 1, 2, 61]
            for T in _triggers(depth, look, gst, 1200)[:3]:                   # flush points next to the first triggers: before, on, after
                Ls += [L for L in range(max(0, (T - 40) // 8), (T + 24) // 8) if abs(8 * L + 22 - T) <= gst + 6]
            for L in sorted(set(Ls)):
                cases.append((cr, L, depth, look, _words(rng, 37, full(L, 1), cr, L)))
        for nb in (1, 7, 9, 33, 37):                                          # soft rows: extra groups, a trailing partial group, too short
            L = 90
            for ns in (full(L, 5), full(L, 2) + per - 1, full(L) - 7 * per, full(L) // 2 // per * per + 1):
                cases.append((cr, L, 192, 36, _words(rng, nb, ns, cr, L)))
    return cases

@pytest.fixture(scope="module")
def envelope():
    return [(cr, L, d, la, s, oracle_py.viterbi_blocks_n(s, cr, L, d, la, nthreads=8)) for cr, L, d, la, s in _cases()]

@pytest.mark.parametrize("v, hb, defer", KERNELS)
def test_standalone_envelope_every_kernel(envelope, v, hb, defer):
    """Every case of the envelope equals the oracle bit for bit; a block whose soft values end before the flush point is compared on the
    bytes the oracle produced."""
    with _engine(v, hb, defer) as e:
        for cr, L, depth, look, soft, (o, n) in envelope:
            g = e.viterbi_k7(soft, cr, L, depth, look)
            for i in range(len(soft)):
                assert (g[i, :n[i]] == o[i, :n[i]]).all(), (v, hb, defer, cr, L, depth, look, soft.shape, i, int(n[i]), np.argwhere(g[i, :n[i]] != o[i, :n[i]])[:4])

def test_standalone_staging_paths():
    """Soft values in device memory (aligned, unaligned, odd stride) and in host memory; results in device and host memory; out_stride = L + 2
    and wider.  Before each case the handle's workspaces hold the rows of a call on 0xFF soft values, and the caller's stride padding holds
    nonzero bytes that must survive."""
    import torch
    rng = np.random.default_rng(0x57A)
    e = api.Engine(0)
    try:
        for cr, (per, gst) in PER.items():
            L = 77; ns = (-(-(8 * L + 22) // gst) + 3) * per; nb = 37
            soft = _words(rng, nb, ns, cr, L)
            o = oracle_py.viterbi_blocks(soft, cr, L, 192, 36)
            for s_where, s_extra, s_shift in (("dev", 0, 0), ("dev", 16 - ns % 16, 0), ("dev", 16 - ns % 16, 1), ("dev", 1, 0), ("host", 0, 0), ("host", 5, 3)):
                for o_where, o_extra in (("dev", 0), ("dev", 13), ("host", 0), ("host", 9)):
                    poison = np.full((nb, ns), 7, np.uint8); poison[:, 1::2] = 0xFF
                    e.viterbi_k7(poison, cr, L + 40, 192, 36)                       # the handle's staging rows hold other values now
                    sst = ns + s_extra
                    sbuf = np.full(nb * sst + s_shift + 16, 0xA5, np.uint8)
                    rows = np.lib.stride_tricks.as_strided(sbuf[s_shift:], (nb, ns), (sst, 1)); rows[:] = soft
                    ost = L + 2 + o_extra
                    obuf = np.full(nb * ost + 16, 0x5C, np.uint8)
                    if s_where == "dev": ts = torch.from_numpy(sbuf).cuda(); sp = ts.data_ptr() + s_shift
                    else: sp = sbuf.ctypes.data + s_shift
                    if o_where == "dev": to = torch.from_numpy(obuf).cuda(); op = to.data_ptr()
                    else: op = obuf.ctypes.data
                    e.viterbi_raw(sp, sst, ns, nb, cr, L, op, ost, 192, 36)
                    torch.cuda.synchronize()
                    got = to.cpu().numpy() if o_where == "dev" else obuf
                    grid = got[:nb * ost].reshape(nb, ost)
                    what = (cr, s_where, s_extra, s_shift, o_where, o_extra)
                    assert (grid[:, :L + 2] == o).all(), what
                    assert (grid[:, L + 2:] == 0x5C).all() and (got[nb * ost:] == 0x5C).all(), ("stride padding written",) + what
    finally:
        e.close()

def test_selection_boundaries():
    """With default options, launches of 16 383 / 16 384 / 49 152 / 49 153 code blocks of L = 12 take the four-lane, lane, lane and four-lane
    kernel, and every row equals the oracle."""
    rng = np.random.default_rng(0x5E1)
    e = api.Engine(0)
    try:
        for cr, (per, gst) in PER.items():
            L = 12; ns = (-(-(8 * L + 22) // gst) + 1) * per
            uniq = _words(rng, 96, ns, cr, L)
            o = oracle_py.viterbi_blocks(uniq, cr, L)
            for n, name in ((16383, "k_viterbi_re"), (16384, "k_viterbi_lane"), (49152, "k_viterbi_lane"), (49153, "k_viterbi_re")):
                idx = np.arange(n) * 7 % 96
                g = e.viterbi_k7(uniq[idx], cr, L)
                assert e.last_viterbi_kernel() == name, (n, e.last_viterbi_kernel())
                bad = np.nonzero((g != o[idx]).any(1))[0]
                assert len(bad) == 0, (cr, n, bad[:8])
    finally:
        e.close()

def test_config5_at_scale():
    """BASELINE config #5, L = 2 500 at rate 3/4: 16 384 blocks (the lane kernel) and 49 153 (the four-lane kernel), tiled on the device from
    64 unique words; every row equals its word's oracle answer (slab and ring indexing far into the grid)."""
    import torch
    rng = np.random.default_rng(0xC5)
    L, cr = 2500, api.CR_34; ns = -(-(8 * L + 22) // 3) * 4
    uniq = _words(rng, 64, ns, cr, L)
    o = torch.from_numpy(oracle_py.viterbi_blocks(uniq, cr, L, nthreads=8)).cuda()
    du = torch.from_numpy(uniq).cuda()
    e = api.Engine(0)
    try:
        for n, name in ((16384, "k_viterbi_lane"), (49153, "k_viterbi_re")):
            idx = (torch.arange(n, device="cuda") * 29 + 3) % 64
            ds = du[idx].contiguous(); dout = torch.zeros((n, L + 2), dtype=torch.uint8, device="cuda")
            e.viterbi_raw(ds.data_ptr(), ns, ns, n, cr, L, dout.data_ptr(), L + 2)
            torch.cuda.synchronize()
            assert e.last_viterbi_kernel() == name
            bad = torch.nonzero((dout != o[idx]).any(1)).flatten()
            assert bad.numel() == 0, (n, bad[:8].tolist())
            del ds, dout
    finally:
        e.close()

def test_refused_arguments():
    """code_rate -1 and 3, depth 0 / 12 / 264, depth + lookahead = 281, soft_stride < nsoft, out_stride < L + 2: SB200_E_INVALID, the output is
    untouched, and the handle decodes afterwards."""
    e = api.Engine(0)
    try:
        rng = np.random.default_rng(0xBAD)
        L = 30; ns = (8 * L + 22 + 2) * 2; soft = _words(rng, 5, ns, api.CR_12, L)
        o = oracle_py.viterbi_blocks(soft, api.CR_12, L)
        for cr, depth, look, sst, ost in ((-1, 256, 24, ns, L + 2), (3, 256, 24, ns, L + 2), (0, 0, 24, ns, L + 2), (0, 12, 24, ns, L + 2), (0, 264, 16, ns, L + 2),
                                          (0, 256, 25, ns, L + 2), (0, 200, 81, ns, L + 2), (0, 256, 24, ns - 1, L + 2), (0, 256, 24, ns, L + 1)):
            out = np.full((5, L + 2), 0x3C, np.uint8)
            rc = e._lib.sb200_viterbi_k7(e._h, soft.ctypes.data, sst, ns, 5, cr, L, depth, look, out.ctypes.data, ost, None)
            assert rc == -1, (cr, depth, look, sst, ost, rc)
            assert (out == 0x3C).all(), (cr, depth, look, sst, ost)
            assert (e.viterbi_k7(soft, api.CR_12, L) == o).all()
    finally:
        e.close()
