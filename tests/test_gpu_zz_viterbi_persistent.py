"""k_viterbi_re as persistent CTAs on the device, where they loop (pytest -m gpu): receive batches of 65 536 slots in which every code rate's
work list is longer than one round of CTAs, frames differ in rate, length, noise, carrier offset, truncation and verdict, and every
slot must equal the CPU oracle on the unique capture it points to (scale_inputs.py; test_cpu_scale_inputs.py checks that the inputs
do this).  What the host emulation (test_cpu_re_emu_persistent.py) cannot see is exercised here: the group ticket and its broadcast, many
CTAs whose groups end at different times, the shared-memory ring reused under independent thread scheduling, the three code-rate
launches each on its own group counter, and the per-chunk counter blocks of the pipelined paths.

Slot i is compared with oracle row perm[i]: the status everywhere; with an event every other field, peak_index included; the bytes up
to `length` for FRAME_OK and CRC32_FAIL.  Sorted after the per-chain suites; it owns its engines and gives their memory back."""
import os
import numpy as np, pytest
import oracle_py
import scale_inputs as S
from sora_b200 import api
from test_gpu_zz_viterbi_ragged import _words

pytestmark = pytest.mark.gpu
N = 65536
ROW = 2560
FIELDS_11A = ("rate_kbps", "length", "crc32", "nsym", "detect_index", "cfo_est", "peak_index")
FIELDS_11N = ("mcs", "length", "crc32", "nsym", "detect_index", "cfo_est", "lsig_length")
DECODED = (oracle_py.E_FRAME_OK, oracle_py.E_CRC32_FAIL)

class _engine:
    def __enter__(self):
        self.e = api.Engine(0); return self.e
    def __exit__(self, *a):
        import torch
        self.e.close(); torch.cuda.synchronize(); torch.cuda.empty_cache()

@pytest.fixture(scope="module")
def u11a():
    u = S.uniques_11a()
    r, o = oracle_py.rx11a_batch(u.iq, u.off, u.length, out_stride=ROW, nthreads=os.cpu_count())
    return u, r, o

def _check(what, e, u, ores, oout, perm, res, out, fields=FIELDS_11A, rate_key="rate_kbps"):
    """Every slot against its unique's oracle row; the first mismatches (slot, unique, rate, length, kind, what differs) in the message."""
    ost = ores["status"][perm]
    bad = {}
    for i in np.nonzero(res["status"] != ost)[0][:8]: bad.setdefault(int(i), []).append(f"status {int(res['status'][i]):#x} want {int(ost[i]):#x}")
    ev = ost != oracle_py.E_NO_FRAME
    for k in fields:
        for i in np.nonzero(ev & (res[k] != ores[k][perm]))[0][:8]: bad.setdefault(int(i), []).append(f"{k} {res[k][i]} want {ores[k][perm[i]]}")
    dec = np.isin(ost, DECODED); lens = ores["length"][perm].astype(np.int64); col = np.arange(out.shape[1])[None, :]
    for a in range(0, len(perm), 8192):
        b = min(a + 8192, len(perm))
        diff = ((out[a:b] != oout[perm[a:b], :out.shape[1]]) & (col < lens[a:b, None])).any(1) & dec[a:b]
        for i in np.nonzero(diff)[0][:8]: bad.setdefault(a + int(i), []).append("bytes")
    nbad = int((res["status"] != ost).sum())
    msg = [f"slot {i} unique {int(perm[i])} rate {ores[rate_key][perm[i]]} length {int(ores['length'][perm[i]])} kind {u.kind[perm[i]]}: {', '.join(v)}" for i, v in sorted(bad.items())[:12]]
    assert not bad, (what, e.last_viterbi_kernel(), f"{nbad} statuses differ", msg)

def _run_device(e, iq_dev, off, ln):
    """rx11a_batch on device-resident IQ and slot table; results and bytes to the host."""
    import torch
    od = torch.from_numpy(off.astype(np.int64)).cuda(); ld = torch.from_numpy(ln.astype(np.int32)).cuda()
    res = np.zeros(len(off), api.RESULT_DTYPE); out = np.zeros((len(off), ROW), np.uint8)
    e.rx11a_raw(iq_dev.data_ptr(), iq_dev.shape[0], od.data_ptr(), ld.data_ptr(), len(off), out.ctypes.data, ROW, res.ctypes.data)
    torch.cuda.synchronize()
    return res, out

def test_config2_device_resident(u11a):
    """(a) 65 536 device-resident slots with default options: k_viterbi_re decodes; two calls on one handle (the counters of the second
    start from zero again), a second permutation, then the table sorted by decoded length, descending and ascending.  The order of the
    work lists comes from atomics, so no output may depend on it."""
    import torch
    u, ores, oout = u11a
    iq_dev = torch.from_numpy(u.iq).cuda()
    with _engine() as e:
        off, ln, perm = S.tile(u, N, 1)
        for call in range(2):
            res, out = _run_device(e, iq_dev, off, ln)
            assert e.last_viterbi_kernel() == "k_viterbi_re"
            _check(f"device call {call}", e, u, ores, oout, perm, res, out)
        off, ln, perm = S.tile(u, N, 2)
        _check("second permutation", e, u, ores, oout, perm, *_run_device(e, iq_dev, off, ln))
        for order in ("descending", "ascending"):
            key = ores["length"][perm].astype(np.int64) * (-1 if order == "descending" else 1)
            p = perm[np.argsort(key, kind="stable")]
            _check(f"sorted by length, {order}", e, u, ores, oout, p, *_run_device(e, iq_dev, u.off[p], u.length[p]))
    del iq_dev

def test_pipelined_paths(u11a):
    """(b) The chunked paths, each against the oracle: host IQ and table at the default chunk size (16 chunks over three streams, each
    chunk with its own counter block), host_decimate 4 with host_decimate_mix 0, 1 and 2, and device IQ with chunk_frames_device 4 096
    and 3 000 (the last chunk ragged)."""
    import torch
    u, ores, oout = u11a
    off, ln, perm = S.tile(u, N, 3)
    with _engine() as e:
        res, out = e.rx11a_batch(u.iq, off, ln, out_stride=ROW)
        assert e.last_transfer()[1] == 16, e.last_transfer()
        _check("host IQ, 16 chunks", e, u, ores, oout, perm, res, out)
        e.set_option("host_decimate", 4)
        for mix in (0, 1, 2):
            e.set_option("host_decimate_mix", mix)
            res, out = e.rx11a_batch(u.iq, off, ln, out_stride=ROW)
            assert e.last_transfer()[1] == 16, (mix, e.last_transfer())
            _check(f"host_decimate 4, mix {mix}", e, u, ores, oout, perm, res, out)
        e.set_option("host_decimate", 0); e.set_option("host_decimate_mix", 1)
        iq_dev = torch.from_numpy(u.iq).cuda()
        for chunk in (4096, 3000):
            e.set_option("chunk_frames_device", chunk)
            _check(f"device IQ, chunk_frames_device {chunk}", e, u, ores, oout, perm, *_run_device(e, iq_dev, off, ln))
        del iq_dev

def test_streams_four_lane_every_pass():
    """(c) rx11a_streams on 20 480 captures tiled from 256 unique ones of 3 .. 5 frames (mostly rate 3/4), with viterbi_lane_min
    0xFFFFFFFF so the four-lane kernel decodes: counts, fields, sample_index and bytes equal oracle_py.rx11a_run on each unique capture."""
    u = S.uniques_streams()
    off, ln, perm = S.tile(u, 20480, 4)
    orun = []
    for i in range(len(u.off)):
        o = int(u.off[i]); orun.append(oracle_py.rx11a_run(u.iq[o:o + int(u.length[i])], max_frames=8, out_stride=ROW))
    with _engine() as e:
        e.set_option("viterbi_lane_min", 0xFFFFFFFF)
        res, out, sidx, cnt = e.rx11a_streams(u.iq, off, ln, max_frames=8, out_stride=ROW)
        assert e.last_viterbi_kernel() == "k_viterbi_re"
        bad = []
        for s in range(len(perm)):
            ro, oo = orun[perm[s]]; n = len(ro)
            if cnt[s] != n: bad.append((s, int(perm[s]), "count", int(cnt[s]), n)); continue
            r = res[s, :n]
            for k in ("status", "rate_kbps", "length", "crc32", "nsym", "cfo_est"):
                if (r[k] != ro[k]).any(): bad.append((s, int(perm[s]), k, r[k].tolist(), ro[k].tolist()))
            if (sidx[s, :n] != ro["sample_index"]).any(): bad.append((s, int(perm[s]), "sample_index", sidx[s, :n].tolist(), ro["sample_index"].tolist()))
            seg = np.diff(np.concatenate([[0], ro["sample_index"].astype(np.int64)]))      # detect_index: the library counts from each restart
            cum = np.concatenate([[0], np.cumsum(4 * (seg // 8))[:-1]])
            if (r["detect_index"] + cum != ro["detect_index"]).any(): bad.append((s, int(perm[s]), "detect_index"))
            for k in range(n):
                if ro["status"][k] in DECODED:
                    L = int(ro["length"][k])
                    if (out[s, k, :L] != oo[k, :L]).any(): bad.append((s, int(perm[s]), "bytes", k, int(ro["rate_kbps"][k]), L))
            if len(bad) > 12: break
        assert not bad, (e.last_viterbi_kernel(), bad[:12])

def test_rx11n_at_scale():
    """(d) rx11n_batch on 65 536 slots tiled from about 600 2x2 captures at MCS 8 .. 14 with ht_mcs_limit 15, against oracle_py.rx11n_batch."""
    u = S.uniques_11n()
    oracle_py.set_ht_mcs_limit(15)
    try:
        ores, oout = oracle_py.rx11n_batch(u.iq[0], u.iq[1], u.off, u.length, nthreads=os.cpu_count())
    finally:
        oracle_py.set_ht_mcs_limit(11)
    off, ln, perm = S.tile(u, N, 5)
    with _engine() as e:
        e.set_option("ht_mcs_limit", 15)
        res, out = e.rx11n_batch(u.iq[0], u.iq[1], off, ln)
        assert e.last_viterbi_kernel() == "k_viterbi_re"
        _check("rx11n_batch", e, u, ores, oout, perm, res, out, FIELDS_11N, "mcs")

@pytest.mark.parametrize("cr", (api.CR_12, api.CR_23))
def test_standalone_at_scale(cr):
    """(e) sb200_viterbi_k7 on 65 536 blocks at rates 1/2 and 2/3, windows 256/24 and 192/36, tiled on the device from 64 noisy and
    garbage words: every row equals its word's oracle answer (the rate-3/4 counterpart is test_config5_at_scale)."""
    import torch
    per, gst = {api.CR_12: (2, 1), api.CR_23: (3, 2)}[cr]
    L = 700; ns = (-(-(8 * L + 22) // gst) + 1) * per
    uniq = _words(np.random.default_rng(0x5CA + cr), 64, ns, cr, L)
    du = torch.from_numpy(uniq).cuda()
    idx = (torch.arange(N, device="cuda") * 29 + 3) % 64
    idx = idx[torch.randperm(N, generator=torch.Generator().manual_seed(cr)).cuda()]
    ds = du[idx].contiguous(); dout = torch.zeros((N, L + 2), dtype=torch.uint8, device="cuda")
    with _engine() as e:
        for depth, look in ((256, 24), (192, 36)):
            o = torch.from_numpy(oracle_py.viterbi_blocks(uniq, cr, L, depth, look, nthreads=os.cpu_count())).cuda()
            dout.zero_()
            e.viterbi_raw(ds.data_ptr(), ns, ns, N, cr, L, dout.data_ptr(), L + 2, depth, look)
            torch.cuda.synchronize()
            assert e.last_viterbi_kernel() == "k_viterbi_re"
            bad = torch.nonzero((dout != o[idx]).any(1)).flatten()
            assert bad.numel() == 0, (cr, depth, look, bad.numel(), bad[:8].tolist(), idx[bad[:8]].tolist())
    del ds, dout, du
