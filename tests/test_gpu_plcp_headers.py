"""PLCP header cases (tests/plcp_inputs.py) on the device against the CPU oracle (pytest -m gpu): every refused and accepted header of
the 802.11a / b / n matrices, field by field, with the delivered bytes of decoded and CRC-failed frames; the same cases chained in
continuous captures, where what a context carries from one event to the next shows; rows narrower than the frames; and the legacy
entry points on a refused header.  The header table itself is pinned against the restatement of the parsers by test_cpu_plcp_headers.py,
and is asserted here too, so a device that agreed with a wrong oracle would still fail."""
import ctypes as C
import numpy as np, pytest
import oracle_py
import plcp_inputs as P
from sora_b200 import api, synth

pytestmark = pytest.mark.gpu

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

def _want(c):
    w = {"status": P.expected_status(c), **c["expect"]}
    return w if w["status"] != P.E_NONE else {"status": P.E_NONE}

def _same(res, ores, out, oout, fields, cases, nbytes):
    """Device == oracle on every field of every event, bytes of decoded / CRC-failed frames, and both == the restated header table."""
    assert (res["status"] == ores["status"]).all(), [(c["name"], hex(a), hex(b)) for c, a, b in zip(cases, res["status"], ores["status"]) if a != b]
    ev = ores["status"] != P.E_NONE
    for k in fields:
        bad = [(c["name"], int(a), int(b)) for c, a, b, e in zip(cases, res[k], ores[k], ev) if e and a != b]
        assert not bad, (k, bad)
    for i, c in enumerate(cases):
        if ores["status"][i] in (P.E_OK, P.E_CRC32):
            n = min(nbytes(int(ores["length"][i])), out.shape[1])
            assert (out[i, :n] == oout[i, :n]).all(), c["name"]
        w = _want(c)
        assert {k: int(res[i][k]) for k in w} == w, (c["name"], w)

LANE_MIN_DEFAULT = 16384                               # the library's own choice: the lane kernel from 16 384 code blocks on
F11A = ("rate_kbps", "length", "crc32", "nsym", "detect_index", "cfo_est")
F11B = ("rate_kbps", "length", "crc32", "sample_index", "detect_vec")
F11N = ("mcs", "length", "crc32", "nsym", "detect_index", "cfo_est", "lsig_length")

@pytest.mark.parametrize("viterbi", ["k_viterbi_re", "k_viterbi_lane"])
def test_headers_11a_batch(eng, viterbi):
    cases = P.cases_11a(); iq, off, ln = P.slots_of(cases)
    ores, oout = oracle_py.rx11a_batch(iq, off, ln, out_stride=2560)
    try:
        if viterbi == "k_viterbi_lane": eng.set_option("viterbi_lane_min", 0)
        res, out = eng.rx11a_batch(iq, off, ln, out_stride=2560)
        assert eng.last_viterbi_kernel() == viterbi
    finally:
        eng.set_option("viterbi_lane_min", LANE_MIN_DEFAULT)
    _same(res, ores, out, oout, F11A, cases, lambda L: L)

def test_headers_11b_batch(eng):
    cases = P.cases_11b(); iq, off, ln = P.slots_of(cases)
    ores, oout = oracle_py.rx11b_batch(iq, off, ln, out_stride=4096)
    res, out = eng.rx11b_batch(iq, off, ln, out_stride=4096)
    # a claim beyond 4096 bytes: the oracle's frame buffer wraps at 4096, the device clips at its 4096-byte row, and the reference writes
    # past its buffer, so the bytes of such a frame are not defined: its fields are compared, not its bytes
    _same(res, ores, out, oout, F11B, cases, lambda L: L - 1 if L <= 4096 else 0)

@pytest.mark.parametrize("mcs_limit", [11, 15])
def test_headers_11n_batch(eng, mcs_limit):
    cases = P.cases_11n(mcs_limit)
    iq0, off, ln = P.slots_of(cases, "iq0"); iq1, _, _ = P.slots_of(cases, "iq1")
    oracle_py.set_ht_mcs_limit(mcs_limit); eng.set_option("ht_mcs_limit", mcs_limit)
    try:
        ores, oout = oracle_py.rx11n_batch(iq0, iq1, off, ln, out_stride=1536)
        res, out = eng.rx11n_batch(iq0, iq1, off, ln, out_stride=1536)
    finally:
        oracle_py.set_ht_mcs_limit(11); eng.set_option("ht_mcs_limit", 11)
    _same(res, ores, out, oout, F11N, cases, lambda L: L)


def _stream_check(res, cnt, ores, oout, out, fields, nbytes, want, keep=None):
    assert cnt == len(ores), (cnt, ores, res[:cnt])
    for k in range(len(ores)):
        for f in ("status",) + fields:
            assert res[k][f] == ores[k][f], (k, f, res[k], ores[k])
        if ores[k]["status"] in (P.E_OK, P.E_CRC32):
            n = nbytes(int(ores[k]["length"])); assert (out[k, :n] == oout[k, :n]).all(), k
    ev = [r for r in res[:cnt] if keep is None or int(r["status"]) in keep]
    assert [{f: int(r[f]) for f in w} for r, w in zip(ev, want)] == want and len(ev) == len(want)

def test_streams_11a(eng):
    iq, want = P.stream_11a()
    ores, oout = oracle_py.rx11a_run(iq, max_frames=16, out_stride=2560)
    res, out, sidx, cnt = eng.rx11a_streams(iq, [0], [len(iq)], max_frames=16, out_stride=2560)
    _stream_check(res[0], cnt[0], ores, oout, out[0], ("rate_kbps", "length", "crc32", "nsym", "cfo_est"), lambda L: L, want)

def test_streams_11b(eng):
    iq, want = P.stream_11b()
    ores, oout = oracle_py.rx11b_run(iq, max_frames=32, out_stride=4096)
    res, out, cnt = eng.rx11b_streams(iq, [0], [len(iq)], max_frames=32, out_stride=4096)
    _stream_check(res[0], cnt[0], ores, oout, out[0], ("rate_kbps", "length", "sample_index", "detect_vec"), lambda L: L - 1, want,
                  keep=(P.E_OK, P.E_CRC32, P.E_PLCP))

@pytest.mark.parametrize("mcs_limit", [11, 15])
def test_streams_11n(eng, mcs_limit):
    """The MCS an L-SIG refusal reports is the event before's (CF_HTRxVector is never reset), its L-SIG length is 0."""
    iq0, iq1, want = P.stream_11n(mcs_limit)
    oracle_py.set_ht_mcs_limit(mcs_limit); eng.set_option("ht_mcs_limit", mcs_limit)
    try:
        ores, oout = oracle_py.rx11n_run(iq0, iq1, max_frames=16, out_stride=1536)
        res, out, sidx, cnt = eng.rx11n_streams(iq0, iq1, [0], [len(iq0)], max_frames=16)
        bres, _ = eng.rx11n_batch(iq0, iq1, [0], [len(iq0)])           # one slot = a fresh context: the first event only
    finally:
        oracle_py.set_ht_mcs_limit(11); eng.set_option("ht_mcs_limit", 11)
    assert (sidx[0, :cnt[0]] == ores["sample_index"]).all()
    _stream_check(res[0], cnt[0], ores, oout, out[0], ("mcs", "length", "crc32", "nsym", "cfo_est", "lsig_length"), lambda L: L, want)
    assert bres["status"][0] == P.E_OK and bres["mcs"][0] == 9

def test_batch_11n_lsig_refusal_reports_mcs_0(eng):
    """In one-slot-per-frame mode every slot starts from a fresh context: an L-SIG refusal reports MCS 0 whatever the slots before held."""
    byname = {c["name"]: c for c in P.cases_11n()}
    cases = [byname[n] for n in ("mcs_9", "lsig_parity", "mcs_10", "lsig_rate_illegal")]
    iq0, off, ln = P.slots_of(cases, "iq0"); iq1, _, _ = P.slots_of(cases, "iq1")
    res, _ = eng.rx11n_batch(iq0, iq1, off, ln)
    assert list(res["status"]) == [P.E_OK, P.E_PLCP, P.E_OK, P.E_PLCP] and list(res["mcs"]) == [9, 0, 10, 0]


def test_out_stride_narrower_than_frames(eng):
    """Rows of 100 bytes with 1500- and 2500-byte frames side by side: each row holds its own frame's first 100 bytes, nothing of the next."""
    cs = [P.case_11a("a1500", 54000, P.psdu(1500, 61)), P.case_11a("a2500", 48000, P.psdu(2500, 62)), P.case_11a("b1500", 36000, P.psdu(1500, 63))]
    res, out = eng.rx11a_batch(*P.slots_of(cs), out_stride=100)
    assert (res["status"] == P.E_OK).all() and out.shape == (3, 100)
    for c, o in zip(cs, out): assert (o == c["body"][:100]).all(), c["name"]
    cs = [P.case_11b("b1500", 11000, P.psdu(1500, 64)), P.case_11b("b2000", 5500, P.psdu(2000, 65)), P.case_11b("c1500", 11000, P.psdu(1500, 66))]
    res, out = eng.rx11b_batch(*P.slots_of(cs), out_stride=100)
    assert (res["status"] == P.E_OK).all()
    for c, o in zip(cs, out): assert (o == c["body"][:100]).all(), c["name"]
    cs = [P.case_11n("n1500", 10, P.psdu(1500, 67)), P.case_11n("n1000", 9, P.psdu(1000, 68)), P.case_11n("n1400", 10, P.psdu(1400, 69))]
    iq0, off, ln = P.slots_of(cs, "iq0"); iq1, _, _ = P.slots_of(cs, "iq1")
    res, out = eng.rx11n_batch(iq0, iq1, off, ln, out_stride=100)
    assert (res["status"] == P.E_OK).all()
    for c, o in zip(cs, out): assert (o == c["body"][:100]).all(), c["name"]


class _Stream(C.Structure): _fields_ = [("start", C.c_void_p), ("size", C.c_uint32), ("end", C.c_void_p), ("scan", C.c_void_p), ("mask", C.c_uint32)]

def _rx_blocks(cap):
    cap = cap[: len(cap) // 28 * 28]
    blocks = np.zeros((len(cap) // 28, 128), np.uint8); blocks[:, 0] = 1; blocks[:, 16:] = np.ascontiguousarray(cap).reshape(-1, 28 * 2).view(np.uint8)
    return blocks

def test_legacy_shim_11a_invalid_sig():
    """BB11ARxFrameDemod on a SIGNAL with its parity flipped, between two good frames: BB11A_E_INVALID_SIG, then the next frame."""
    lib = api.load_library()
    class Ctx(C.Structure):
        _fields_ = [("SampleRate", C.c_uint), ("thr", C.c_uint32), ("maxblk", C.c_uint), ("minblk", C.c_uint), ("work", C.c_void_p), ("frame", C.c_void_p),
                    ("framemax", C.c_uint), ("framesize", C.c_uint), ("datarate", C.c_uint), ("frametype", C.c_uint), ("engine", C.c_void_p), ("events", C.c_void_p), ("shift", C.c_uint)]
    for f in ("BB11ARxCarrierSense", "BB11ARxFrameDemod"): getattr(lib, f).restype = C.c_int32
    b = P.psdu(200, 71)
    cs = [P.case_11a("ok", 24000, b), P.case_11a("parity", 24000, b, synth.signal_word_11a(24000, 200) ^ 1 << 17), P.case_11a("ok2", 12000, P.psdu(80, 72))]
    blocks = _rx_blocks(np.concatenate([c["iq"] for c in cs]))
    work = C.c_uint32(1); frame = np.zeros(4096, np.uint8); st = _Stream(); ctx = Ctx()
    lib.SoraGenRadioRxStreamOffline(C.byref(st), C.c_void_p(blocks.ctypes.data), C.c_uint32(blocks.size))
    lib.BB11ARxContextInit(C.byref(ctx), 40, 250000, 150, 112, C.byref(work))
    got = []
    for _ in range(10000):
        hr = lib.BB11ARxCarrierSense(C.byref(ctx), C.byref(st))
        if hr == 0x201:
            lib.BB11APrepareRx(C.byref(ctx), C.c_void_p(frame.ctypes.data), 4096)
            got.append((lib.BB11ARxFrameDemod(C.byref(ctx), C.byref(st)) & 0xFFFFFFFF, ctx.framesize, ctx.datarate))
        if st.scan == st.start and got: break
    lib.BB11ARxContextCleanup(C.byref(ctx))
    assert [g[0] for g in got] == [0x202, 0x80006002, 0x202], [hex(g[0]) for g in got]
    assert got[0][1:] == (200, 24000) and got[2][1:] == (80, 12000)

def test_legacy_shim_11b_plcp_header_crc():
    """BB11BRx on a PLCP header with a CRC-16 bit flipped, between two good frames: BB11B_E_PLCP_HEADER_CRC and b_errPLCPHeader counts it."""
    lib = api.load_library()
    class C16(C.Structure): _fields_ = [("re", C.c_int16), ("im", C.c_int16)]
    class Common(C.Structure):
        _fields_ = [("b_length", C.c_uint), ("b_dataRate", C.c_ubyte), ("b_isLongPreamble", C.c_char), ("b_crc32", C.c_ulong), ("b_errEnergyLoss", C.c_uint), ("b_errFrame", C.c_uint),
                    ("b_errPLCPHeader", C.c_uint), ("b_goodFrameCounter", C.c_uint), ("b_outputPt", C.c_void_p), ("b_maxOutputSize", C.c_uint32)]
    class Rx(C.Structure):
        _fields_ = [("b_maxDescCount", C.c_uint), ("b_resetFlag", C.c_int), ("b_energyLeast", C.c_short), ("b_workIndicator", C.c_void_p), ("b_shiftRight", C.c_int), ("b_dcOffset", C16),
                    ("BB11bCommon", Common), ("engine", C.c_void_p), ("events", C.c_void_p)]
    class Spd(C.Structure):
        _fields_ = [("b_minDescCount", C.c_uint), ("b_maxDescCount", C.c_uint), ("b_threshold", C.c_uint), ("b_thresholdLH", C.c_uint), ("b_thresholdHL", C.c_uint), ("b_gainLevel", C.c_uint),
                    ("b_gainLevelNext", C.c_uint), ("b_resetFlag", C.c_int), ("b_workIndicator", C.c_void_p), ("b_dcOffset", C16), ("b_reestimateOffset", C.c_char), ("b_evalEnergy", C.c_ulong),
                    ("rx", C.c_void_p)]
    for f in ("BB11BSpd", "BB11BRx"): getattr(lib, f).restype = C.c_int32
    gap = np.zeros((2000, 2), np.int16)
    cs = [P.case_11b("ok", 11000, P.psdu(120, 73)), P.case_11b("crc16", 2000, P.psdu(60, 74), synth.plcp_11b(60, 2000) + (0x0004,)),
          P.case_11b("ok2", 2000, P.psdu(60, 75))]
    blocks = _rx_blocks(np.concatenate([x for c in cs for x in (c["iq"], gap)]))
    work = C.c_uint32(1); outbuf = np.zeros(4096, np.uint8); st = _Stream(); rx = Rx(); spd = Spd()
    lib.SoraGenRadioRxStreamOffline(C.byref(st), C.c_void_p(blocks.ctypes.data), C.c_uint32(blocks.size))
    lib.BB11BRxSpdContextInit(C.byref(rx), C.byref(spd), C.byref(work), 0xFFFFFFF, blocks.shape[0], 15, 4000, 4000, 4000, 0)
    lib.BB11BPrepareRx(C.byref(rx), C.c_void_p(outbuf.ctypes.data), 4096)
    got = []
    for _ in range(1000):
        spd.b_resetFlag = 1
        if lib.BB11BSpd(C.byref(spd), C.byref(st)) != 0x101: break
        rx.b_resetFlag = 1
        for _ in range(8):
            hr = lib.BB11BRx(C.byref(rx), C.byref(st)) & 0xFFFFFFFF
            if hr in (0x7F, 0x80050105, 0x80050210): got.append(hr)
            if hr in (0x7F, 0x80050105, 0x80050100, 0x80050103, 0x80050210): break
            rx.b_resetFlag = 0
    errs = rx.BB11bCommon.b_errPLCPHeader; good = rx.BB11bCommon.b_goodFrameCounter
    lib.BB11BRxSpdContextCleanUp(C.byref(rx))
    assert got == [0x7F, 0x80050210, 0x7F], [hex(g) for g in got]
    assert errs == 1 and good == 2
