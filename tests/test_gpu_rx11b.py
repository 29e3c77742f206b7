"""GPU parity tests, 802.11b: CUDA path through the C ABI vs the CPU oracle on the same IQ."""
import os, numpy as np, pytest
import oracle_py
from sora_b200 import api, synth
from test_cpu_oracle_11b import _fixture, FRAME

pytestmark = pytest.mark.gpu

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

def _cmp(eng, iq2, off, ln):
    res, out = eng.rx11b_batch(iq2, off, ln)
    ores, oout = oracle_py.rx11b_batch(iq2, off, ln, out_stride=out.shape[1])
    assert (res["status"] == ores["status"]).all(), (res["status"], ores["status"])
    ev = ores["status"] != oracle_py.E_NO_FRAME
    for k in ("rate_kbps", "length", "crc32", "sample_index", "detect_vec"):
        assert (res[k][ev] == ores[k][ev]).all(), (k, res[k], ores[k])
    for i in np.nonzero(ev)[0]:
        if ores["status"][i] in (1, oracle_py.E_CRC32_FAIL):
            L = int(ores["length"][i]) - 1
            assert (out[i, :L] == oout[i, :L]).all(), f"slot {i}"
    return res, out

def test_reference_fixtures(eng):
    for name, rate in (("1long44.mf.bin", 1000), ("2long44.mf.bin", 2000)):
        iq = _fixture(name)
        res, out = _cmp(eng, iq, np.array([0], np.uint64), np.array([len(iq)], np.uint32))
        assert res[0]["status"] == 1 and res[0]["rate_kbps"] == rate and (out[0, :113] == FRAME[:113]).all()

@pytest.mark.parametrize("rate", [1000, 2000, 5500, 11000])
def test_all_rates(eng, rate):
    for snr, gain in ((None, 1.0), (40, 0.3), (28, 0.25), (18, 0.2)):
        iq, ps = synth.make_frames_11b(5, psdu_len=96, rate_kbps=rate, snr_db=snr, gain=gain, seed0=rate + 7)
        F, slot, _ = iq.shape
        res, out = _cmp(eng, iq.reshape(-1, 2), np.arange(F, dtype=np.uint64) * slot, np.full(F, slot, np.uint32))
        if snr in (None, 40):
            # frame 2 of the clean 11 Mbps frames at gain 1.0 (peak 32512) fails its FCS in the reference's own chain too
            # (test_gpu_rx11b_reference.py::test_full_scale_11m_equals_the_reference); every other frame must decode
            ok = np.ones(F, bool)
            if rate == 11000 and snr is None: ok[2] = False
            assert (res["status"][ok] == 1).all() and (out[ok, :95] == ps[ok, :95]).all()

def test_edges(eng):
    rng = np.random.default_rng(4)
    noise = rng.normal(0, 2500, (3, 28 * 300, 2)).astype(np.int16)
    _cmp(eng, noise.reshape(-1, 2), np.arange(3, dtype=np.uint64) * 8400, np.full(3, 8400, np.uint32))
    iq, _ = synth.make_frames_11b(4, psdu_len=200, rate_kbps=11000, snr_db=40, gain=0.3)
    F, slot, _ = iq.shape
    ln = np.array([slot, slot // 2, 3000, 27], np.uint32)          # truncated / tiny slots
    _cmp(eng, iq.reshape(-1, 2), np.arange(F, dtype=np.uint64) * slot, ln)
    z = np.zeros((2, 5600, 2), np.int16)
    _cmp(eng, z.reshape(-1, 2), np.arange(2, dtype=np.uint64) * 5600, np.full(2, 5600, np.uint32))


def _capture_11b(seed, specs, noise=0.0):
    """A continuous 44 Msps capture: frames made by the transmit oracle (rate, length, corrupt?) separated by silence."""
    rng = np.random.default_rng(seed); parts = [np.zeros((rng.integers(300, 900) // 4 * 4, 2), np.int16)]; pays = []
    for rate, L, corrupt in specs:
        p = rng.integers(0, 256, L).astype(np.uint8); pays.append(p)
        td = oracle_py.tx11b_modulate(p, rate).astype(np.int16) << 8
        if corrupt: k = len(td) * 3 // 4; td[k:k + 400] = -td[k:k + 400]
        parts.append(td); parts.append(np.zeros((int(rng.integers(700, 3000)), 2), np.int16))
    iq = np.concatenate(parts)
    if noise: iq = (iq + rng.normal(0, noise, iq.shape)).clip(-32768, 32767).astype(np.int16)
    return iq, pays

def test_streams_match_oracle_driver(eng):
    """Continuous captures through sb200_rx11b_streams == the restated MAC11b_Receive loop (oracle Rx11b::run): same events in the
    same order, same positions, same bytes — including a CRC failure, the seek past the last FCS byte and the carried-over state."""
    caps = [_capture_11b(1, [(11000, 300, False), (2000, 60, False), (5500, 200, True), (11000, 1000, False), (1000, 40, False)], noise=60.0),
            _capture_11b(2, [(5500, 500, False), (11000, 77, False)]),
            _capture_11b(3, [(2000, 100, True), (1000, 30, False), (11000, 1496, False)], noise=120.0),
            (np.zeros((5000, 2), np.int16), [])]
    off = np.cumsum([0] + [(len(c[0]) + 3) // 4 * 4 for c in caps[:-1]]).astype(np.uint64)
    total = int(off[-1]) + len(caps[-1][0]); iq = np.zeros((total, 2), np.int16)
    for o, c in zip(off, caps): iq[int(o):int(o) + len(c[0])] = c[0]
    ln = np.array([len(c[0]) for c in caps], np.uint32)
    res, out, cnt = eng.rx11b_streams(iq, off, ln, max_frames=8, out_stride=2048)
    nok = 0
    for s, c in enumerate(caps):
        ores, oout = oracle_py.rx11b_run(c[0], max_frames=8, out_stride=2048)
        assert cnt[s] == len(ores), (s, cnt[s], len(ores), res[s, :cnt[s]], ores)
        for k in range(len(ores)):
            for fld in ("status", "rate_kbps", "length", "sample_index", "detect_vec"):
                assert res[s, k][fld] == ores[k][fld], (s, k, fld, res[s, k], ores[k])
            assert (res[s, k]["crc32"] & 0xFFFFFF) == (ores[k]["crc32"] & 0xFFFFFF)
            if ores[k]["status"] in (1, 0x80000006):
                n = int(ores[k]["length"]) - 1                       # the sink stops one byte short of the FCS end (PHY_11b.hpp:728-739)
                assert (out[s, k, :n] == oout[k, :n]).all(), (s, k)
            nok += int(ores[k]["status"] == 1)
        assert (res[s, cnt[s]:]["status"] == 0).all()
    assert nok >= 7 and cnt[3] == 0
    # max_frames smaller than the number of events: the first ones, in order
    res2, _, cnt2 = eng.rx11b_streams(iq, off, ln, max_frames=2, out_stride=64)
    for s in range(len(caps)):
        assert cnt2[s] == min(2, cnt[s]) and (res2[s, :cnt2[s]] == res[s, :cnt2[s]]).all()


def test_legacy_c_api_shim_11b():
    """The driver loop of kernel/bb/demod11/demod11b.cpp:73-174 (BB11BSpd until power is detected, BB11BRx until the frame is settled)
    written against include/sora_b200_legacy.h via ctypes, over RX_BLOCKs holding frames from the transmit oracle."""
    import ctypes as C
    lib = api.load_library()
    class Stream(C.Structure): _fields_ = [("start", C.c_void_p), ("size", C.c_uint32), ("end", C.c_void_p), ("scan", C.c_void_p), ("mask", C.c_uint32)]
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
    cap, pays = _capture_11b(5, [(11000, 400, False), (2000, 90, False), (5500, 150, True), (1000, 33, False)], noise=40.0)
    cap = cap[: len(cap) // 28 * 28]
    blocks = np.zeros((len(cap) // 28, 128), np.uint8); blocks[:, 0] = 1; blocks[:, 16:] = np.ascontiguousarray(cap).reshape(-1, 28 * 2).view(np.uint8)
    ores, oout = oracle_py.rx11b_run(cap, max_frames=16, out_stride=4096)
    frames = [(int(o["status"]), int(o["length"]), int(o["rate_kbps"]), ob) for o, ob in zip(ores, oout) if o["status"] in (1, oracle_py.E_CRC32_FAIL)]
    work = C.c_uint32(1); outbuf = np.zeros(4096, np.uint8)
    st = Stream(); rx = Rx(); spd = Spd()
    lib.SoraGenRadioRxStreamOffline(C.byref(st), C.c_void_p(blocks.ctypes.data), C.c_uint32(blocks.size))
    lib.BB11BRxSpdContextInit(C.byref(rx), C.byref(spd), C.byref(work), 0xFFFFFFF, blocks.shape[0], 15, 4000, 4000, 4000, 0)
    lib.BB11BPrepareRx(C.byref(rx), C.c_void_p(outbuf.ctypes.data), 4096)
    got = []; done = False
    for _ in range(1000):
        spd.b_resetFlag = 1
        hr = lib.BB11BSpd(C.byref(spd), C.byref(st))
        if hr != 0x101: break                              # BB11B_CHANNEL_CLEAN: the offline loop ends (demod11b.cpp:102-103)
        rx.b_resetFlag = 1
        for _ in range(8):
            hr = lib.BB11BRx(C.byref(rx), C.byref(st)) & 0xFFFFFFFF
            if hr in (0x7F, 0x80050105): got.append((hr, rx.BB11bCommon.b_length, rx.BB11bCommon.b_dataRate, outbuf[:rx.BB11bCommon.b_length].copy()))
            if hr in (0x7F, 0x80050105, 0x80050100, 0x80050103): break     # demod11b.cpp:172-173
            rx.b_resetFlag = 0
    good = rx.BB11bCommon.b_goodFrameCounter; bad = rx.BB11bCommon.b_errFrame
    lib.BB11BRxSpdContextCleanUp(C.byref(rx))
    assert len(got) == len(frames) == 4, (len(got), len(frames), [hex(g[0]) for g in got])
    code = {1000: 0x0A, 2000: 0x14, 5500: 0x37, 11000: 0x6E}
    for (hr, n, rc, by), (stt, L, rate, ob) in zip(got, frames):
        assert hr == (0x7F if stt == 1 else 0x80050105) and n == L and rc == code[rate] and (by[:L - 1] == ob[:L - 1]).all()
    assert good == 3 and bad == 1
