"""GPU tests for the legacy 802.11b transmitter (pytest -m gpu): sb200_tx11b_legacy_batch against the restatement (oracle_tx11b_legacy.py) and,
where oracle/_ref travelled with the tree, the reference's compiled encoder; device TX -> device RX; and the legacy entry points of
sora_b200_legacy.h through ctypes."""
import ctypes as C, zlib, numpy as np, pytest
import oracle_py
import oracle_tx11b_legacy as O
from sora_b200 import api

pytestmark = pytest.mark.gpu
RATES = [1000, 2000, 5500, 11000]
E_FAIL = C.c_int32(0x80004005).value


@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)


def payloads(rng, F):
    lens = list(rng.integers(0, 1600, F)); lens[0] = 0; lens[1] = 1; lens[2] = 4091; lens[3] = 63
    return [rng.integers(0, 256, int(n)).astype(np.uint8) for n in lens]


@pytest.mark.parametrize("filt", [0, 1, 2])
@pytest.mark.parametrize("short", [False, True])
@pytest.mark.parametrize("rate", RATES)
def test_device_equals_oracle_mixed_lengths(eng, rate, short, filt):
    rng = np.random.default_rng(rate * 7 + short * 3 + filt)
    pay = payloads(rng, 9)
    out, ns = eng.tx11b_legacy_batch(pay, rate, short_preamble=short, filter=filt)
    for i, p in enumerate(pay):
        want = O.modulate(p, rate, short, filt)
        assert ns[i] == len(want) and (out[i, :ns[i]] == want).all(), (i, len(p))
        assert (out[i, ns[i]:] == 0).all()
    if filt == 0 and O.ref_available():
        for i in (0, 2, 5):
            b, _ = O.ref_encode(np.concatenate([pay[i], np.frombuffer(zlib.crc32(bytes(pay[i])).to_bytes(4, "little"), np.uint8)]), rate, short)
            assert (out[i, :ns[i]] == b).all()


def test_fcs_in_payload_and_device_pointers(eng):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(3)
    pay = [rng.integers(0, 256, n).astype(np.uint8) for n in (4, 40, 1000)]
    pay[1][-4:] = [1, 2, 3, 4]                                           # an FCS that is not the CRC: sent verbatim
    lens = np.array([len(p) for p in pay], np.uint32); offs = np.concatenate([[0], np.cumsum(lens[:-1])]).astype(np.uint64)
    stride = 64 * 1024 * 2
    dev = torch.device("cuda", 0)
    d_pay = torch.from_numpy(np.concatenate(pay)).to(dev); d_off = torch.from_numpy(offs.view(np.int64)).to(dev); d_len = torch.from_numpy(lens.view(np.int32)).to(dev)
    d_out = torch.full((len(pay), stride, 2), 99, dtype=torch.int8, device=dev); d_ns = torch.zeros(len(pay), dtype=torch.int32, device=dev)
    for filt in (0, 1, 2):
        for short in (0, 1):
            eng.tx11b_legacy_raw(d_pay.data_ptr(), int(lens.sum()), d_off.data_ptr(), d_len.data_ptr(), len(pay), 11000, short, api.Engine.TX11B_LEGACY_FCS_IN_PAYLOAD,
                                 filt, d_out.data_ptr(), stride, d_ns.data_ptr())
            torch.cuda.synchronize()
            out = d_out.cpu().numpy(); ns = d_ns.cpu().numpy()
            for i, p in enumerate(pay):
                want = O.modulate(p, 11000, bool(short), filt, fcs_in_payload=True)
                assert ns[i] == len(want) and (out[i, :ns[i]] == want).all() and (out[i, ns[i]:] == 0).all()


def test_refusals(eng):
    p = [np.zeros(10, np.uint8)]
    for kw in (dict(rate_kbps=6000), dict(filter=3)):
        with pytest.raises(api.Sb200Error):
            eng.tx11b_legacy_batch(p, kw.get("rate_kbps", 2000), filter=kw.get("filter", 1))
    out = np.zeros((1, 1 << 16, 2), np.int8); ns = np.zeros(1, np.uint32); off = np.zeros(1, np.uint64); ln = np.array([10], np.uint32)
    with pytest.raises(api.Sb200Error, match="PBCC"):
        eng.tx11b_legacy_raw(p[0].ctypes.data, 10, off.ctypes.data, ln.ctypes.data, 1, 11000, 0, 2, 1, out.ctypes.data, 1 << 16, ns.ctypes.data)
    with pytest.raises(api.Sb200Error):                                  # out_stride too small
        eng.tx11b_legacy_raw(p[0].ctypes.data, 10, off.ctypes.data, ln.ctypes.data, 1, 1000, 0, 0, 1, out.ctypes.data, 1024, ns.ctypes.data)
    ln[0] = 3
    with pytest.raises(api.Sb200Error):                                  # FCS in payload needs 4 bytes
        eng.tx11b_legacy_raw(p[0].ctypes.data, 10, off.ctypes.data, ln.ctypes.data, 1, 11000, 0, 1, 1, out.ctypes.data, 1 << 16, ns.ctypes.data)


@pytest.mark.parametrize("rate", RATES)
def test_device_tx_then_device_rx(eng, rate):
    rng = np.random.default_rng(rate + 1)
    pay = [rng.integers(0, 256, n).astype(np.uint8) for n in (1, 100, 777, 1500)]
    out, ns = eng.tx11b_legacy_batch(pay, rate, short_preamble=False, filter=1)
    slot = (280 + int(ns.max()) + 56 + 27) // 28 * 28
    iq = np.zeros((len(pay), slot, 2), np.int16)
    for i in range(len(pay)): iq[i, 280:280 + ns[i]] = out[i, :ns[i]].astype(np.int16) << 8
    res, got = eng.rx11b_batch(iq.reshape(-1, 2), np.arange(len(pay), dtype=np.uint64) * slot, np.full(len(pay), slot, np.uint32))
    for i, p in enumerate(pay):
        assert res[i]["status"] == api.FRAME_OK and res[i]["rate_kbps"] == rate and res[i]["length"] == len(p) + 4, (i, res[i])
        assert (got[i, :len(p)] == p).all()


# ---- the legacy entry points (sora_b200_legacy.h) ---------------------------------------------------------------------------------------
class TXV(C.Structure):
    _fields_ = [("DateRate", C.c_uint8), ("PreambleType", C.c_uint8), ("ModSelect", C.c_uint8)]
class MDL(C.Structure):
    pass
MDL._fields_ = [("Next", C.POINTER(MDL)), ("StartVa", C.c_void_p), ("ByteOffset", C.c_uint32), ("ByteCount", C.c_uint32)]
class TXD(C.Structure):
    _fields_ = [("pSampleBuffer", C.c_void_p), ("SampleBufferSize", C.c_uint32), ("SignalLength", C.c_uint32)]
class PKT(C.Structure):
    _fields_ = [("pMdl", C.POINTER(MDL)), ("pTxDesc", C.POINTER(TXD)), ("fStatus", C.c_int32), ("PacketSize", C.c_uint32), ("Reserved1", C.c_uint32),
                ("Reserved2", C.c_uint32), ("Reserved3", C.c_uint32), ("Reserved4", C.c_uint32), ("pReserved", C.c_void_p)]
MAX_SYM = (1500 + 24 + 4) * 8 * 4 * 11 * 2


def _lib():
    lib = api.load_library()
    for n in ("BB11BPMDBufferTx4XWithShortHeader", "BB11BPMDBufferTx4XWithLongHeader", "BB11BPMDPacketTx4X", "BB11BPMDPacketGenSignal"):
        getattr(lib, n).restype = C.c_int32
    return lib


@pytest.mark.parametrize("short", [False, True])
def test_buffer_entry_points_scramble_in_place(short):
    lib = _lib(); v = TXV()
    lib.BB11BTxVectorInit(C.byref(v), C.c_uint8(0x37), C.c_uint8(0), C.c_uint8(1 if short else 0))
    assert (v.DateRate, v.ModSelect, v.PreambleType) == (0x37, 0, 1 if short else 0)
    psdu = np.concatenate([np.arange(200, dtype=np.uint8), np.zeros(4, np.uint8)]); psdu[-4:] = np.frombuffer(zlib.crc32(bytes(psdu[:-4])).to_bytes(4, "little"), np.uint8)
    buf = psdu.copy(); out = np.zeros((1 << 16, 2), np.int8); n = C.c_uint32(0)
    fn = lib.BB11BPMDBufferTx4XWithShortHeader if short else lib.BB11BPMDBufferTx4XWithLongHeader
    assert fn(C.byref(v), C.c_void_p(buf.ctypes.data), C.c_uint32(200), C.c_void_p(out.ctypes.data), C.byref(n)) == 0
    want, scr = O.encode(psdu, 5500, short)
    assert n.value == len(want) and (out[:n.value] == want).all() and (buf == scr).all()
    v.ModSelect = 1
    assert fn(C.byref(v), C.c_void_p(buf.ctypes.data), C.c_uint32(200), C.c_void_p(out.ctypes.data), C.byref(n)) == E_FAIL      # PBCC


def test_packet_entry_points():
    lib = _lib(); v = TXV(0x14, 1, 0)
    rng = np.random.default_rng(12)
    a = rng.integers(0, 256, 30).astype(np.uint8); b = rng.integers(0, 256, 11).astype(np.uint8)
    fcs = zlib.crc32(bytes(a) + bytes(b))
    m2 = MDL(None, C.c_void_p(b.ctypes.data), 0, len(b)); m1 = MDL(C.pointer(m2), C.c_void_p(a.ctypes.data - 3), 3, len(a))
    samples = np.zeros((MAX_SYM // 2, 2), np.int8); txd = TXD(C.c_void_p(samples.ctypes.data), MAX_SYM, 0)
    pkt = PKT(C.pointer(m1), C.pointer(txd), 0, len(a) + len(b), fcs)
    a0, b0 = a.copy(), b.copy()
    temp = np.zeros(MAX_SYM + 64, np.uint8)
    assert lib.BB11BPMDPacketGenSignal(C.byref(pkt), C.byref(v), C.c_void_p(temp.ctypes.data), C.c_uint32(MAX_SYM)) == 0
    psdu = np.concatenate([a0, b0, np.frombuffer(fcs.to_bytes(4, "little"), np.uint8)])
    enc, scr = O.encode(psdu, 2000, True)
    assert (temp[:2 * len(enc)] == enc.reshape(-1).view(np.uint8)).all() and (temp[2 * len(enc): 2 * len(enc) + 64] == 0).all()
    assert txd.SignalLength == 2 * len(enc) and (samples[:len(enc)] == oracle_py.fir37_legacy(enc, 0)).all()
    assert (np.concatenate([a, b]) == scr[:-4]).all() and pkt.Reserved1 == int.from_bytes(bytes(scr[-4:]), "little")     # scrambled in place
    out = np.zeros((1 << 16, 2), np.int8); n = C.c_uint32(0)
    pkt.Reserved1 = fcs; a[:] = a0; b[:] = b0
    assert lib.BB11BPMDPacketTx4X(C.byref(v), C.byref(pkt), C.c_void_p(out.ctypes.data), C.c_uint32(0), C.byref(n)) == 0
    assert n.value == len(enc) and (out[:n.value] == enc).all()
    v.PreambleType = 2
    assert lib.BB11BPMDPacketTx4X(C.byref(v), C.byref(pkt), C.c_void_p(out.ctypes.data), C.c_uint32(0), C.byref(n)) == E_FAIL          # bbb_tx.c:94-97
    v.PreambleType = 1
    assert lib.BB11BPMDPacketGenSignal(C.byref(pkt), C.byref(v), C.c_void_p(temp.ctypes.data), C.c_uint32(MAX_SYM - 1)) == E_FAIL       # short buffers
    txd.SampleBufferSize = MAX_SYM - 1
    assert lib.BB11BPMDPacketGenSignal(C.byref(pkt), C.byref(v), C.c_void_p(temp.ctypes.data), C.c_uint32(MAX_SYM)) == E_FAIL
