"""GPU tests for the legacy 802.11a transmitter (pytest -m gpu): sb200_tx11a_legacy_batch against the oracle (oracle_tx11a_legacy.py) bit for
bit, padding included; device TX -> device RX at 40 and 44 Msps; and BB11ATxFrameMod / BB11AModulateACK of sora_b200_legacy.h through ctypes."""
import ctypes as C, os
import numpy as np, pytest
import oracle_tx11a_legacy as O
from sora_b200 import api

pytestmark = pytest.mark.gpu
E_FAIL = C.c_int32(0x80004005).value
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PRE = O.preamble()


@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)


def _check(out, ns, pay, kbps, sr, append_crc=True):
    for i, p in enumerate(pay):
        want = O.modulate(p, kbps, sr, append_crc=append_crc)
        assert ns[i] == len(want), (i, len(p), ns[i], len(want))
        assert (out[i, :ns[i]] == want).all(), (i, len(p), np.flatnonzero((out[i, :ns[i]] != want).any(axis=1))[:8])
        assert (out[i, ns[i]:] == 0).all()


@pytest.mark.parametrize("sr", [40, 44])
@pytest.mark.parametrize("kbps", O.RATES)
def test_device_equals_oracle_mixed_lengths(eng, kbps, sr):
    rng = np.random.default_rng(kbps + sr)
    lens = [0, 1, 2, 3, 13, 63, 64, 1500, 4092] + list(rng.integers(0, 2400, 5))
    pay = [rng.integers(0, 256, int(n)).astype(np.uint8) for n in lens]
    out, ns = eng.tx11a_legacy_batch(pay, kbps, PRE, sample_rate_mhz=sr)
    _check(out, ns, pay, kbps, sr)


@pytest.mark.parametrize("sr", [40, 44])
def test_every_length_0_to_64_and_a_sweep(eng, sr):
    rng = np.random.default_rng(sr)
    for kbps in (6000, 9000, 54000):
        lens = list(range(65)) + list(range(65, 4093, 97)) + [4092]
        pay = [rng.integers(0, 256, n).astype(np.uint8) for n in lens]
        out, ns = eng.tx11a_legacy_batch(pay, kbps, PRE, sample_rate_mhz=sr)
        _check(out, ns, pay, kbps, sr)


@pytest.mark.parametrize("sr", [40, 44])
def test_fcs_in_payload_device_pointers(eng, sr):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(3)
    pay = [rng.integers(0, 256, n).astype(np.uint8) for n in (4, 14, 40, 1000, 4096)]
    pay[2][-4:] = [1, 2, 3, 4]                                          # an FCS that is not the CRC: sent verbatim
    lens = np.array([len(p) for p in pay], np.uint32); offs = np.concatenate([[0], np.cumsum(lens[:-1])]).astype(np.uint64)
    stride = api.Engine.tx11a_legacy_nsamples(4096, 12000, sr) + 64
    dev = torch.device("cuda", 0)
    d_pay = torch.from_numpy(np.concatenate(pay)).to(dev); d_off = torch.from_numpy(offs.view(np.int64)).to(dev); d_len = torch.from_numpy(lens.view(np.int32)).to(dev)
    d_pre = torch.from_numpy(PRE.copy()).to(dev)
    d_out = torch.full((len(pay), stride, 2), 99, dtype=torch.int8, device=dev); d_ns = torch.zeros(len(pay), dtype=torch.int32, device=dev)
    eng.tx11a_legacy_raw(d_pay.data_ptr(), int(lens.sum()), d_off.data_ptr(), d_len.data_ptr(), len(pay), 12000, sr, api.Engine.TX11A_LEGACY_FCS_IN_PAYLOAD,
                         d_pre.data_ptr(), d_out.data_ptr(), stride, d_ns.data_ptr())
    torch.cuda.synchronize()
    _check(d_out.cpu().numpy(), d_ns.cpu().numpy(), pay, 12000, sr, append_crc=False)


def test_device_reproduces_ofdm_bin(eng):
    ref = np.fromfile(os.path.join(GOLD, "ofdm.bin"), np.int8).reshape(-1, 2)
    out, ns = eng.tx11a_legacy_batch([np.full(200, 0x31, np.uint8)], 24000, PRE)
    assert (out[0, :3680] == ref[:3680]).all()


def test_refusals(eng):
    p = [np.zeros(10, np.uint8)]
    with pytest.raises(api.Sb200Error):
        eng.tx11a_legacy_batch(p, 11000, PRE)                           # not an 802.11a rate
    with pytest.raises(api.Sb200Error):
        eng.tx11a_legacy_batch(p, 6000, PRE, sample_rate_mhz=20)        # the reference ASSERTs
    with pytest.raises(api.Sb200Error):
        eng.tx11a_legacy_batch([np.zeros(4093, np.uint8)], 6000, PRE)   # MPDU + FCS 4097
    with pytest.raises(api.Sb200Error):
        eng.tx11a_legacy_batch([np.zeros(4097, np.uint8)], 6000, PRE, fcs_in_payload=True)
    with pytest.raises(api.Sb200Error):
        eng.tx11a_legacy_batch([np.zeros(3, np.uint8)], 6000, PRE, fcs_in_payload=True)
    with pytest.raises(api.Sb200Error):                                 # slot too small
        eng.tx11a_legacy_batch(p, 6000, PRE, out_stride=api.Engine.tx11a_legacy_nsamples(14, 6000) - 64)


@pytest.mark.parametrize("sr", [40, 44])
@pytest.mark.parametrize("kbps", O.RATES)
def test_device_tx_then_device_rx(eng, kbps, sr):
    rng = np.random.default_rng(kbps * 3 + sr)
    pay = [rng.integers(0, 256, n).astype(np.uint8) for n in (1, 100, 777, 1500)]
    out, ns = eng.tx11a_legacy_batch(pay, kbps, PRE, sample_rate_mhz=sr)
    slot = (800 + int(ns.max()) + 1200 + 27) // 28 * 28
    iq = np.zeros((len(pay), slot, 2), np.int16)
    for i in range(len(pay)): iq[i, 800:800 + ns[i]] = out[i, :ns[i]].astype(np.int16) << 8
    off = np.arange(len(pay), dtype=np.uint64) * slot; ln = np.full(len(pay), slot, np.uint32)
    res, got = eng.rx11a_batch(iq.reshape(-1, 2), off, ln, sample_rate_mhz=sr) if sr == 44 else eng.rx11a_batch(iq.reshape(-1, 2), off, ln)
    for i, p in enumerate(pay):
        assert res[i]["status"] == api.FRAME_OK and res[i]["rate_kbps"] == kbps and res[i]["length"] == len(p) + 4, (i, res[i])
        assert (got[i, :len(p)] == p).all()


# ---- the legacy entry points (sora_b200_legacy.h) ---------------------------------------------------------------------------------------
class TXV(C.Structure):
    _fields_ = [("SampleRate", C.c_uint), ("ti_uiDataRate", C.c_uint), ("ti_uiBufferLength", C.c_uint)]
class MDL(C.Structure):
    pass
MDL._fields_ = [("Next", C.POINTER(MDL)), ("StartVa", C.c_void_p), ("ByteOffset", C.c_uint32), ("ByteCount", C.c_uint32)]
class TXD(C.Structure):
    _fields_ = [("pSampleBuffer", C.c_void_p), ("SampleBufferSize", C.c_uint32), ("SignalLength", C.c_uint32)]
class PKT(C.Structure):
    _fields_ = [("pMdl", C.POINTER(MDL)), ("pTxDesc", C.POINTER(TXD)), ("fStatus", C.c_int32), ("PacketSize", C.c_uint32), ("Reserved1", C.c_uint32),
                ("Reserved2", C.c_uint32), ("Reserved3", C.c_uint32), ("Reserved4", C.c_uint32), ("pReserved", C.c_void_p)]
class MAC(C.Structure):
    _fields_ = [("Address", C.c_uint8 * 6)]


def _lib():
    lib = api.load_library()
    lib.BB11ATxFrameMod.restype = C.c_int32
    lib.BB11AModulateACK.restype = C.c_uint32
    lib.BB11ATxSetPreamble.argtypes = [C.c_void_p]
    return lib


@pytest.mark.parametrize("sr", [40, 44])
def test_frame_mod_and_ack(sr):
    lib = _lib(); v = TXV(0, 0xD, 77)
    lib.BB11ATxContextInit(C.byref(v), C.c_uint(sr))
    assert (v.SampleRate, v.ti_uiDataRate, v.ti_uiBufferLength) == (sr, 0xD, 0)
    rng = np.random.default_rng(sr)
    a = rng.integers(0, 256, 30).astype(np.uint8); b = rng.integers(0, 256, 11).astype(np.uint8)
    fcs = 0x12345678                                                    # sent as it is: BB11ATxFrameMod does not compute the FCS
    m2 = MDL(None, C.c_void_p(b.ctypes.data), 0, len(b)); m1 = MDL(C.pointer(m2), C.c_void_p(a.ctypes.data - 3), 3, len(a))
    cap = 1 << 16
    samples = np.full(cap, 0xAA, np.uint8); txd = TXD(C.c_void_p(samples.ctypes.data), cap, 0)
    pkt = PKT(C.pointer(m1), C.pointer(txd), 0, len(a) + len(b), fcs)
    lib.BB11ATxSetPreamble(None)
    assert lib.BB11ATxFrameMod(C.byref(v), C.byref(pkt)) == E_FAIL    # preamble not set
    ra = MAC((C.c_uint8 * 6)(*range(0x10, 0x16)))
    assert lib.BB11AModulateACK(C.c_uint(sr), C.byref(ra), C.c_void_p(samples.ctypes.data)) == 0 and (samples == 0xAA).all()
    pre = PRE.copy()
    lib.BB11ATxSetPreamble(C.c_void_p(pre.ctypes.data))
    assert lib.BB11ATxFrameMod(C.byref(v), C.byref(pkt)) == 0
    psdu = np.concatenate([a, b, np.frombuffer(fcs.to_bytes(4, "little"), np.uint8)])
    want = O.modulate(psdu, 36000, sr, append_crc=False)
    assert txd.SignalLength == 2 * len(want) and txd.SignalLength % 128 == 0
    assert (samples[:txd.SignalLength] == want.reshape(-1).view(np.uint8)).all() and (samples[txd.SignalLength:] == 0xAA).all()
    # BB11AModulateACK == BB11ATxFrameMod at 6 Mbps of the same 14 bytes (Test11AACK)
    ack = O.ack_frame(list(range(0x10, 0x16)))
    buf = np.full(cap, 0xAA, np.uint8)
    n = lib.BB11AModulateACK(C.c_uint(sr), C.byref(ra), C.c_void_p(buf.ctypes.data))
    m = MDL(None, C.c_void_p(ack.ctypes.data), 0, 10); s2 = np.full(cap, 0x55, np.uint8); t2 = TXD(C.c_void_p(s2.ctypes.data), cap, 0)
    p2 = PKT(C.pointer(m), C.pointer(t2), 0, 10, int.from_bytes(bytes(ack[10:]), "little"))
    v6 = TXV(sr, 0xB, 0)
    assert lib.BB11ATxFrameMod(C.byref(v6), C.byref(p2)) == 0
    assert n == t2.SignalLength == 2 * O.padded_samples(14, 6000, sr) and (buf[:n] == s2[:n]).all() and (buf[n:] == 0xAA).all()
    assert (buf[:n] == O.modulate(ack, 6000, sr, append_crc=False).reshape(-1).view(np.uint8)).all()
    # E_FAIL, nothing written
    samples[:] = 0xAA
    for bad in (dict(rate=0x7), dict(sr=20), dict(size=4093), dict(cap=txd.SignalLength - 1), dict(chain=len(a) + len(b) + 1)):
        vv = TXV(bad.get("sr", sr), bad.get("rate", 0xD), 0)
        txd.SampleBufferSize = bad.get("cap", cap); pkt.PacketSize = bad.get("size", bad.get("chain", len(a) + len(b)))
        assert lib.BB11ATxFrameMod(C.byref(vv), C.byref(pkt)) == E_FAIL, bad
        assert (samples == 0xAA).all(), bad
    assert lib.BB11AModulateACK(C.c_uint(20), C.byref(ra), C.c_void_p(buf.ctypes.data)) == 0
