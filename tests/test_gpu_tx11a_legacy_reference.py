"""GPU tests for the legacy 802.11a transmitter against the reference's own BB11ATxFrameMod and BB11AModulateACK, compiled from atx_*.c by
oracle/build_ref_tx11a_legacy.sh into oracle/_ref/libtx11a_legacy_ref.so (pytest -m gpu; skipped without that library): sb200_tx11a_legacy_batch
on mixed batches, and the library's own BB11ATxFrameMod / BB11AModulateACK entry points (sora_b200_legacy.h) on the same packets.  Nothing
here goes through the oracle."""
import ctypes as C, zlib
import numpy as np, pytest
import oracle_tx11a_legacy as O
from sora_b200 import api

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not O.ref_tx_available(), reason="oracle/_ref/libtx11a_legacy_ref.so not built (needs the reference tree)")]
PRE = O.preamble()


@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)


def _fcs(mpdu):
    return np.frombuffer(zlib.crc32(bytes(mpdu)).to_bytes(4, "little"), np.uint8)


def _payloads(rng, n):
    """n MPDUs + FCS of random lengths 4 .. 4096, random bytes, some all-zero / all-0xFF, some with an FCS that is not the CRC."""
    out = []
    for i in range(n):
        m = int(rng.integers(0, 4093))
        body = rng.integers(0, 256, m).astype(np.uint8) if i % 5 else np.full(m, (0, 0xFF)[i % 2], np.uint8)
        out.append(np.concatenate([body, _fcs(body) if i % 3 else rng.integers(0, 256, 4).astype(np.uint8)]))
    return out


def test_mixed_batches_equal_the_compiled_transmitter(eng):
    """Every rate at 40 and 44 Msps, about 3000 frames in all, lengths 0 .. 4092 (+ FCS): sb200_tx11a_legacy_batch equals the compiled
    BB11ATxFrameMod sample for sample, padding included, with the FCS appended by the device or sent as it is, from host and device pointers."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(2024)
    dev = torch.device("cuda", 0)
    total = 0
    for j, (kbps, sr) in enumerate([(k, s) for k in O.RATES for s in (40, 44)]):
        psdus = _payloads(rng, 188)
        want = [O.ref_modulate(p, kbps, sr) for p in psdus]
        fcs_in = j % 2 == 1
        pay = psdus if fcs_in else [p[:-4] for p in psdus]
        if not fcs_in:                                                  # the device appends the CRC: those frames carry it
            want = [O.ref_modulate(np.concatenate([p, _fcs(p)]), kbps, sr) for p in pay]
        if j % 4 < 2:
            out, ns = eng.tx11a_legacy_batch(pay, kbps, PRE, sample_rate_mhz=sr, fcs_in_payload=fcs_in)
        else:
            lens = np.array([len(p) for p in pay], np.uint32); offs = np.concatenate([[0], np.cumsum(lens[:-1])]).astype(np.uint64)
            stride = api.Engine.tx11a_legacy_nsamples(4096, kbps, sr)
            d_pay = torch.from_numpy(np.concatenate(pay)).to(dev); d_off = torch.from_numpy(offs.view(np.int64)).to(dev)
            d_len = torch.from_numpy(lens.view(np.int32)).to(dev); d_pre = torch.from_numpy(PRE.copy()).to(dev)
            d_out = torch.full((len(pay), stride, 2), 99, dtype=torch.int8, device=dev); d_ns = torch.zeros(len(pay), dtype=torch.int32, device=dev)
            eng.tx11a_legacy_raw(d_pay.data_ptr(), int(lens.sum()), d_off.data_ptr(), d_len.data_ptr(), len(pay), kbps, sr,
                                 api.Engine.TX11A_LEGACY_FCS_IN_PAYLOAD if fcs_in else 0, d_pre.data_ptr(), d_out.data_ptr(), stride, d_ns.data_ptr())
            torch.cuda.synchronize()
            out, ns = d_out.cpu().numpy(), d_ns.cpu().numpy()
        for i, w in enumerate(want):
            assert ns[i] == len(w), (kbps, sr, i, len(pay[i]), ns[i], len(w))
            bad = np.flatnonzero((out[i, :ns[i]] != w).any(axis=1))
            assert bad.size == 0, (kbps, sr, i, len(pay[i]), bad[:8])
            assert (out[i, ns[i]:] == 0).all()
        total += len(pay)
    assert total >= 3000


# ---- the library's legacy entry points (sora_b200_legacy.h) against the compiled ones ---------------------------------------------------
class TXV(C.Structure):
    _fields_ = [("SampleRate", C.c_uint), ("ti_uiDataRate", C.c_uint), ("ti_uiBufferLength", C.c_uint)]
class TXD(C.Structure):
    _fields_ = [("pSampleBuffer", C.c_void_p), ("SampleBufferSize", C.c_uint32), ("SignalLength", C.c_uint32)]
class PKT(C.Structure):
    _fields_ = [("pMdl", C.POINTER(O.MDL)), ("pTxDesc", C.POINTER(TXD)), ("fStatus", C.c_int32), ("PacketSize", C.c_uint32), ("Reserved1", C.c_uint32),
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
def test_shim_entry_points_equal_the_compiled_ones(sr):
    """The same MDL chains (non-zero ByteOffsets, a zero-length MDL) and FCS through the library's BB11ATxFrameMod and the compiled one, on
    one context each across rates: the same buffer, the same SignalLength, and the bytes past the signal left as they were.  Then
    BB11AModulateACK of both for several receiver addresses."""
    lib = _lib(); rng = np.random.default_rng(sr)
    pre = PRE.copy(); lib.BB11ATxSetPreamble(C.c_void_p(pre.ctypes.data))
    v = TXV(0, 0, 0); lib.BB11ATxContextInit(C.byref(v), C.c_uint(sr))
    ctx = O.RefContext()
    cap = 2 * O.padded_samples(4096, 6000, sr) + 256
    for i in range(40):
        kbps = O.RATES[i % 8]
        m = int(rng.integers(0, 4093)) if i % 4 else int(rng.integers(0, 65))
        mpdu = rng.integers(0, 256, m).astype(np.uint8); fcs = int(rng.integers(0, 2 ** 32))
        a, b = sorted(rng.integers(0, m + 1, 2))
        parts = ([mpdu], [mpdu[:a], mpdu[a:]], [mpdu[:a], mpdu[:0], mpdu[a:]], [mpdu[:a], mpdu[a:b], mpdu[:0], mpdu[b:]])[i % 4]
        assert sum(p.size for p in parts) == m
        offs = [1 + 7 * k for k in range(len(parts))]
        mdls = [O.MDL(None, C.c_void_p(p.ctypes.data - o if p.size else 0x1000), o, p.size) for p, o in zip(parts, offs)]
        for x, y in zip(mdls, mdls[1:]): x.Next = C.pointer(y)
        mine = np.full(cap, 0xA5, np.uint8); txd = TXD(C.c_void_p(mine.ctypes.data), cap, 0)
        pkt = PKT(C.pointer(mdls[0]), C.pointer(txd), 0, m, fcs)
        v.ti_uiDataRate = O.CODE[kbps]
        assert lib.BB11ATxFrameMod(C.byref(v), C.byref(pkt)) == 0
        hr, ref, sl = O.ref_frame_mod_raw(parts, fcs, O.CODE[kbps], sr, ctx=ctx, offsets=offs, out=np.full(cap, 0xA5, np.uint8))
        assert hr == 0 and txd.SignalLength == sl, (i, kbps, m, txd.SignalLength, sl)
        assert (mine == ref).all(), (i, kbps, m, np.flatnonzero(mine != ref)[:8])
        assert (mine[sl:] == 0xA5).all()
    for ra in ([0] * 6, [0xFF] * 6, list(rng.integers(0, 256, 6)), list(rng.integers(0, 256, 6))):
        buf = np.full(cap, 0xA5, np.uint8)
        n = lib.BB11AModulateACK(C.c_uint(sr), C.byref(MAC((C.c_uint8 * 6)(*ra))), C.c_void_p(buf.ctypes.data))
        rn, rbuf = O.ref_ack(np.array(ra, np.uint8), sr)
        assert n == rn and (buf[:n] == rbuf[:n]).all() and (buf[n:] == 0xA5).all(), ra
