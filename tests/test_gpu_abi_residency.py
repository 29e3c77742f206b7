"""Residency of the C ABI's pointer arguments (pytest -m gpu).  include/sora_b200.h promises that sample, table and result pointers may each
live in host or device memory, detected per pointer.  Every entry point that takes pointers runs one small seeded batch all on the host, all
on the device, with each argument alone moved to the device and, where the header allows it, with each argument alone moved back to the
host.  Every argument's bytes after the call (results, sample counts, the untouched parts of the outputs, the inputs) must equal those of
the all-host run."""
import ctypes as C
import numpy as np, pytest
import torch
from sora_b200 import api, synth

pytestmark = pytest.mark.gpu
V, U32, U64 = C.c_void_p, C.c_uint32, C.c_uint64
FILL = 0xA5                                            # outputs start as this pattern on both sides: bytes a call must not write stay so
BAD_OFF = 2 ** 64 - 8                                  # off + len of a non-empty slot wraps past zero

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

def _fill(nbytes):
    return np.full(nbytes, FILL, np.uint8)

def _run(call, args, dev=(), shift=None):
    """call(p), p[name] = address of args[name]: the numpy array itself, or a device copy for names in `dev` (shift[name] bytes past an
    aligned address).  Returns the bytes of every argument after the call."""
    ptr, keep = {}, {}
    for k, a in args.items():
        if a is None:
            ptr[k] = 0; continue
        a = np.ascontiguousarray(a).copy(); b = a.reshape(-1).view(np.uint8)
        if k in dev:
            o = (shift or {}).get(k, 0)
            t = torch.zeros(b.size + o, dtype=torch.uint8, device="cuda"); t[o:] = torch.from_numpy(b).cuda()
            ptr[k] = t.data_ptr() + o; keep[k] = (t, o)
        else:
            ptr[k] = b.ctypes.data; keep[k] = (b, None)
    torch.cuda.synchronize()
    call(ptr)
    torch.cuda.synchronize()
    return {k: (x if o is None else x[o:].cpu().numpy()) for k, (x, o) in keep.items()}

def _matrix(call, args, groups, extra=()):
    """All host, all device, each group alone on the device, each group alone back on the host, then `extra` (dev, shift) cases."""
    ref = _run(call, args)
    names = [n for g in groups for n in g]
    cases, seen = [], set()
    for dev in [names] + [list(g) for g in groups] + [[n for n in names if n not in g] for g in groups]:
        if frozenset(dev) not in seen:
            seen.add(frozenset(dev)); cases.append((dev, None))
    for dev, shift in cases + list(extra):
        got = _run(call, args, dev, shift)
        for k in ref:
            assert np.array_equal(got[k], ref[k]), (sorted(dev), shift, k)
    return ref

def _each(*names):
    return [(n,) for n in names]

def _slots(F, slot):
    return np.arange(F, dtype=np.uint64) * slot, np.full(F, slot, np.uint32)

def _status(raw, dtype):
    return raw.view(dtype)["status"]

# ---- receive ------------------------------------------------------------------------------------------------------------------

def _frames_11a():
    iq, _ = synth.make_frames(4, psdu_len=200, rate_kbps=24000, snr_db=28, seed0=0xAB10)
    F, slot, _ = iq.shape
    return (iq, F, slot) + _slots(F, slot)

def _frames_11a_ex(rate):
    if rate == 20:                                     # even samples of a 40 Msps capture: what TDownSample2 hands on
        iq40, _ = synth.make_frames(3, psdu_len=150, rate_kbps=12000, snr_db=30, seed0=0xAB20)
        iq = np.ascontiguousarray(iq40[:, ::2]); F, slot, _ = iq.shape
        return (iq, F, slot) + _slots(F, slot)
    from test_cpu_oracle import _capture_44
    caps = [_capture_44(r, 120 + 10 * i, 70 + i, snr_db=30) for i, r in enumerate((6000, 36000))]
    slot = max(len(c[0]) for c in caps); F = len(caps)
    flat = np.zeros((F, slot, 2), np.int16); ln = np.zeros(F, np.uint32); off = np.arange(F, dtype=np.uint64) * slot
    for i, (c, _) in enumerate(caps): flat[i, :len(c)] = c; ln[i] = len(c)
    return flat, F, slot, off, ln

def test_rx11a_batch(eng):
    iq, F, slot, off, ln = _frames_11a()
    args = dict(iq=iq, off=off, len=ln, out=_fill(F * 256), res=_fill(F * api.RESULT_DTYPE.itemsize))
    ref = _matrix(lambda p: eng.rx11a_raw(p["iq"], F * slot, p["off"], p["len"], F, p["out"], 256, p["res"]), args, _each(*args))
    assert (_status(ref["res"], api.RESULT_DTYPE) == api.FRAME_OK).any()

@pytest.mark.parametrize("rate", [20, 44])
def test_rx11a_batch_ex(eng, rate):
    flat, F, slot, off, ln = _frames_11a_ex(rate)
    args = dict(iq=flat, off=off, len=ln, out=_fill(F * 256), res=_fill(F * api.RESULT_DTYPE.itemsize))
    call = lambda p: eng._check(eng._lib.sb200_rx11a_batch_ex(eng._h, p["iq"], F * slot, p["off"], p["len"], F, rate, p["out"], 256, p["res"], None), "sb200_rx11a_batch_ex")
    ref = _matrix(call, args, _each(*args))
    assert (_status(ref["res"], api.RESULT_DTYPE) == api.FRAME_OK).any()

def _frames_11b():
    iq, _ = synth.make_frames_11b(2, psdu_len=100, rate_kbps=2000, snr_db=35, gain=0.15, seed0=0xAB30)
    F, slot, _ = iq.shape
    return iq, F, slot

def test_rx11b_batch(eng):
    iq, F, slot = _frames_11b(); off, ln = _slots(F, slot)
    args = dict(iq=iq, off=off, len=ln, out=_fill(F * 256), res=_fill(F * api.RESULT11B_DTYPE.itemsize))
    ref = _matrix(lambda p: eng.rx11b_raw(p["iq"], F * slot, p["off"], p["len"], F, p["out"], 256, p["res"]), args, _each(*args))
    assert (_status(ref["res"], api.RESULT11B_DTYPE) == api.FRAME_OK).any()

def test_rx11b_streams(eng):
    iq, F, slot = _frames_11b(); M = 2
    off = np.array([0], np.uint64); ln = np.array([F * slot], np.uint32)            # one capture holding both frames
    args = dict(iq=iq, off=off, len=ln, out=_fill(M * 256), res=_fill(M * api.RESULT11B_DTYPE.itemsize), cnt=_fill(4))
    call = lambda p: eng._check(eng._lib.sb200_rx11b_streams(eng._h, V(p["iq"]), U64(F * slot), V(p["off"]), V(p["len"]), U32(1), U32(M), V(p["out"]), U32(256),
                                                             V(p["res"]), V(p["cnt"]), V(0)), "sb200_rx11b_streams")
    ref = _matrix(call, args, _each(*args))
    assert ref["cnt"].view(np.uint32)[0] >= 1 and (_status(ref["res"], api.RESULT11B_DTYPE) == api.FRAME_OK).any()

def _frames_11n():
    iq0, iq1, _ = synth.make_frames_11n(2, psdu_len=120, mcs=9, snr_db=28, lead=400, trail=200, seed0=0xAB40)
    F, slot, _ = iq0.shape
    return (iq0, iq1, F, slot) + _slots(F, slot)

def test_rx11n_batch(eng):
    iq0, iq1, F, slot, off, ln = _frames_11n()
    args = dict(iq0=iq0, iq1=iq1, off=off, len=ln, out=_fill(F * 256), res=_fill(F * api.RESULT11N_DTYPE.itemsize))
    call = lambda p: eng.rx11n_raw(p["iq0"], p["iq1"], F * slot, p["off"], p["len"], F, p["out"], 256, p["res"])
    ref = _matrix(call, args, [("iq0", "iq1")] + _each("off", "len", "out", "res"))
    assert (_status(ref["res"], api.RESULT11N_DTYPE) == api.FRAME_OK).any()

def test_rx11a_streams(eng):
    """Stream mode takes its tables and returns its results in host memory; only the capture may live on either side."""
    iq, _ = synth.make_frames(4, psdu_len=100, rate_kbps=36000, snr_db=30, seed0=0xAB50)
    F, slot, _ = iq.shape; S, M = 2, 3
    off = np.arange(S, dtype=np.uint64) * (2 * slot); ln = np.full(S, 2 * slot, np.uint32)
    args = dict(iq=iq, off=off, len=ln, out=_fill(S * M * 256), res=_fill(S * M * api.RESULT_DTYPE.itemsize), sidx=_fill(S * M * 4), cnt=_fill(S * 4))
    call = lambda p: eng._check(eng._lib.sb200_rx11a_streams(eng._h, V(p["iq"]), U64(F * slot), V(p["off"]), V(p["len"]), U32(S), U32(M), V(p["out"]), U32(256),
                                                             V(p["res"]), V(p["sidx"]), V(p["cnt"]), V(0)), "sb200_rx11a_streams")
    ref = _matrix(call, args, [("iq",)])
    assert (ref["cnt"].view(np.uint32) >= 1).all()

def _fir_input():
    return np.random.default_rng(0xAB60).integers(-3000, 3000, (1001, 2)).astype(np.int16)

def test_fir_decimate2(eng):
    x = _fir_input()
    args = dict(iq=x, out=_fill(501 * 4 + 16))                                     # 16 bytes past the result must stay untouched
    _matrix(lambda p: eng.fir_decimate2_raw(p["iq"], 1001, 0, 0, p["out"]), args, _each(*args))

def _rx_blocks(n):
    return np.random.default_rng(0xAB70 + n).integers(0, 256, n * 128).astype(np.uint8)

def test_rxblocks_unpack(eng):
    args = dict(blocks=_rx_blocks(9), out=_fill(9 * 112))
    call = lambda p: eng._check(eng._lib.sb200_rxblocks_unpack(eng._h, V(p["blocks"]), U64(9), U32(2), V(p["out"]), V(0)), "sb200_rxblocks_unpack")
    _matrix(call, args, _each(*args))

def test_rxblocks_desc(eng):
    args = dict(blocks=_rx_blocks(11), vbits=_fill(11 * 4), stamps=_fill(11 * 4))
    call = lambda p: eng._check(eng._lib.sb200_rxblocks_desc(eng._h, V(p["blocks"]), U64(11), V(p["vbits"]), V(p["stamps"]), V(0)), "sb200_rxblocks_desc")
    _matrix(call, args, _each(*args))

# ---- transmit -----------------------------------------------------------------------------------------------------------------

def _payloads(lens, seed):
    r = np.random.default_rng(seed); ln = np.array(lens, np.uint32)
    off = np.concatenate([[0], np.cumsum(ln[:-1])]).astype(np.uint64)
    return r.integers(0, 256, int(ln.sum())).astype(np.uint8), off, ln

def test_tx11a_batch(eng):
    pay, off, ln = _payloads([40, 300, 77], 0xAB80); F = 3
    stride = 20 + 640 + 160 * (2 + -(-(300 + 7) * 8 // 144)) + 32
    args = dict(pay=pay, off=off, len=ln, seeds=np.array([0x11, 0x5A, 0x7F], np.uint8), out=_fill(F * stride * 4), ns=_fill(F * 4))
    call = lambda p: eng.tx11a_raw(p["pay"], pay.size, p["off"], p["len"], p["seeds"], F, 36000, 20, 16, p["out"], stride, p["ns"])
    _matrix(call, args, _each(*args))

def test_tx11b_batch(eng):
    pay, off, ln = _payloads([30, 64], 0xAB90); F = 2
    stride = ((24 * 88 + (64 + 4) * 16 + 5) * 4 + 15) // 8 * 8
    args = dict(pay=pay, off=off, len=ln, out=_fill(F * stride * 2), ns=_fill(F * 4), fp=_fill(F * 4))
    call = lambda p: eng.tx11b_raw(p["pay"], pay.size, p["off"], p["len"], F, 5500, 1, 0, 8, p["out"], stride, p["ns"], 0, p["fp"])
    _matrix(call, args, _each(*args))

def _fir37_input(F=3, L=96, gap=16):
    chips = np.random.default_rng(0xABA0).integers(-128, 128, (F * (L + gap), 2)).astype(np.int8)
    return chips, np.arange(F, dtype=np.uint64) * (L + gap), np.array([L, 0, L - 24], np.uint32)

def test_tx11b_fir37(eng):
    """Frames with gaps between them: the bytes outside the frames stay as they were, on either side."""
    F, L, gap = 3, 96, 16
    chips, off, ln = _fir37_input(F, L, gap)
    args = dict(chips=chips, off=off, len=ln, out=_fill(chips.nbytes))
    call = lambda p: eng.tx11b_fir37_raw(p["chips"], len(chips), p["off"], p["len"], F, 1, p["out"])
    ref = _matrix(call, args, _each(*args))
    assert (ref["out"][2 * L: 2 * (L + gap)] == FILL).all()

def test_tx11b_legacy_batch(eng):
    pay, off, ln = _payloads([20, 50], 0xABB0); F = 2
    stride = (4 * (1056 + 54 * 16) + 37 + 127) // 128 * 128
    args = dict(pay=pay, off=off, len=ln, out=_fill(F * stride * 2), ns=_fill(F * 4))
    call = lambda p: eng.tx11b_legacy_raw(p["pay"], pay.size, p["off"], p["len"], F, 5500, 1, 0, 1, p["out"], stride, p["ns"])
    _matrix(call, args, _each(*args))

def test_tx11a_legacy_batch(eng):
    """The preamble is used in place when it is device memory aligned to 4 bytes, else copied: host, aligned and misaligned by 2 bytes."""
    import oracle_tx11a_legacy
    pay, off, ln = _payloads([60, 25], 0xABC0); F = 2
    stride = api.Engine.tx11a_legacy_nsamples(64, 24000, 44)
    args = dict(pay=pay, off=off, len=ln, pre=oracle_tx11a_legacy.preamble(), out=_fill(F * stride * 2), ns=_fill(F * 4))
    call = lambda p: eng.tx11a_legacy_raw(p["pay"], pay.size, p["off"], p["len"], F, 24000, 44, 0, p["pre"], p["out"], stride, p["ns"])
    names = list(args)
    _matrix(call, args, _each(*names), extra=[(["pre"], {"pre": 2}), (names, {"pre": 2})])

def test_tx11n_batch(eng):
    pay, off, ln = _payloads([50, 120], 0xABD0); F = 2
    stride = 10 + 1600 + 160 * (-(-((120 + 4) * 8 + 22) // 104) + 1)
    args = dict(pay=pay, off=off, len=ln, seeds=np.array([0x33, 0x44], np.uint8), out0=_fill(F * stride * 4), out1=_fill(F * stride * 4), ns=_fill(F * 4))
    call = lambda p: eng.tx11n_raw(p["pay"], pay.size, p["off"], p["len"], p["seeds"], F, 9, 10, p["out0"], p["out1"], stride, p["ns"])
    _matrix(call, args, _each("pay", "off", "len", "seeds") + [("out0", "out1"), ("ns",)])

def _viterbi_input():
    """Three rate-1/2 code blocks of a 120-byte frame, soft values in rows of `stride` bytes."""
    rng = np.random.default_rng(0xABE0); L, nb = 120, 3
    nbits = 8 * L + 16 + 6; nbits += (-nbits) % 48
    bits = rng.integers(0, 2, (nb, nbits)).astype(np.uint8); bits[:, 8 * L + 16:] = 0
    coded = synth.puncture(*synth.conv_encode(bits), (1, 2)); nsoft = coded.shape[1]; stride = (nsoft + 15) // 16 * 16
    soft = np.zeros((nb, stride), np.uint8); soft[:, :nsoft] = np.where(coded > 0, rng.integers(5, 8, coded.shape), rng.integers(0, 3, coded.shape))
    return soft, stride, nsoft, nb, L

def test_viterbi_k7(eng):
    """Device soft values aligned to 16 bytes are decoded in place, anything else is restrided first: host, aligned, misaligned by 2."""
    soft, stride, nsoft, nb, L = _viterbi_input()
    args = dict(soft=soft, out=_fill(nb * (L + 8)))
    call = lambda p: eng.viterbi_raw(p["soft"], stride, nsoft, nb, api.CR_12, L, p["out"], L + 8)
    ref = _matrix(call, args, _each(*args), extra=[(["soft"], {"soft": 2}), (["soft", "out"], {"soft": 2})])
    assert (ref["out"].reshape(nb, L + 8)[:, L + 2:] == FILL).all()

# ---- table ranges that wrap past 2^64 -----------------------------------------------------------------------------------------

def _tx11a(eng, pay, off, ln):
    out, ns = np.zeros(2 * 4000, np.int8), np.zeros(1, np.uint32)
    eng.tx11a_raw(pay.ctypes.data, pay.size, off.ctypes.data, ln.ctypes.data, 0, 1, 6000, 0, 8, out.ctypes.data, 4000, ns.ctypes.data)

def _tx11b(eng, pay, off, ln):
    out, ns = np.zeros(2 * 40000 + 16, np.int8), np.zeros(1, np.uint32); o = -out.ctypes.data % 16
    eng.tx11b_raw(pay.ctypes.data, pay.size, off.ctypes.data, ln.ctypes.data, 1, 1000, 0, 0, 8, out.ctypes.data + o, 40000, ns.ctypes.data)

def _tx11n(eng, pay, off, ln):
    o0, o1, ns = np.zeros(4 * 4000, np.int8), np.zeros(4 * 4000, np.int8), np.zeros(1, np.uint32)
    eng.tx11n_raw(pay.ctypes.data, pay.size, off.ctypes.data, ln.ctypes.data, 0, 1, 8, 0, o0.ctypes.data, o1.ctypes.data, 4000, ns.ctypes.data)

def _rx11a_streams(eng, iq, off, ln):
    eng.rx11a_streams(iq, off, ln, max_frames=1, out_stride=64)

def _rx11n_streams(eng, iq, off, ln):
    eng.rx11n_streams(iq, iq.copy(), off, ln, max_frames=1, out_stride=64)

@pytest.mark.parametrize("call", [_tx11a, _tx11b, _tx11n, _rx11a_streams, _rx11n_streams], ids=lambda f: f.__name__.strip("_"))
def test_range_wrapping_past_2_64_is_rejected(eng, call):
    """A slot at offset 2^64 - 8 with a non-zero length would end past zero: refused with SB200_E_INVALID, host-resident data."""
    data = np.zeros(256, np.uint8) if call in (_tx11a, _tx11b, _tx11n) else np.zeros((256, 2), np.int16)
    with pytest.raises(api.Sb200Error, match=r"failed \(-1\)"):
        call(eng, data, np.array([BAD_OFF], np.uint64), np.array([16], np.uint32))

# ---- launch counts and timing accessors ----------------------------------------------------------------------------------------

def _bk_rx11a(e, rate=40):
    iq, F, slot, off, ln = _frames_11a() if rate == 40 else _frames_11a_ex(rate)
    return lambda: e.rx11a_batch(iq.reshape(-1, 2), off, ln, out_stride=256, sample_rate_mhz=rate)
def _bk_rx11a_taps(e):
    iq, F, slot, off, ln = _frames_11a()
    return lambda: e.rx11a_taps(iq.reshape(-1, 2), off, ln, 40)
def _bk_rx11n(e, mcs_limit=None, taps=False):
    if mcs_limit: e.set_option("ht_mcs_limit", mcs_limit)
    iq0, iq1, F, slot, off, ln = _frames_11n()
    if taps: return lambda: e.rx11n_taps(iq0.reshape(-1, 2), iq1.reshape(-1, 2), off, ln, max_sym=40)
    return lambda: e.rx11n_batch(iq0.reshape(-1, 2), iq1.reshape(-1, 2), off, ln, out_stride=256)
def _bk_rx11b(e):
    iq, F, slot = _frames_11b(); off, ln = _slots(F, slot)
    return lambda: e.rx11b_batch(iq.reshape(-1, 2), off, ln, out_stride=256)
def _bk_tx11b_fir37(e):
    chips, off, ln = _fir37_input(); out = np.zeros_like(chips)
    return lambda: e.tx11b_fir37_raw(chips.ctypes.data, len(chips), off.ctypes.data, ln.ctypes.data, len(off), 1, out.ctypes.data)
def _bk_viterbi(e):
    soft, stride, nsoft, nb, L = _viterbi_input(); out = np.zeros(nb * (L + 8), np.uint8)
    return lambda: e.viterbi_raw(soft.ctypes.data, stride, nsoft, nb, api.CR_12, L, out.ctypes.data, L + 8)
def _bk_pay(seed, lens):
    pay, off, ln = _payloads(lens, seed)
    return [pay[int(o): int(o) + int(n)] for o, n in zip(off, ln)]
def _bk_tx11a_legacy(e, fcs=False):
    import oracle_tx11a_legacy
    p = _bk_pay(0xABC0, [60, 25])
    return lambda: e.tx11a_legacy_batch(p, 24000, oracle_tx11a_legacy.preamble(), sample_rate_mhz=44, fcs_in_payload=fcs)

BOOKKEEPING = {                                        # entry: (setup, launches of the first call, of the second, last_kernel_ms() >= 0, last_kernel_times() works)
    "rx11a_batch":        (_bk_rx11a, 8, 8, True, True),
    "rx11a_batch_ex_20":  (lambda e: _bk_rx11a(e, 20), 8, 8, True, True),
    "rx11a_batch_ex_44":  (lambda e: _bk_rx11a(e, 44), 9, 9, True, True),
    "rx11a_taps":         (_bk_rx11a_taps, 8, 8, True, True),
    "rx11n_batch":        (_bk_rx11n, 7, 7, True, True),
    "rx11n_batch_mcs15":  (lambda e: _bk_rx11n(e, 15), 8, 8, True, True),
    "rx11n_taps":         (lambda e: _bk_rx11n(e, taps=True), 7, 7, True, True),
    "rx11b_batch":        (_bk_rx11b, 1, 1, True, False),
    "fir_decimate2":      (lambda e: lambda: e.fir_decimate2(_fir_input()), 1, 1, True, False),
    "rxblocks_unpack":    (lambda e: lambda: e.rxblocks_unpack(_rx_blocks(9), 2), 1, 1, False, False),
    "rxblocks_desc":      (lambda e: lambda: e.rxblocks_desc(_rx_blocks(11)), 1, 1, False, False),
    "tx11b_fir37":        (_bk_tx11b_fir37, 1, 1, True, False),
    "viterbi_k7":         (_bk_viterbi, 1, 1, True, False),
    "tx11a":              (lambda e: lambda: e.tx11a_batch(_bk_pay(0xAB80, [40, 300, 77]), 36000, seeds=[0x11, 0x5A, 0x7F], lead=20, sample_bits=16), 3, 2, True, False),
    "tx11n":              (lambda e: lambda: e.tx11n_batch(_bk_pay(0xABD0, [50, 120]), 9, seeds=[0x33, 0x44], lead=10), 3, 2, True, False),
    "tx11b":              (lambda e: lambda: e.tx11b_batch(_bk_pay(0xAB90, [30, 64]), 5500, init_phase=1), 3, 3, True, False),
    "tx11b_legacy":       (lambda e: lambda: e.tx11b_legacy_batch(_bk_pay(0xABB0, [20, 50]), 5500, short_preamble=True), 3, 3, True, False),
    "tx11b_legacy_fcs":   (lambda e: lambda: e.tx11b_legacy_batch(_bk_pay(0xABB0, [20, 50]), 5500, short_preamble=True, fcs_in_payload=True), 2, 2, True, False),
    "tx11a_legacy":       (_bk_tx11a_legacy, 3, 2, True, False),
    "tx11a_legacy_fcs":   (lambda e: _bk_tx11a_legacy(e, True), 2, 1, True, False),
}

@pytest.mark.parametrize("name", list(BOOKKEEPING))
def test_launch_count_and_timing_accessors(name):
    """sb200_launch_count delta of a first and a second call on a fresh default engine, and whether sb200_last_kernel_ms / _times answer
    after it: the first transmit call on a handle also counts k_tx11a_preamble; the RX_BLOCK calls record no events."""
    setup, first, second, ms_ok, times_ok = BOOKKEEPING[name]
    e = api.Engine(0)
    try:
        call = setup(e)
        n0 = e.launches; call(); n1 = e.launches; call(); n2 = e.launches
        assert (n1 - n0, n2 - n1) == (first, second)
        assert (e.last_kernel_ms() >= 0) == ms_ok
        try:
            e.last_kernel_times(); times = True
        except api.Sb200Error:
            times = False
        assert times == times_ok
    finally:
        e.close()
