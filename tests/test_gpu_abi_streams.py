"""When the C ABI touches memory (pytest -m gpu).  include/sora_b200.h: a call returns once it no longer needs any host buffer of the
caller; with device buffers and host-resident tables it does not wait for its stream; calls on one handle run in the order they were
made, whatever streams they are given.  test_gpu_abi_residency.py checks where each pointer may live, synchronising around every call;
this file checks when the library reads and writes.

Method: before a call, a bounded torch.cuda._sleep (GATE_MS) holds the caller's stream, so everything the call queues is still pending
when Python gets control back.  Whatever the test then does to host memory happens before the device could read it, and an event
recorded behind the gate tells whether the call waited for the stream.  Each case runs once; none repeats anything to catch a race.
Outputs start as a fill pattern, so bytes written late or not at all show up.  References: the oracle or the numpy models where they exist, else the synchronous
all-host run of the same call (which test_gpu_abi_residency.py ties to the oracle)."""
import contextlib, ctypes as C, threading
import numpy as np, pytest
import torch
from sora_b200 import api, synth
import oracle_py, oracle_tx11a_legacy, wideband_inputs
import test_gpu_abi_residency as R

pytestmark = pytest.mark.gpu
V, U32, U64 = C.c_void_p, C.c_uint32, C.c_uint64
GATE_MS = 150                                          # every gate is bounded: at most this long on the device
FILL = R.FILL
TABLES = ("off", "len")                                # slot / payload tables: host-resident unless a case says otherwise

# ---- streams, the gate, page-locked memory --------------------------------------------------------------------------------------

_rt = None
def _cudart():
    global _rt
    if _rt is None:
        api.load_library()                            # the runtime the library links (and torch shares)
        _rt = C.CDLL("libcudart.so.12")
        _rt.cudaStreamCreateWithFlags.argtypes = [C.POINTER(C.c_void_p), C.c_uint]
        _rt.cudaStreamDestroy.argtypes = [C.c_void_p]
        lib = api.load_library()
        lib.sb200_host_alloc.argtypes = [C.c_size_t]; lib.sb200_host_alloc.restype = C.c_void_p
        lib.sb200_host_free.argtypes = [C.c_void_p]; lib.sb200_host_free.restype = None
    return _rt

@contextlib.contextmanager
def caller_stream(kind):
    """(torch stream, handle passed to the library): the legacy default stream, cudaStreamPerThread, or a stream created non-blocking.
    Synchronised, and destroyed if created here, when the block ends."""
    raw = None
    if kind == "legacy":
        s = torch.cuda.default_stream(); handle = 0
        assert s.cuda_stream == 0
    elif kind == "per_thread":
        s = torch.cuda.ExternalStream(2); handle = 2    # cudaStreamPerThread
    else:
        p = C.c_void_p(); assert _cudart().cudaStreamCreateWithFlags(C.byref(p), 1) == 0   # cudaStreamNonBlocking
        raw = p.value; s = torch.cuda.ExternalStream(raw); handle = raw
    try:
        yield s, handle
    finally:
        s.synchronize()
        if raw: _cudart().cudaStreamDestroy(raw)

KINDS = ["legacy", "per_thread", "nonblocking"]

_cycles = None
def gate(s):
    """Hold stream s for about GATE_MS: a spin kernel whose clock count is calibrated once with CUDA events."""
    global _cycles
    if _cycles is None:
        torch.cuda._sleep(1_000_000); torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); torch.cuda._sleep(20_000_000); b.record(); b.synchronize()
        _cycles = int(20_000_000 * (GATE_MS * 0.9) / a.elapsed_time(b))
    with torch.cuda.stream(s):
        torch.cuda._sleep(_cycles)

@contextlib.contextmanager
def pinned_pool():
    """alloc(nbytes) -> numpy uint8 view of sb200_host_alloc memory; everything freed when the block ends (after a device synchronise)."""
    ptrs = []
    def alloc(n):
        p = api.load_library().sb200_host_alloc(max(n, 1)); assert p
        ptrs.append(p)
        return np.ctypeslib.as_array((C.c_uint8 * n).from_address(p))
    _cudart()
    try:
        yield alloc
    finally:
        torch.cuda.synchronize()
        for p in ptrs: api.load_library().sb200_host_free(p)

# ---- buffers --------------------------------------------------------------------------------------------------------------------

def _bytes(a):
    return np.ascontiguousarray(a).reshape(-1).view(np.uint8).copy()

def _place(args, kinds, alloc=None):
    """p[name] = address of a buffer holding args[name], as kinds[name] says: "host" (pageable numpy), "dev" (device tensor), "pinned"."""
    p, bufs = {}, {}
    for k, a in args.items():
        b = _bytes(a); kind = kinds.get(k, "host")
        if kind == "dev":
            t = torch.from_numpy(b).cuda(); p[k] = t.data_ptr()
        elif kind == "pinned":
            t = alloc(b.size); t[:] = b; p[k] = t.ctypes.data
        else:
            t = b; p[k] = b.ctypes.data
        bufs[k] = t
    return p, bufs

def _host(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else np.array(x, copy=True)

def _masks(ent, ref):
    """A receive row holds the delivered frame's bytes and, past its length, whatever the handle's workspace held from earlier calls:
    only the bytes of frames decoded OK count."""
    dt = ent.dtypes.get("res")
    if dt is None or "out" not in ent.outs:
        return {}
    r = ref["res"].view(dt); row = ref["out"].size // len(r)
    m = np.zeros((len(r), row), bool)
    for i in np.flatnonzero(r["status"] == api.FRAME_OK):
        m[i, :min(int(r["length"][i]), row)] = True
    return {"out": m.reshape(-1)}

def _check_outs(what, ent, got, ref):
    masks = _masks(ent, ref)
    for k in sorted(ent.outs, key=lambda k: k not in ent.dtypes):      # results first: a diverging slot and field
        g, w = got[k], ref[k]
        if k in masks: g, w = g[masks[k]], w[masks[k]]
        _same(f"{what} {k}", g, w, ent.dtypes.get(k))

def _same(what, got, want, dtype=None):
    """Equal bytes; otherwise the first diverging slot and field (result buffers) or byte offset."""
    if np.array_equal(got, want):
        return
    if dtype is not None and got.size % dtype.itemsize == 0:
        g, w = got.view(dtype), want.view(dtype)
        for i in range(len(g)):
            for f in dtype.names:
                if g[f][i] != w[f][i]:
                    pytest.fail(f"{what}: slot {i} field {f}: got {g[f][i]!r}, want {w[f][i]!r}")
    i = int(np.flatnonzero(got != want)[0])
    pytest.fail(f"{what}: first diverging byte {i} of {got.size}: got {got[i]}, want {want[i]}")

# ---- the entry points -----------------------------------------------------------------------------------------------------------
# Entry(args, outs, call(p, stream), roll, host, opts, dtypes): `roll` names every input a caller could hand over in host memory and the
# byte shift (np.roll) that turns it into another valid input; `host` the arguments stream mode takes in host memory only.

class Entry:
    def __init__(self, args, outs, call, roll, host=(), opts=None, dtypes=None):
        self.args, self.outs, self.call, self.roll, self.host, self.opts, self.dtypes = args, outs, call, roll, set(host), opts or {}, dtypes or {}

def _rx11a(e):
    iq, F, slot, off, ln = R._frames_11a()
    args = dict(iq=iq, off=off, len=ln, out=R._fill(F * 256), res=R._fill(F * api.RESULT_DTYPE.itemsize))
    return Entry(args, ("out", "res"), lambda p, s: e.rx11a_raw(p["iq"], F * slot, p["off"], p["len"], F, p["out"], 256, p["res"], s),
                 {"iq": iq.nbytes // F}, dtypes={"res": api.RESULT_DTYPE})

def _rx11a_ex(rate):
    def make(e):
        flat, F, slot, off, ln = R._frames_11a_ex(rate)
        args = dict(iq=flat, off=off, len=ln, out=R._fill(F * 256), res=R._fill(F * api.RESULT_DTYPE.itemsize))
        call = lambda p, s: e._check(e._lib.sb200_rx11a_batch_ex(e._h, p["iq"], F * slot, p["off"], p["len"], F, rate, p["out"], 256, p["res"], s), "sb200_rx11a_batch_ex")
        return Entry(args, ("out", "res"), call, {"iq": flat.nbytes // F}, dtypes={"res": api.RESULT_DTYPE})
    return make

def _rx11b(e):
    iq, F, slot = R._frames_11b(); off, ln = R._slots(F, slot)
    args = dict(iq=iq, off=off, len=ln, out=R._fill(F * 256), res=R._fill(F * api.RESULT11B_DTYPE.itemsize))
    return Entry(args, ("out", "res"), lambda p, s: e.rx11b_raw(p["iq"], F * slot, p["off"], p["len"], F, p["out"], 256, p["res"], s),
                 {"iq": iq.nbytes // F}, dtypes={"res": api.RESULT11B_DTYPE})

def _rx11b_streams(e):
    iq, F, slot = R._frames_11b(); M = 2
    args = dict(iq=iq, off=np.array([0], np.uint64), len=np.array([F * slot], np.uint32), out=R._fill(M * 256),
                res=R._fill(M * api.RESULT11B_DTYPE.itemsize), cnt=R._fill(4))
    call = lambda p, s: e._check(e._lib.sb200_rx11b_streams(e._h, V(p["iq"]), U64(F * slot), V(p["off"]), V(p["len"]), U32(1), U32(M), V(p["out"]), U32(256),
                                                            V(p["res"]), V(p["cnt"]), V(s)), "sb200_rx11b_streams")
    return Entry(args, ("out", "res", "cnt"), call, {"iq": iq.nbytes // F}, dtypes={"res": api.RESULT11B_DTYPE})

def _rx11n(e):
    iq0, iq1, F, slot, off, ln = R._frames_11n()
    args = dict(iq0=iq0, iq1=iq1, off=off, len=ln, out=R._fill(F * 256), res=R._fill(F * api.RESULT11N_DTYPE.itemsize))
    call = lambda p, s: e.rx11n_raw(p["iq0"], p["iq1"], F * slot, p["off"], p["len"], F, p["out"], 256, p["res"], s)
    return Entry(args, ("out", "res"), call, {"iq0": iq0.nbytes // F, "iq1": iq1.nbytes // F}, dtypes={"res": api.RESULT11N_DTYPE})

def _rx11a_streams(e):
    iq, _ = synth.make_frames(4, psdu_len=100, rate_kbps=36000, snr_db=30, seed0=0xAB50)
    F, slot, _ = iq.shape; S, M = 2, 3
    args = dict(iq=iq, off=np.arange(S, dtype=np.uint64) * (2 * slot), len=np.full(S, 2 * slot, np.uint32), out=R._fill(S * M * 256),
                res=R._fill(S * M * api.RESULT_DTYPE.itemsize), sidx=R._fill(S * M * 4), cnt=R._fill(S * 4))
    call = lambda p, s: e._check(e._lib.sb200_rx11a_streams(e._h, V(p["iq"]), U64(F * slot), V(p["off"]), V(p["len"]), U32(S), U32(M), V(p["out"]), U32(256),
                                                            V(p["res"]), V(p["sidx"]), V(p["cnt"]), V(s)), "sb200_rx11a_streams")
    return Entry(args, ("out", "res", "sidx", "cnt"), call, {"iq": iq.nbytes // F}, host=("off", "len", "out", "res", "sidx", "cnt"), dtypes={"res": api.RESULT_DTYPE})

def _rx11n_streams(e):
    iq0, iq1, F, slot, _, _ = R._frames_11n(); M = 2
    args = dict(iq0=iq0, iq1=iq1, off=np.array([0], np.uint64), len=np.array([F * slot], np.uint32), out=R._fill(M * 256),
                res=R._fill(M * api.RESULT11N_DTYPE.itemsize), sidx=R._fill(M * 4), cnt=R._fill(4))
    call = lambda p, s: e._check(e._lib.sb200_rx11n_streams(e._h, V(p["iq0"]), V(p["iq1"]), U64(F * slot), V(p["off"]), V(p["len"]), U32(1), U32(M), V(p["out"]),
                                                            U32(256), V(p["res"]), V(p["sidx"]), V(p["cnt"]), V(s)), "sb200_rx11n_streams")
    return Entry(args, ("out", "res", "sidx", "cnt"), call, {"iq0": iq0.nbytes // F, "iq1": iq1.nbytes // F},
                 host=("off", "len", "out", "res", "sidx", "cnt"), dtypes={"res": api.RESULT11N_DTYPE})

def _fir(e):
    args = dict(iq=R._fir_input(), out=R._fill(501 * 4 + 16))
    return Entry(args, ("out",), lambda p, s: e.fir_decimate2_raw(p["iq"], 1001, 0, 0, p["out"], s), {"iq": 4})

CH_N, CH_D, CH_STRIDE = 5000, 4, 1252
CH_CHANNELS = [(0, 0), (api.phase_inc(-20e6, 160e6), 0), (2 ** 30, 12345)]
CH_TAPS = wideband_inputs.lowpass(63, 0.1)
def _channelize_input():
    return np.random.default_rng(0xAB61).integers(-32768, 32768, (CH_N, 2)).astype(np.int16)

def _channelize(e):
    args = dict(iq=_channelize_input(), out=R._fill(len(CH_CHANNELS) * CH_STRIDE * 4))
    return Entry(args, ("out",), lambda p, s: e.channelize_raw(p["iq"], CH_N, CH_CHANNELS, CH_D, CH_TAPS, p["out"], CH_STRIDE, s), {"iq": 4})

def _rxblocks_unpack(e):
    args = dict(blocks=R._rx_blocks(9), out=R._fill(9 * 112))
    call = lambda p, s: e._check(e._lib.sb200_rxblocks_unpack(e._h, V(p["blocks"]), U64(9), U32(2), V(p["out"]), V(s)), "sb200_rxblocks_unpack")
    return Entry(args, ("out",), call, {"blocks": 128})

def _rxblocks_desc(e):
    args = dict(blocks=R._rx_blocks(11), vbits=R._fill(11 * 4), stamps=R._fill(11 * 4))
    call = lambda p, s: e._check(e._lib.sb200_rxblocks_desc(e._h, V(p["blocks"]), U64(11), V(p["vbits"]), V(p["stamps"]), V(s)), "sb200_rxblocks_desc")
    return Entry(args, ("vbits", "stamps"), call, {"blocks": 128})

def _tx11a(e):
    pay, off, ln = R._payloads([40, 300, 77], 0xAB80); F = 3
    stride = 20 + 640 + 160 * (2 + -(-(300 + 7) * 8 // 144)) + 32
    args = dict(pay=pay, off=off, len=ln, seeds=np.array([0x11, 0x5A, 0x7F], np.uint8), out=R._fill(F * stride * 4), ns=R._fill(F * 4))
    call = lambda p, s: e.tx11a_raw(p["pay"], pay.size, p["off"], p["len"], p["seeds"], F, 36000, 20, 16, p["out"], stride, p["ns"], s)
    return Entry(args, ("out", "ns"), call, {"pay": 1, "seeds": 1})

def _tx11b(e):
    pay, off, ln = R._payloads([30, 64], 0xAB90); F = 2
    stride = ((24 * 88 + (64 + 4) * 16 + 5) * 4 + 15) // 8 * 8
    args = dict(pay=pay, off=off, len=ln, out=R._fill(F * stride * 2), ns=R._fill(F * 4), fp=R._fill(F * 4))
    call = lambda p, s: e.tx11b_raw(p["pay"], pay.size, p["off"], p["len"], F, 5500, 1, 0, 8, p["out"], stride, p["ns"], s, p["fp"])
    return Entry(args, ("out", "ns", "fp"), call, {"pay": 1})

def _tx11n(e):
    pay, off, ln = R._payloads([50, 120], 0xABD0); F = 2
    stride = 10 + 1600 + 160 * (-(-((120 + 4) * 8 + 22) // 104) + 1)
    args = dict(pay=pay, off=off, len=ln, seeds=np.array([0x33, 0x44], np.uint8), out0=R._fill(F * stride * 4), out1=R._fill(F * stride * 4), ns=R._fill(F * 4))
    call = lambda p, s: e.tx11n_raw(p["pay"], pay.size, p["off"], p["len"], p["seeds"], F, 9, 10, p["out0"], p["out1"], stride, p["ns"], s)
    return Entry(args, ("out0", "out1", "ns"), call, {"pay": 1, "seeds": 1})

def _fir37(e):
    chips, off, ln = R._fir37_input()
    args = dict(chips=chips, off=off, len=ln, out=R._fill(chips.nbytes))
    return Entry(args, ("out",), lambda p, s: e.tx11b_fir37_raw(p["chips"], len(chips), p["off"], p["len"], len(off), 1, p["out"], s), {"chips": 2})

def _tx11b_legacy(e):
    pay, off, ln = R._payloads([20, 50], 0xABB0); F = 2
    stride = (4 * (1056 + 54 * 16) + 37 + 127) // 128 * 128
    args = dict(pay=pay, off=off, len=ln, out=R._fill(F * stride * 2), ns=R._fill(F * 4))
    call = lambda p, s: e.tx11b_legacy_raw(p["pay"], pay.size, p["off"], p["len"], F, 5500, 1, 0, 1, p["out"], stride, p["ns"], s)
    return Entry(args, ("out", "ns"), call, {"pay": 1})

def _tx11a_legacy(e):
    pay, off, ln = R._payloads([60, 25], 0xABC0); F = 2
    stride = api.Engine.tx11a_legacy_nsamples(64, 24000, 44)
    args = dict(pay=pay, off=off, len=ln, pre=oracle_tx11a_legacy.preamble(), out=R._fill(F * stride * 2), ns=R._fill(F * 4))
    call = lambda p, s: e.tx11a_legacy_raw(p["pay"], pay.size, p["off"], p["len"], F, 24000, 44, 0, p["pre"], p["out"], stride, p["ns"], s)
    return Entry(args, ("out", "ns"), call, {"pay": 1, "pre": 4})

def _viterbi(e):
    soft, stride, nsoft, nb, L = R._viterbi_input()
    args = dict(soft=soft, out=R._fill(nb * (L + 8)))
    return Entry(args, ("out",), lambda p, s: e.viterbi_raw(p["soft"], stride, nsoft, nb, api.CR_12, L, p["out"], L + 8, stream=s), {"soft": stride})

def _with(make, host=(), **opts):
    def f(e):
        ent = make(e); ent.opts = opts; ent.host |= set(host)
        return ent
    return f

ENTRIES = {
    "rx11a_batch": _rx11a,
    "rx11a_batch_chunked_device": _with(_rx11a, chunk_frames_device=2),   # front end on the handle's own stream, Viterbi on the caller's
    "rx11a_batch_chunked_host": _with(_rx11a, host=("iq",), chunk_frames=3),   # pageable capture, copies on the handle's copy stream
    "rx11a_batch_ex_20": _rx11a_ex(20), "rx11a_batch_ex_44": _rx11a_ex(44),
    "rx11b_batch": _rx11b, "rx11b_streams": _rx11b_streams, "rx11n_batch": _rx11n,
    "rx11a_streams": _rx11a_streams, "rx11n_streams": _rx11n_streams,
    "fir_decimate2": _fir, "channelize": _channelize, "rxblocks_unpack": _rxblocks_unpack, "rxblocks_desc": _rxblocks_desc,
    "tx11a_batch": _tx11a, "tx11b_batch": _tx11b, "tx11n_batch": _tx11n, "tx11b_fir37": _fir37,
    "tx11b_legacy_batch": _tx11b_legacy, "tx11a_legacy_batch": _tx11a_legacy, "viterbi_k7": _viterbi,
}
STREAM_MODE = ("rx11a_streams", "rx11n_streams")       # host tables and results by contract: these calls always return with results final

def _run_host(ent, args):
    """The synchronous all-host run: bytes of every output."""
    out = R._run(lambda p: ent.call(p, 0), args)
    return {k: out[k] for k in ent.outs}

@pytest.fixture(scope="module")
def warm():
    """name -> (engine with the entry's options, Entry, reference outputs of its all-host run); the engines close with the module."""
    cache = {}
    def get(name):
        if name not in cache:
            e = api.Engine(0)
            ent = ENTRIES[name](e)
            for k, v in ent.opts.items(): e.set_option(k, v)
            cache[name] = (e, ent, _run_host(ent, ent.args))
        return cache[name]
    yield get
    for e, _, _ in cache.values(): e.close()

def _alt(ent):
    return {k: np.roll(_bytes(ent.args[k]), r) for k, r in ent.roll.items()}

# ---- A: producer -> call -> consumer on one caller stream -------------------------------------------------------------------------

@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("name", list(ENTRIES))
def test_a_producer_call_consumer_on_one_stream(warm, name, kind):
    """Inputs start as garbage and are written by copy_ on the caller's stream after the gate; the call follows; the outputs are cloned on
    the stream.  Every buffer on the device (stream mode: the captures; the chunked host path: everything but the capture)."""
    e, ent, ref = warm(name)
    kinds = {k: "host" if k in ent.host else "dev" for k in ent.args}
    with caller_stream(kind) as (s, h):
        p, bufs = _place(ent.args, kinds)
        src = {k: bufs[k].clone() for k in ent.args if kinds[k] == "dev" and k not in ent.outs}
        for k in src: bufs[k].random_(0, 256)
        torch.cuda.synchronize()
        gate(s)
        with torch.cuda.stream(s):
            for k in src: bufs[k].copy_(src[k])
        ent.call(p, h)
        with torch.cuda.stream(s):
            got = {k: bufs[k].clone() if kinds[k] == "dev" else None for k in ent.outs}
        s.synchronize(); torch.cuda.synchronize()
        _check_outs(f"A {name} {kind}", ent, {k: _host(got[k] if got[k] is not None else bufs[k]) for k in ent.outs}, ref)

# ---- B: page-locked host inputs, device results ------------------------------------------------------------------------------------

B_ENTRIES = [n for n in ENTRIES if n not in STREAM_MODE and n != "rx11a_batch_chunked_device"]

@pytest.mark.parametrize("name", B_ENTRIES)
def test_b_page_locked_inputs_are_read_before_the_call_returns(warm, name):
    """Inputs in sb200_host_alloc memory, results on the device: right after the call returns, every input is overwritten with another
    valid input.  The results must be those of the original input."""
    e, ent, ref = warm(name)
    alt = _alt(ent)
    ref_alt = _run_host(ent, {**ent.args, **alt})
    assert any(not np.array_equal(ref_alt[k], ref[k]) for k in ent.outs), "the other input must give other results"
    kinds = {k: "pinned" if k in ent.roll else "dev" if k in ent.outs else "host" for k in ent.args}
    with pinned_pool() as alloc, caller_stream("nonblocking") as (s, h):
        p, bufs = _place(ent.args, kinds, alloc)
        torch.cuda.synchronize()
        gate(s)
        ent.call(p, h)
        for k, a in alt.items(): bufs[k][:] = a
        s.synchronize()
        _check_outs(f"B {name}", ent, {k: _host(bufs[k]) for k in ent.outs}, ref)

# ---- C: host_decimate's pinned staging across calls ------------------------------------------------------------------------------

def _oracle_11a(what, iq, off, ln, res, out, stride):
    ores, oout = oracle_py.rx11a_batch(iq.reshape(-1, 2), off, ln, out_stride=stride)
    for i in range(len(off)):
        for f in ("status", "rate_kbps", "length", "crc32", "nsym", "detect_index", "cfo_est"):
            assert res[f][i] == ores[f][i], f"{what}: slot {i} field {f}: got {res[f][i]}, oracle {ores[f][i]}"
        if res["status"][i] == api.FRAME_OK:
            n = min(int(res["length"][i]), stride)
            assert (out[i, :n] == oout[i, :n]).all(), f"{what}: slot {i}: delivered bytes differ from the oracle"
    assert (res["status"] == api.FRAME_OK).sum() >= len(off) // 2, f"{what}: too few frames decoded to mean anything"

def test_c_host_decimate_staging_is_not_reused_while_a_copy_is_queued():
    """Pageable host captures, results on the device, host_decimate 2 with every chunk gathered: call 1 gathers exactly four chunks, one per
    pinned staging buffer, and returns with their copies queued behind the gate; call 2 gathers another capture.  Both equal the oracle."""
    caps = [synth.make_frames(8, psdu_len=150, rate_kbps=24000, snr_db=30, seed0=seed)[0] for seed in (0xC0DE00, 0xC0DE80)]
    F, slot, _ = caps[0].shape; off, ln = R._slots(F, slot); S = 256
    e = api.Engine(0)
    try:
        e.set_option("host_decimate", 2); e.set_option("host_decimate_mix", 0); e.set_option("chunk_frames", 2)
        with caller_stream("nonblocking") as (s, h):
            res = [torch.full((F * api.RESULT_DTYPE.itemsize,), FILL, dtype=torch.uint8, device="cuda") for _ in caps]
            out = [torch.full((F * S,), FILL, dtype=torch.uint8, device="cuda") for _ in caps]
            host = [np.ascontiguousarray(c) for c in caps]
            torch.cuda.synchronize()
            gate(s)
            e.rx11a_raw(host[0].ctypes.data, F * slot, off.ctypes.data, ln.ctypes.data, F, out[0].data_ptr(), S, res[0].data_ptr(), h)
            assert e.last_transfer()[1:] == (4, 4), e.last_transfer()
            e.rx11a_raw(host[1].ctypes.data, F * slot, off.ctypes.data, ln.ctypes.data, F, out[1].data_ptr(), S, res[1].data_ptr(), h)
            s.synchronize()
        for j in range(2):
            _oracle_11a(f"C call {j + 1}", caps[j], off, ln, res[j].cpu().numpy().view(api.RESULT_DTYPE), out[j].cpu().numpy().reshape(F, S), S)
    finally:
        e.close()

# ---- D: one handle, two streams --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["rx11a_batch", "rx11n_batch", "channelize", "viterbi_k7"])
def test_d_calls_on_one_handle_keep_their_order_across_streams(warm, name):
    """Call 1 on gated stream A, call 2 (another input) on stream B, device buffers, host tables: once B is done, A must be too, since
    call 2 could not finish before call 1.  Both results equal their references."""
    e, ent, ref = warm(name)
    alt = _alt(ent); ref_alt = _run_host(ent, {**ent.args, **alt})
    kinds = {k: "host" if k in TABLES else "dev" for k in ent.args}
    with caller_stream("nonblocking") as (sa, ha), caller_stream("nonblocking") as (sb, hb):
        p1, b1 = _place(ent.args, kinds); p2, b2 = _place({**ent.args, **alt}, kinds)
        torch.cuda.synchronize()
        gate(sa)
        ent.call(p1, ha); ent.call(p2, hb)
        sb.synchronize(); a_done = sa.query()
        sa.synchronize()
        assert a_done, f"D {name}: call 2 on stream B finished while call 1 on stream A was still queued"
        _check_outs(f"D {name} call 1", ent, {k: _host(b1[k]) for k in ent.outs}, ref)
        _check_outs(f"D {name} call 2", ent, {k: _host(b2[k]) for k in ent.outs}, ref_alt)

# ---- E: concurrent handles -------------------------------------------------------------------------------------------------------

def _work_rx11a(e, h):
    iq, _ = synth.make_frames(6, psdu_len=200, rate_kbps=24000, snr_db=30, seed0=0xE11A00)
    F, slot, _ = iq.shape; off, ln = R._slots(F, slot)
    e.set_option("host_decimate", 2); e.set_option("chunk_frames", 2)
    def run():
        res = np.zeros(F, api.RESULT_DTYPE); out = np.zeros((F, 256), np.uint8)
        e.rx11a_raw(iq.ctypes.data, F * slot, off.ctypes.data, ln.ctypes.data, F, out.ctypes.data, 256, res.ctypes.data, h)
        return res, out
    return run

def _work_rx11b(e, h):
    iq, _ = synth.make_frames_11b(3, psdu_len=100, rate_kbps=11000, snr_db=35, gain=0.15, seed0=0xE11B00)
    F, slot, _ = iq.shape; off, ln = R._slots(F, slot)
    def run():
        res = np.zeros(F, api.RESULT11B_DTYPE); out = np.zeros((F, 256), np.uint8)
        e.rx11b_raw(iq.ctypes.data, F * slot, off.ctypes.data, ln.ctypes.data, F, out.ctypes.data, 256, res.ctypes.data, h)
        return res, out
    return run

def _work_rx11n(e, h):
    iq0, iq1, _ = synth.make_frames_11n(2, psdu_len=200, mcs=14, snr_db=40, lead=400, trail=200, seed0=0xE11E00)
    F, slot, _ = iq0.shape; off, ln = R._slots(F, slot)
    e.set_option("ht_mcs_limit", 15)
    def run():
        res = np.zeros(F, api.RESULT11N_DTYPE); out = np.zeros((F, 256), np.uint8)
        e.rx11n_raw(iq0.ctypes.data, iq1.ctypes.data, F * slot, off.ctypes.data, ln.ctypes.data, F, out.ctypes.data, 256, res.ctypes.data, h)
        return res, out
    return run

def _work_channelize_streams(e, h):
    """Two rows of one 40 Msps capture (channel 0 as it is, channel 1 with a constant phase) on the device, then decoded as streams."""
    iq, _ = synth.make_frames(4, psdu_len=100, rate_kbps=36000, snr_db=30, seed0=0xE1C000)
    x = np.ascontiguousarray(iq.reshape(-1, 2)); n = len(x); stride = (n + 3) // 4 * 4; K, M = 2, 4
    rows = torch.zeros(K * stride * 2, dtype=torch.int16, device="cuda"); torch.cuda.synchronize()
    off = np.arange(K, dtype=np.uint64) * stride; ln = np.full(K, n, np.uint32)
    def run():
        e.channelize_raw(x.ctypes.data, n, [(0, 0), (0, 1 << 29)], 1, np.array([32767], np.int16), rows.data_ptr(), stride, h)
        res = np.zeros(K * M, api.RESULT_DTYPE); out = np.zeros((K * M, 256), np.uint8); sidx = np.zeros(K * M, np.uint32); cnt = np.zeros(K, np.uint32)
        e._check(e._lib.sb200_rx11a_streams(e._h, V(rows.data_ptr()), U64(K * stride), V(off.ctypes.data), V(ln.ctypes.data), U32(K), U32(M), V(out.ctypes.data),
                                            U32(256), V(res.ctypes.data), V(sidx.ctypes.data), V(cnt.ctypes.data), V(h)), "sb200_rx11a_streams")
        return res, out, sidx, cnt
    return run

def test_e_concurrent_handles_on_their_own_streams():
    """Four host threads, each with its own engine and non-blocking stream, start together on a barrier and run one call each (ctypes
    releases the GIL): the same results as the same calls one after another."""
    works = [_work_rx11a, _work_rx11b, _work_rx11n, _work_channelize_streams]
    engines = []
    try:
        with contextlib.ExitStack() as stack:
            streams = [stack.enter_context(caller_stream("nonblocking")) for _ in works]
            engines = [api.Engine(0) for _ in works]
            runs = [w(e, h) for w, e, (_, h) in zip(works, engines, streams)]
            serial = [r() for r in runs]
            torch.cuda.synchronize()
            barrier, got, errors = threading.Barrier(len(runs)), [None] * len(runs), []
            def body(i):
                try:
                    barrier.wait(); got[i] = runs[i]()
                except BaseException as x:              # reported by the main thread
                    errors.append((i, x))
            threads = [threading.Thread(target=body, args=(i,)) for i in range(len(runs))]
            for t in threads: t.start()
            for t in threads: t.join()
            assert not errors, errors
        for w, a, b in zip(works, serial, got):
            for j, (x, y) in enumerate(zip(a, b)):
                _same(f"E {w.__name__} output {j}", _bytes(y), _bytes(x), a[0].dtype if j == 0 else None)
            assert (a[0]["status"] == api.FRAME_OK).any(), w.__name__
    finally:
        for e in engines: e.close()

# ---- F: the first call of a fresh engine on a non-blocking stream ----------------------------------------------------------------

def test_f_first_calls_on_a_non_blocking_stream():
    """Tables uploaded at create (802.11a receive), lazily on the first call (802.11n receive, transmit) or the channelizer's NCO table:
    the first call of a fresh engine on a non-blocking stream equals the oracle or the model.  (A regression guard: a race with the upload
    cannot be forced from here.)"""
    with caller_stream("nonblocking") as (s, h):
        e = api.Engine(0)
        try:
            iq, F, slot, off, ln = R._frames_11a()
            res = np.zeros(F, api.RESULT_DTYPE); out = np.zeros((F, 256), np.uint8)
            e.rx11a_raw(iq.ctypes.data, F * slot, off.ctypes.data, ln.ctypes.data, F, out.ctypes.data, 256, res.ctypes.data, h)
            _oracle_11a("F rx11a", iq, off, ln, res, out, 256)
        finally:
            e.close()
        e = api.Engine(0)
        try:
            iq0, iq1, F, slot, off, ln = R._frames_11n()
            res = np.zeros(F, api.RESULT11N_DTYPE); out = np.zeros((F, 256), np.uint8)
            e.rx11n_raw(iq0.ctypes.data, iq1.ctypes.data, F * slot, off.ctypes.data, ln.ctypes.data, F, out.ctypes.data, 256, res.ctypes.data, h)
            ores, oout = oracle_py.rx11n_batch(iq0.reshape(-1, 2), iq1.reshape(-1, 2), off, ln, out_stride=256)
            for f in ("status", "mcs", "length", "crc32", "nsym", "detect_index", "cfo_est", "lsig_length"):
                assert (res[f] == ores[f]).all(), ("F rx11n", f, res[f], ores[f])
            assert (res["status"] == api.FRAME_OK).all() and (out[:, :120] == oout[:, :120]).all()
        finally:
            e.close()
        e = api.Engine(0)
        try:
            x = _channelize_input(); out = np.full((len(CH_CHANNELS), CH_STRIDE, 2), -1, np.int16)
            e.channelize_raw(x.ctypes.data, CH_N, CH_CHANNELS, CH_D, CH_TAPS, out.ctypes.data, CH_STRIDE, h)
            n_out = -(-CH_N // CH_D)
            assert (out[:, :n_out] == wideband_inputs.channelize(x, CH_CHANNELS, CH_D, CH_TAPS)).all()
        finally:
            e.close()
        e = api.Engine(0)
        try:
            pay = [np.arange(77, dtype=np.uint8), np.full(300, 0x5A, np.uint8)]
            flat, offs, lens = api._payload_table(pay); stride = 640 + 160 * (2 + -(-(300 + 7) * 8 // 144) + 1) + 32
            out = np.full((2, stride, 2), 0x55, np.int8); ns = np.zeros(2, np.uint32)
            e.tx11a_raw(flat.ctypes.data, flat.size, offs.ctypes.data, lens.ctypes.data, 0, 2, 36000, 0, 8, out.ctypes.data, stride, ns.ctypes.data, h)
            for i, pl in enumerate(pay):
                want = oracle_py.tx11a_modulate(pl, 36000, 0xFF, 0)
                assert ns[i] == len(want) and (out[i, :len(want)] == want).all(), ("F tx11a", i)
        finally:
            e.close()

# ---- G: which calls return without waiting for their stream -----------------------------------------------------------------------

# sb200_rx11a_batch_ex at 44 Msps resamples into a device-resident slot table of its own and checks it like a caller's device table:
# one read-back, so it waits for the stream (unless slot_table_immutable is set).
WAITS = ("rx11a_batch_ex_44",)
G_ENTRIES = [n for n in ENTRIES if n != "rx11a_batch_chunked_host"]

@pytest.mark.parametrize("name", G_ENTRIES)
def test_g_device_buffers_and_host_tables_do_not_wait(warm, name):
    """On an engine that has made this call before: with every buffer on the device and host-resident tables the call returns while the
    gate still holds its stream; stream-mode calls return with their host results final."""
    e, ent, ref = warm(name)
    kinds = {k: "host" if k in ent.host or k in TABLES else "dev" for k in ent.args}
    with caller_stream("nonblocking") as (s, h):
        p, bufs = _place(ent.args, kinds)
        ent.call(p, h); s.synchronize()                 # the same call once with these buffers: workspaces sized
        for k in ent.outs:
            if kinds[k] == "dev": bufs[k].fill_(FILL)
            else: bufs[k][:] = FILL
        torch.cuda.synchronize()
        waited = _gated_call(ent, p, s, h)
        early = {k: _host(bufs[k]) for k in ent.outs if kinds[k] == "host"}
        s.synchronize()
        _check_outs(f"G {name}", ent, {k: early[k] if k in early else _host(bufs[k]) for k in ent.outs}, ref)
        if name in STREAM_MODE or name in WAITS:
            assert waited, f"G {name}: expected to wait for its stream"
        else:
            assert not waited, f"G {name}: waited for its stream although every buffer is on the device and the tables on the host"

def _gated_call(ent, p, s, h):
    """Gate s, call, and tell whether the call waited for what its stream held before it: the gate has passed when it returns (the
    call's host time is far below GATE_MS).  s.query() would not tell: a call that waited may still leave its own work queued."""
    gate(s)
    g = torch.cuda.Event(); g.record(s)
    ent.call(p, h)
    return g.query()

@pytest.mark.parametrize("immutable", [0, 1])
def test_g_device_slot_tables(warm, immutable):
    """Device-resident slot tables are checked on the device and the check read back, so the call waits for its stream; a repeated call
    under slot_table_immutable 1 reuses the cached check and does not."""
    e, ent, ref = warm("rx11a_batch")
    kinds = {k: "dev" for k in ent.args}
    try:
        e.set_option("slot_table_immutable", immutable)
        with caller_stream("nonblocking") as (s, h):
            p, bufs = _place(ent.args, kinds)
            ent.call(p, h); s.synchronize()
            for k in ent.outs: bufs[k].fill_(FILL)
            torch.cuda.synchronize()
            waited = _gated_call(ent, p, s, h)
            s.synchronize()
            _check_outs("G device tables", ent, {k: _host(bufs[k]) for k in ent.outs}, ref)
            assert waited != bool(immutable), f"slot_table_immutable {immutable}: waited for the stream: {waited}"
    finally:
        e.set_option("slot_table_immutable", 0)
