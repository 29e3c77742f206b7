"""GPU tests of the radio channel simulator (sb200_channel_sim, pytest -m gpu): bit for bit against the numpy model of tests/sim_model.py
over lengths around a tile, row counts, tap counts, clock steps and fractional delays, increments, noise levels and rail inputs, tap sums
at the limit and thousands of links; the pointer residency, stream, launch bookkeeping and argument checks of the C ABI; device-resident
chains transmitter -> simulator -> batch receiver against the CPU oracle on the model's output; and the error rate of 4096 links."""
import ctypes as C
import numpy as np, pytest
import torch
import oracle_py
import sim_model as SM
from sora_b200 import api
from test_gpu_abi_residency import _matrix, _each, _fill
from test_cpu_channel_sim import frame_11a, frame_11b, frame_11n, link_for, decode_11a, decode_11b, decode_11n

pytestmark = pytest.mark.gpu
V, U32, U64 = C.c_void_p, C.c_uint32, C.c_uint64
S32 = 1 << 32

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

def _tile(T):
    return 2048 if T <= 2 else 1024

def _rows(nl, T, n, seed, lim=32768):
    return np.random.default_rng(seed).integers(-lim, lim, (nl, T, n, 2)).astype(np.int16)

def _taps(nl, R, T, L, seed, total=60000):
    """Random Q14 taps with every (link, r) row's sum of |re| + |im| at most `total` (exactly `total` when total == 65535)."""
    rng = np.random.default_rng(seed)
    g = rng.integers(-3000, 3000, (nl, R, T, L, 2)).astype(np.float64); g[:, :, :, 0, 0] += 12000
    s = np.abs(g).sum((2, 3, 4), keepdims=True)
    g = np.trunc(g * np.minimum(total / s, 1.0)).astype(np.int64)
    if total == 65535:                                                   # top the largest tap up to an exact 65535
        d = 65535 - np.abs(g).sum((2, 3, 4)); g[:, :, 0, 0, 0] += d * np.sign(g[:, :, 0, 0, 0] + (g[:, :, 0, 0, 0] == 0))
    return g.astype(np.int16)

STEPS = [S32, S32 - (1 << 24), S32 + (1 << 24), api.clock_step(20), api.clock_step(-40), S32 + 12345]

def _links(nl, seed, sigma=(0, 300, 25600)):
    rng = np.random.default_rng(seed)
    return [(int(rng.integers(0, 40)) * S32 + int(rng.choice([0, 128, 255])) * (1 << 24) + int(rng.integers(0, 1 << 24)),
             STEPS[i % len(STEPS)], int(rng.integers(-2 ** 31, 2 ** 32)), int(rng.integers(0, 2 ** 32)) if i % 2 else 0, sigma[i % len(sigma)])
            for i in range(nl)]

def _same(eng, x, links, taps, n_out, seed):
    got = eng.channel_sim(x, links, taps, n_out, seed); want = SM.sim(x, links, taps, n_out, seed)
    assert got.shape == want.shape and (got == want).all(), np.argwhere((got != want).any(-1))[:5]


@pytest.mark.parametrize("T,R,L", [(1, 1, 1), (1, 1, 16), (2, 2, 17), (4, 4, 64), (1, 4, 2), (4, 1, 17), (2, 4, 64), (4, 2, 1)])
def test_lengths_rows_and_taps(eng, T, R, L):
    """n_out around the tile the call picks, T and R in {1, 2, 4} with T != R, L in {1, 2, 17, 64}; full-scale random input."""
    tm = _tile(T)
    for k, n in enumerate((1, 5, tm - 1, tm, tm + 1, 2 * tm + 77)):
        nl = 3
        _same(eng, _rows(nl, T, n + 50, 10 * k + T), _links(nl, k + 7 * L), _taps(nl, R, T, L, k + R), n, 0x1234 + k)

def test_steps_and_fractions(eng):
    """step at 2^32 - 2^24, 2^32 and 2^32 + 2^24, tau0 fractions at p = 0, 128 and 255 (and just around them), wrapping and negative
    increments; n_in shorter and longer than the clock needs."""
    links = []
    for step in (S32 - (1 << 24), S32, S32 + (1 << 24)):
        for p in (0, 128, 255):
            for d in (0, (1 << 23) - 1, 1 << 23, (1 << 24) - 1):
                links.append((5 * S32 + p * (1 << 24) + d, step, (-0x12345) % 2 ** 32 if p else 2 ** 31 + 1, 0xFFF00000, 0))
    nl = len(links)
    for n_in, n_out in ((3000, 3000), (2000, 3000), (4000, 2500)):
        _same(eng, _rows(nl, 1, n_in, n_in), links, _taps(nl, 2, 1, 3, n_in), n_out, 1)

def test_noise_levels_and_rails(eng):
    """sigma 0, 1, 256 and the largest (2^24 - 1) on rail inputs through taps summing to exactly 65535: every stage clips."""
    nl, n = 4, 5000
    x = np.where(np.random.default_rng(3).random((nl, 2, n, 2)) < 0.5, -32768, 32767).astype(np.int16)
    links = [(0, S32, 0, 0, 0), (S32 // 2, S32 + 999, 2 ** 30, 7, 1), (3 * S32, S32 - 999, 0, 0, 256), (0, S32, 0x9E3779B9, 0, (1 << 24) - 1)]
    taps = _taps(nl, 2, 2, 9, 4, total=65535)
    assert (np.abs(taps.astype(np.int64)).sum((2, 3, 4)) == 65535).all()
    got = eng.channel_sim(x, links, taps, n, 2 ** 63 + 5)
    assert (got == SM.sim(x, links, taps, n, 2 ** 63 + 5)).all()
    assert (np.abs(got[3].astype(np.int64)) >= 32767).mean() > 0.3

def test_thousands_of_links(eng):
    """3000 links, every record different, seeds with the high word set; a sample of the links against the model."""
    nl, n = 3000, 700
    x = _rows(nl, 1, n, 5, lim=8000); links = _links(nl, 11); taps = _taps(nl, 2, 1, 5, 12)
    for seed in (0xDEADBEEF00000001, 2 ** 64 - 1):
        got = eng.channel_sim(x, links, taps, n, seed)
        pick = [0, 1, 2, 999, 1500, 2998, 2999]
        want = SM.sim_window(x[pick], [links[l] for l in pick], taps[pick], seed, 0, n, link_ids=pick)
        assert (got[pick] == want).all()


# ---- long captures -------------------------------------------------------------------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count

def test_long_captures(eng):
    """One link longer than 4 x SMs tiles, device-resident: windows at the start, the middle and the end against sim_window."""
    T, R, L = 2, 2, 17; n = (4 * _sms() + 3) * _tile(T) + 777; si = (n + 3) // 4 * 4
    x = _rows(1, T, si, 9); links = [(7 * S32 + (1 << 31), api.clock_step(35), 0xFFFF0000, 123, 900)]; taps = _taps(1, R, T, L, 9)
    dx = torch.from_numpy(x).cuda(); dy = torch.zeros((1, R, si, 2), dtype=torch.int16, device="cuda")
    eng.channel_sim_raw(dx.data_ptr(), T * si, si, T, si, api.sim_links(links), taps, L, 1, 77, dy.data_ptr(), R * si, si, R, n)
    for m0, m1 in ((0, 600), (n // 2 - 300, n // 2 + 300), (n - 600, n)):
        assert (dy[0, :, m0:m1].cpu().numpy() == SM.sim_window(x, links, taps, 77, m0, m1)[0]).all(), m0


# ---- the C ABI ------------------------------------------------------------------------------------------------------------------------
def test_a_window_is_the_slice(eng):
    """y of a shorter n_out equals the first outputs of a longer one; the rows of a transposed output layout (row stride = nlinks x link
    stride, the layout of rx11n_batch's iq0 / iq1) equal those of the nested one."""
    nl, T, R, L, n = 5, 2, 2, 8, 3000
    x = _rows(nl, T, n, 21); links = _links(nl, 21); taps = _taps(nl, R, T, L, 21)
    full = eng.channel_sim(x, links, taps, n, 5)
    assert (eng.channel_sim(x, links, taps, 1234, 5) == full[:, :, :1234]).all()
    y = np.zeros((R, nl, n, 2), np.int16)
    eng.channel_sim_raw(api._ptr(np.ascontiguousarray(x)), T * n, n, T, n, api.sim_links(links), taps, L, nl, 5, api._ptr(y), n, nl * n, R, n)
    assert (y.transpose(1, 0, 2, 3) == full).all()

def test_residency(eng):
    """x, links, taps and y each host or device; the samples between the output rows untouched."""
    nl, T, R, L, n, gap = 3, 2, 2, 5, 1001, 24
    x = np.full((nl, T, 1004, 2), 0x5A5A, np.int16); x[:, :, :n] = _rows(nl, T, n, 50)
    links = api.sim_links(_links(nl, 50)); taps = _taps(nl, R, T, L, 50)
    ols, ors = R * (1004 + gap), 1004 + gap
    args = dict(x=x, links=links.view(np.uint8), taps=taps, y=_fill(nl * ols * 4 + 16))
    ref = _matrix(lambda p: eng.channel_sim_raw(p["x"], T * 1004, 1004, T, n, p["links"], p["taps"], L, nl, 9, p["y"], ols, ors, R, n), args, _each(*args))
    y = ref["y"][:nl * ols * 4].view(np.int16).reshape(nl, R, ors, 2)
    assert (y[:, :, :n] == SM.sim(x[:, :, :n], links, taps, n, 9)).all()
    assert (y[:, :, n:].view(np.uint8) == 0xA5).all() and (ref["y"][nl * ols * 4:] == 0xA5).all()

def test_a_callers_stream(eng):
    nl, T, R, L, n = 4, 1, 2, 16, 20001; si = (n + 3) // 4 * 4
    x = _rows(nl, T, si, 51); links = _links(nl, 51); taps = _taps(nl, R, T, L, 51)
    dx = torch.from_numpy(x).cuda(); s = torch.cuda.Stream(); s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        dy = torch.zeros((nl, R, si, 2), dtype=torch.int16, device="cuda")
        eng.channel_sim_raw(dx.data_ptr(), T * si, si, T, n, api.sim_links(links), taps, L, nl, 3, dy.data_ptr(), R * si, si, R, n, s.cuda_stream)
        got = dy[:, :, :n].cpu().numpy()
    assert (got == SM.sim(x[:, :, :n], links, taps, n, 3)).all()

def test_one_launch_and_timing():
    e = api.Engine(0)
    try:
        x = _rows(8, 2, 20000, 60); links = _links(8, 60); taps = _taps(8, 2, 2, 16, 60)
        for _ in range(2):
            n0 = e.launches; e.channel_sim(x, links, taps, 20000, 1)
            assert e.launches - n0 == 1 and e.last_kernel_ms() > 0
    finally:
        e.close()

def _call(eng, x, ils, irs, T, n_in, lk, tp, L, nl, y, ols, ors, R, n_out):
    return eng._lib.sb200_channel_sim(eng._h, V(x), U64(ils), U64(irs), U32(T), U64(n_in), V(lk), V(tp), U32(L), U32(nl), U64(1), V(y), U64(ols), U64(ors),
                                      U32(R), U64(n_out), V(0))

def test_invalid_arguments_are_rejected(eng):
    nl, T, R, L, n = 2, 2, 2, 4, 1000
    x = _rows(nl, T, n, 70); y = np.zeros((nl, R, n, 2), np.int16)
    good = api.sim_links([(0, S32, 0, 0, 100)] * nl); taps = _taps(nl, R, T, L, 70)
    xp, yp, lp, tp = x.ctypes.data, y.ctypes.data, good.ctypes.data, taps.ctypes.data
    ok = (xp, T * n, n, T, n, lp, tp, L, nl, yp, R * n, n, R, n)
    assert _call(eng, *ok) == 0
    def rec(**kw):
        b = good.copy()
        for k, v in kw.items(): b[k][1] = v
        return b
    bads = {"step low": rec(step=S32 - (1 << 24) - 1), "step high": rec(step=S32 + (1 << 24) + 1), "tau0": rec(tau0=1 << 62), "noise": rec(noise_q8=1 << 24)}
    hot = _taps(nl, R, T, L, 70, total=65535); hot[1, 1, 1, 2, 1] += 1 if hot[1, 1, 1, 2, 1] >= 0 else -1
    keep = []
    def k(a): keep.append(a); return a.ctypes.data
    n0 = eng.launches
    cases = {"ntx 0": dict(T=0), "ntx 5": dict(T=5), "nrx 0": dict(R=0), "nrx 5": dict(R=5), "ntaps 0": dict(L=0), "ntaps 65": dict(L=65),
             "n_in > 2^30": dict(n_in=(1 << 30) + 1), "n_out > 2^30": dict(n_out=(1 << 30) + 1), "in stride % 4": dict(irs=n + 2),
             "out stride % 4": dict(ors=n + 2), "link stride % 4": dict(ils=T * n + 2), "rows overlap": dict(ors=n - 4),
             "links overlap": dict(ols=R * n - 4), "transposed overlap": dict(ols=n, ors=n), "null x": dict(x=0), "null y": dict(y=0),
             "null links": dict(lk=0), "null taps": dict(tp=0), "tap sum 65536": dict(tp=k(hot))}
    cases.update({"link " + name: dict(lk=k(b)) for name, b in bads.items()})
    names = ("x", "ils", "irs", "T", "n_in", "lk", "tp", "L", "nl", "y", "ols", "ors", "R", "n_out")
    for name, kw in cases.items():
        a = dict(zip(names, ok)); a.update(kw)
        assert _call(eng, *[a[q] for q in names]) == -1, name
    # the same limits with the tables on the device: checked there
    for name, b in list(bads.items()) + [("tap sum 65536", None)]:
        dl = torch.from_numpy((b if b is not None else good).view(np.uint8).copy()).cuda()
        dt = torch.from_numpy((hot if b is None else taps).copy()).cuda()
        assert _call(eng, xp, T * n, n, T, n, dl.data_ptr(), dt.data_ptr(), L, nl, yp, R * n, n, R, n) == -1, "device " + name
    d = torch.zeros(nl * T * n * 2 + 8, dtype=torch.int16, device="cuda")
    assert _call(eng, d.data_ptr() + 4, T * n, n, T, n - 4, lp, tp, L, nl, yp, R * n, n, R, n) == -1, "misaligned device x"
    assert _call(eng, xp, T * n, n, T, n, lp, tp, L, nl, d.data_ptr() + 4, R * n, n, R, n - 4) == -1, "misaligned device y"
    assert eng.launches == n0, "a refused call launched"
    # accepted edges: both step limits, a tap sum of exactly 65535, a transposed layout
    lim = api.sim_links([(0, S32 - (1 << 24), 0, 0, 0), ((1 << 62) - 1, S32 + (1 << 24), 0, 0, (1 << 24) - 1)])
    ok65535 = _taps(nl, R, T, L, 70, total=65535)
    assert _call(eng, xp, T * n, n, T, n, lim.ctypes.data, ok65535.ctypes.data, L, nl, yp, R * n, n, R, n) == 0
    yt = np.zeros((R, nl, n, 2), np.int16)
    assert _call(eng, xp, T * n, n, T, n, lp, tp, L, nl, yt.ctypes.data, n, nl * n, R, n) == 0


# ---- device-resident chains: transmitter -> simulator -> batch receiver -----------------------------------------------------------------
def _dev_sim(eng, rows, links, taps, n_out, seed):
    """rows: device int16 [nl, T, si, 2] -> device y [nl, R, so, 2] through sb200_channel_sim."""
    nl, T, si = rows.shape[:3]; R, L = taps.shape[-4], taps.shape[-2]; so = (n_out + 3) // 4 * 4
    t = np.ascontiguousarray(np.broadcast_to(taps, (nl,) + taps.shape[-4:]))
    y = torch.zeros((nl, R, so, 2), dtype=torch.int16, device="cuda")
    eng.channel_sim_raw(rows.data_ptr(), T * si, si, T, si, api.sim_links(links), t, L, nl, seed, y.data_ptr(), R * so, so, R, n_out)
    return y, t

@pytest.mark.parametrize("rate", [6000, 24000, 54000])
def test_chain_11a(eng, rate):
    """tx11a (device) -> simulator -> rx11a_batch (device), against the oracle receiver on the model's output."""
    x, psdu, links, taps, n_out, seed = frame_11a(rate, 30, nl=4)
    rows = torch.from_numpy(x).cuda()
    y, t = _dev_sim(eng, rows, links, taps, n_out, seed)
    want = SM.sim(x, links, t, n_out, seed)
    assert (y[:, :, :n_out].cpu().numpy() == want).all()
    so = y.shape[2]; off = np.arange(len(x), dtype=np.uint64) * so; ln = np.full(len(x), n_out, np.uint32)
    res = np.zeros(len(x), api.RESULT_DTYPE); out = np.zeros((len(x), 4096), np.uint8)
    eng.rx11a_raw(y.data_ptr(), len(x) * so, api._ptr(off), api._ptr(ln), len(x), api._ptr(out), 4096, api._ptr(res))
    o, ob = oracle_py.rx11a_batch(want.reshape(-1, 2) if so == n_out else np.ascontiguousarray(y.cpu().numpy()).reshape(-1, 2), off, ln, out_stride=4096)
    for k in ("status", "rate_kbps", "length", "crc32", "detect_index", "cfo_est"): assert (res[k] == o[k]).all(), k
    assert (res["status"] == oracle_py.E_FRAME_OK).all() and all((out[i, :len(psdu)] == psdu).all() for i in range(len(x)))

def test_chain_11b(eng):
    x, psdu, links, taps, n_out, seed = frame_11b(30, nl=3)
    y, t = _dev_sim(eng, torch.from_numpy(x).cuda(), links, taps, n_out, seed)
    yh = y.cpu().numpy(); assert (yh[:, :, :n_out] == SM.sim(x, links, t, n_out, seed)).all()
    so = y.shape[2]; off = np.arange(len(x), dtype=np.uint64) * so; ln = np.full(len(x), n_out, np.uint32)
    res = np.zeros(len(x), api.RESULT11B_DTYPE); out = np.zeros((len(x), 4096), np.uint8)
    eng.rx11b_raw(y.data_ptr(), len(x) * so, api._ptr(off), api._ptr(ln), len(x), api._ptr(out), 4096, api._ptr(res))
    o, ob = oracle_py.rx11b_batch(yh.reshape(-1, 2), off, ln, out_stride=4096)
    for k in ("status", "rate_kbps", "length", "crc32"): assert (res[k] == o[k]).all(), k
    assert all((out[i, :len(psdu) - 1] == psdu[:-1]).all() for i in range(len(x)))

@pytest.mark.parametrize("mcs", [8, 10])
def test_chain_11n(eng, mcs):
    """tx11n's two streams as the rows of a 2x2 link; R = 2 rows out in the transposed layout, as rx11n_batch's iq0 and iq1."""
    x, psdu, links, taps, n_out, seed = frame_11n(mcs, 30, nl=3)
    nl, T, si = x.shape[:3]; so = (n_out + 3) // 4 * 4; L = taps.shape[-2]
    t = np.ascontiguousarray(np.broadcast_to(taps, (nl,) + taps.shape[-4:]))
    rows = torch.from_numpy(x).cuda(); y = torch.zeros((2, nl, so, 2), dtype=torch.int16, device="cuda")
    eng.channel_sim_raw(rows.data_ptr(), T * si, si, T, si, api.sim_links(links), t, L, nl, seed, y.data_ptr(), so, nl * so, 2, n_out)
    want = SM.sim(x, links, t, n_out, seed); yh = y.cpu().numpy()
    assert (yh[:, :, :n_out].transpose(1, 0, 2, 3) == want).all()
    off = np.arange(nl, dtype=np.uint64) * so; ln = np.full(nl, n_out, np.uint32)
    r, o = eng.rx11n_batch(yh[0].reshape(-1, 2), yh[1].reshape(-1, 2), off, ln)
    orr, oo = oracle_py.rx11n_batch(yh[0].reshape(-1, 2), yh[1].reshape(-1, 2), off, ln, out_stride=o.shape[1])
    for k in ("status", "mcs", "length", "crc32"): assert (r[k] == orr[k]).all(), k
    assert (r["status"] == oracle_py.E_FRAME_OK).all() and all((o[i, :len(psdu)] == psdu).all() for i in range(nl))


# ---- error rate at scale ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("snr,ok", [(40, True), (-5, False)])
def test_error_rate_4096_links(eng, snr, ok):
    """One 54 Mbps frame, 4096 links with different clock offsets (-10 .. +10 ppm, carrier offsets matched at 5.2 GHz, at most
    52 kHz: near +-115 kHz the 54 Mbps receiver fails a few % of FCS checks even at 40 dB) and noise: every frame decodes at 40 dB SNR and
    none at -5 dB."""
    x1, psdu, links1, taps, n_out, _ = frame_11a(54000, snr, nl=1)
    nl = 4096; rng = np.random.default_rng(snr + 100)
    tau0, step, inc, ph, sig = links1[0]
    links = [(tau0, api.clock_step(float(p)), api.phase_inc(-float(p) * 1e-6 * 5.2e9, 40e6), int(rng.integers(0, 2 ** 32)), sig) for p in rng.uniform(-10, 10, nl)]
    rows = torch.from_numpy(x1).cuda().expand(nl, -1, -1, -1).contiguous()
    y, _ = _dev_sim(eng, rows, links, taps, n_out, 0xABCDEF0123456789)
    so = y.shape[2]; off = np.arange(nl, dtype=np.uint64) * so; ln = np.full(nl, n_out, np.uint32)
    res = np.zeros(nl, api.RESULT_DTYPE); out = np.zeros((nl, 2048), np.uint8)
    eng.rx11a_raw(y.data_ptr(), nl * so, api._ptr(off), api._ptr(ln), nl, api._ptr(out), 2048, api._ptr(res))
    good = (res["status"] == api.FRAME_OK) & (out[:, :len(psdu)] == psdu).all(1)
    assert good.all() if ok else not good.any(), int(good.sum())
