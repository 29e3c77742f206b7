"""The OFDM transforms against the reference's OWN code: FFT<64> (fft_r4dif.h), IFFT<64> and IFFT<128> (ifft_r4dif.h) compiled from
kernel/core/inc where they lie, with their twiddle and bit-reversal tables (oracle/build_ref_fft.sh -> oracle/_ref/libfft_ref.so).  Every
other test compares the device with oracle/tables.cpp, a restatement of those headers; here the restatement and the host-compiled device
sources must equal the compiled reference byte for byte:
  - 10^6 random full-scale vectors per transform;
  - structured patterns over the int16 edges: all inputs equal, alternating sign, an impulse at every position, a full-scale tone at
    every bin, one input at an edge while the others are zero or at the opposite edge;
  - a searched corpus that drives the reference's debug tap (saturating adds and subtracts that clip, packs that drop significant bits,
    pmaddwd sums that wrap), kept below as constants;
  - the inputs the chains produce: the 802.11a front end's cmul_q15(x >> 1, FreqCoeffs) for every CFO of the rotation table, the raw
    802.11n symbols, what the receivers hand fft64 on full-scale captures, the zero-stuffed IFFT<128> symbols of all three transmitters at
    every rate and MCS, and the STS input of build_sts.
Device sources on the host (tests/cpp/fft_emu.cpp): the scalar r4_butterfly / dft4 chain of k_front11n and the packed pk_r4_butterfly /
pk_dft4 chain of k_front11a, both in the kernels' order, and host_ifft64 with the STS table of tables.cuh.  warp_ifft128
(tx11a_kernels.cuh) is not run here: its header includes the whole 802.11a receive kernel file, which needs most of the CUDA warp
intrinsics to compile for the host.  tests/test_gpu_fft_reference.py ties it, and the device FFT, to the compiled reference on the GPU."""
import ctypes as C, os, shutil, subprocess
import numpy as np, pytest
import oracle_py, rail_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EDGES = np.array([-32768, -32767, -16385, -16384, -8193, -8192, -1, 0, 1, 8191, 8192, 16383, 16384, 32766, 32767], np.int16)
HEX = "0123456789abcde"                     # corpus digit k stands for EDGES[k]

# Found by hill-climbing each tap counter over inputs drawn from EDGES (one digit per int16 component, re then im per point): the most
# pack lanes that drop significant bits in one transform (FFT<64>: 10, IFFT<64>: 8, IFFT<128>: 7 lanes).
FFT64_PACK = ("cbad03b17e5530c4661e38ee18d3930a5515d360d13dad5de0ce1be93d10abbec2e0041e511551b33bc15870e98d86ed9dedeeec18a37de9d3024810d0bd1b01")
IFFT64_PACK = ("50717700e00e8e0a99c03c7b89e0006edbe166ed5d06c007c598b820766b23d778de1b10a08b3ddd810d85841e0e4dc03311b1eb0c76d1d1d7106d5850508119")
IFFT128_PACK = ("570ada377a57e4ca5801b01e2702c7a8a93b9b0e36dc2710683eeca507c065e3da6be0474316ce0d97d705615c0dd9378ced2368b68e72ae9866bb1a8203471e"
                "9a8d60011db35eeb1a3088d6530d8dda0ac02c00820585341a7145a21401c3130335e7210b71003714ec21ce1de07661d1215079e6d1628aa501857d86a603a1")
# A saturated_add that clips in IFFT<128>: a period of 8 points tiled 16 times reaches IFFTSSEEx<8>'s first block unscaled (both radix-4
# stages sum four equal quarters of x >> 2), and this period makes lane 0 of its last add u0.re + 0.707 (u1.re - u1.im) = 16380 + 23165.
# No random or hill-climbed input found one: the count is 0 almost everywhere, so a climb has nothing to follow.
_M, _P = -32768, 32767
IFFT128_SAT = np.tile(np.array([[_P, 0], [_P, _M], [0, _M], [_M, _M], [_M, 0], [_M, _P], [0, _P], [_P, _P]], np.int16), (16, 1))

pytestmark = pytest.mark.skipif(not oracle_py.ref_fft_available(), reason="oracle/_ref/libfft_ref.so not built (needs the reference tree)")

XFORMS = {"fft64": (64, oracle_py.fft64, oracle_py.ref_fft64), "ifft64": (64, oracle_py.ifft64, oracle_py.ref_ifft64),
          "ifft128": (128, oracle_py.ifft128, oracle_py.ref_ifft128)}

def corpus_vec(s, N):
    return EDGES[np.array([HEX.index(c) for c in s])].reshape(N, 2)

def ref_with_taps(name, x):
    """(reference output, tap counts over this call)."""
    return XFORMS[name][2](x), oracle_py.ref_fft_debug()

def check_equal(name, x, what):
    """oracle == reference on every vector of x [n, N, 2]; returns the reference's tap counts over x."""
    _, ora, _ = XFORMS[name]
    r, taps = ref_with_taps(name, x)
    o = ora(x)
    bad = np.flatnonzero((o != r).reshape(len(x), -1).any(1))
    assert bad.size == 0, "%s %s: %d of %d vectors differ, first %d: x=%s ref=%s oracle=%s" % (name, what, bad.size, len(x), bad[0], x[bad[0]].tolist(), r[bad[0]].tolist(), o[bad[0]].tolist())
    return r, taps

def assert_unreachable(name, taps):
    """The tap counters no input can raise.  pmaddwd wraps only when both products are (-32768)^2, and every second operand of a product
    in these transforms is a twiddle (or its flipped / XOR-conjugated form, or the conjre'd input against a twiddle), whose components are
    trunc(32767 cos), trunc(-32767 sin) in [-32767, 32767]: mul_shift's XOR conjugate gives -32768 only from a twiddle im of 32767, i.e.
    sin = -1 at j m / N = 3 / 4, past the last twiddle index.  Every saturated_sub takes two values that were just shifted right by 2 (3 in
    IFFTSSEEx<8>), so it cannot leave int16; nor can any saturated_add of the 64-point transforms, whose operands are at most two such
    values deep.  Only IFFTSSEEx<8> adds the (wrapped) output of a twiddle product, which can clip."""
    assert taps["madd"] == 0 and taps["sat_sub"] == 0, (name, taps)
    if name != "ifft128": assert taps["sat_add"] == 0, (name, taps)

def c16(re, im):
    return np.stack([np.asarray(re), np.asarray(im)], -1).astype(np.int16)

# ---- the compiled reference itself ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(XFORMS))
def test_reference_close_to_float_dft(name):
    """Sanity of the compiled reference (and of its shim): at +-6000 it is a DFT scaled by 1 / N, within a few LSB of float64.  FFT<64>
    gives DFT(x) / 64 with e^{-j}; the inverse transforms give np.fft.ifft(x) (their stages shift right by log2 N in all).  The truncating
    shifts and one's-complement negations bias every component by about -1.6 LSB; measured: largest error 8.7 LSB (64-point), 11.9
    (IFFT<128>), mean 2.4 / 2.9.  A conjugated twiddle or a wrong sign is off by hundreds."""
    N, _, ref = XFORMS[name]
    x = np.random.default_rng(1).integers(-6000, 6001, (2000, N, 2)).astype(np.int16)
    z = x[..., 0] + 1j * x[..., 1].astype(np.float64)
    want = np.fft.fft(z, axis=1) / N if name == "fft64" else np.fft.ifft(z, axis=1)
    r = ref(x); got = r[..., 0] + 1j * r[..., 1]
    err = np.abs(got - want)
    assert err.max() < 16 and err.mean() < 4, (name, err.max(), err.mean())
    assert np.abs(got).max() > 1000, name

# ---- oracle against reference -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(XFORMS))
def test_random_full_scale(name):
    """10^6 vectors of uniform int16 components."""
    N = XFORMS[name][0]
    x = np.random.default_rng(1000 + N + len(name)).integers(-32768, 32768, (1_000_000, N, 2)).astype(np.int16)
    _, taps = check_equal(name, x, "random")
    assert taps["pack"] > 1000, (name, taps)
    assert_unreachable(name, taps)

def structured(N):
    """(name, [n, N, 2]) pattern families over the int16 edges, in both halves."""
    e = EDGES.astype(np.int64); re, im = np.meshgrid(e, e, indexing="ij"); pairs = c16(re.ravel(), im.ravel())     # 225 (re, im) points
    n = np.arange(N)
    out = [("equal", np.repeat(pairs[:, None, :], N, 1))]
    sign = np.where(n % 2 == 0, 1, -1)[None, :, None]
    out.append(("alternating", (pairs[:, None, :].astype(np.int64) * sign).astype(np.int16)))                      # -(-32768) wraps, as in int16
    alt_opp = np.repeat(pairs[:, None, :], N, 1); alt_opp[:, 1::2] = ~alt_opp[:, 1::2]                              # v, ~v, v, ~v ...
    out.append(("alternating_opposite", alt_opp))
    imp = np.zeros((len(pairs), N, N, 2), np.int16)
    imp[:, np.arange(N), np.arange(N)] = pairs[:, None, :]
    out.append(("impulse", imp.reshape(-1, N, 2)))
    tones = []
    for k in range(N):
        for amp, ph in ((32768.0, 0.0), (32768.0, np.pi / 4), (23170.0, 0.3), (46341.0, 0.0)):                 # 46341: clipped corners
            z = amp * np.exp(1j * (2 * np.pi * k * n / N + ph))
            tones.append(c16(np.clip(np.round(z.real), -32768, 32767), np.clip(np.round(z.imag), -32768, 32767)))
    out.append(("tone", np.array(tones)))
    one = []
    for v in EDGES:
        for p in range(N):
            for bg, sel in ((0, (v, v)), (0, (v, ~v)), (~v, (v, v)), (~v, (v, ~v))):
                x = np.full((N, 2), bg, np.int16); x[p] = sel; one.append(x)
    out.append(("one_edge", np.array(one)))
    return out

@pytest.mark.parametrize("name", sorted(XFORMS))
def test_structured_edges(name):
    N = XFORMS[name][0]
    for fam, x in structured(N):
        _, taps = check_equal(name, x, fam)
        assert_unreachable(name, taps)

def corpus():
    return {"fft64": [corpus_vec(FFT64_PACK, 64)], "ifft64": [corpus_vec(IFFT64_PACK, 64)], "ifft128": [corpus_vec(IFFT128_PACK, 128), IFFT128_SAT]}

def test_search_corpus_reaches_every_edge():
    """The kept inputs equal the oracle and make every reachable tap counter non-zero: pack drops significant bits in all three
    transforms, saturated_add clips in IFFT<128>.  The unreachable counters (assert_unreachable) stay zero."""
    want = {"fft64": 10, "ifft64": 8, "ifft128": 7}
    for name, vecs in corpus().items():
        total = dict.fromkeys(oracle_py.REF_FFT_COUNTERS, 0)
        for x in vecs:
            _, taps = check_equal(name, x[None], "corpus")
            for k in total: total[k] += taps[k]
        assert total["pack"] >= want[name], (name, total)
        if name == "ifft128": assert total["sat_add"] >= 1, total
        assert_unreachable(name, total)
    _, taps = ref_with_taps("ifft128", IFFT128_SAT[None])
    assert taps["sat_add"] >= 1, taps

# ---- the inputs the chains produce ---------------------------------------------------------------------------------------------------
def cmul_q15(a, b):
    """oracle/ops.h cmul_q15 on int16 [..., 2] arrays: (a * b) >> 15 per component, the real part through neg16(b.im), truncating pack."""
    a = a.astype(np.int64); b = b.astype(np.int64)
    nbi = (-b[..., 1]).astype(np.int16).astype(np.int64)
    re = (a[..., 0] * b[..., 0] + a[..., 1] * nbi).astype(np.int32) >> 15
    im = (a[..., 0] * b[..., 1] + a[..., 1] * b[..., 0]).astype(np.int32) >> 15
    return c16(re.astype(np.int16), im.astype(np.int16))

def test_rx11a_front_end_domain():
    """k_front11a / Rx11a::on_symbol hand fft64 cmul_q15(x >> 1, FreqCoeffs), FreqCoeffs[i] = (ucos(i cfo), -usin(i cfo)): every int16
    CFO once, each with its own full-scale x (random, or on the rails)."""
    L = oracle_py.lib()
    sinl = np.array([L.sbo_usin(r) for r in range(-32768, 32768)], np.int64); cosl = np.array([L.sbo_ucos(r) for r in range(-32768, 32768)], np.int64)
    cfo = np.arange(-32768, 32768, dtype=np.int64)
    ph = ((cfo[:, None] * np.arange(64)[None, :] + 32768) % 65536)                       # index into the tables above, int16 phase + 32768
    fc = c16(cosl[ph], (-sinl[ph]).astype(np.int16))
    rng = np.random.default_rng(11)
    for kind in ("random", "rails"):
        x = rng.integers(-32768, 32768, (65536, 64, 2)) if kind == "random" else np.where(rng.random((65536, 64, 2)) < 0.5, -32768, 32767)
        v = cmul_q15((x.astype(np.int16) >> 1), fc)
        _, taps = check_equal("fft64", v, "rx11a " + kind)
        assert_unreachable("fft64", taps)

def test_receivers_fft_inputs():
    """What the oracle receivers hand fft64 on the full-scale captures of rail_inputs (gains up to 16, DC offsets, clipped data symbols,
    rail patterns), 802.11a and 802.11n on both antennas: the compiled reference of those inputs is what each receiver got back."""
    n11a = n11n = 0
    for rate in (6000, 54000):
        for name, cap in rail_inputs.cases_11a(rate):
            t = oracle_py.rx11a_taps(cap, max_sym=80)
            if t["nsym"] == 0: continue
            assert (oracle_py.ref_fft64(t["fft_in"]) == t["fft_out"]).all(), (rate, name)
            n11a += t["nsym"]
    for mcs in (8, 14):
        oracle_py.set_ht_mcs_limit(15)
        try:
            for name, (x0, x1) in rail_inputs.cases_11n(mcs, chans=False):
                t = oracle_py.rx11n_taps(x0, x1, max_sym=80)
                if t["fft_in"].shape[1] == 0: continue
                assert (oracle_py.ref_fft64(t["fft_in"]) == t["fft_out"]).all(), (mcs, name)
                n11n += t["fft_in"].shape[1]
        finally:
            oracle_py.set_ht_mcs_limit(11)
    assert n11a >= 100 and n11n >= 50, (n11a, n11n)

def tx_symbols():
    """The zero-stuffed IFFT<128> inputs of the three transmitters, every 802.11a rate and MCS 8..14, long random payloads (scrambled,
    so every constellation point lands in every bin): as logged from the oracle's ifft128."""
    rng = np.random.default_rng(128)
    out = {}
    for rate in (6000, 9000, 12000, 18000, 24000, 36000, 48000, 54000):
        p = rng.integers(0, 256, 1500).astype(np.uint8)
        out["tx11a %d" % rate] = oracle_py.ifft128_inputs(oracle_py.tx11a_modulate, p, rate)[1]
        out["legacy %d" % rate] = oracle_py.ifft128_inputs(oracle_py.tx11a_legacy_modulate, p, rate)[1]
    for mcs in range(8, 15):
        out["tx11n %d" % mcs] = oracle_py.ifft128_inputs(oracle_py.tx11n_modulate, rng.integers(0, 256, 1500).astype(np.uint8), mcs)[1]
    return out

def test_transmitter_domains():
    """Every logged symbol, then symbols built from each transmitter's own levels: every level pair (re, im) it used, put in every bin
    it used (one symbol per pair), and random symbols over those points."""
    rng = np.random.default_rng(3)
    for name, x in tx_symbols().items():
        assert len(x) > 10, name
        check_equal("ifft128", x, name)
        used = np.flatnonzero((x != 0).any(axis=(0, 2)))
        pts = np.unique(x[:, used].reshape(-1, 2), axis=0)
        every = np.zeros((len(pts), 128, 2), np.int16); every[:, used] = pts[:, None, :]
        rand = np.zeros((2000, 128, 2), np.int16); rand[:, used] = pts[rng.integers(0, len(pts), (2000, len(used)))]
        for fam, v in (("every point", every), ("random points", rand)):
            _, taps = check_equal("ifft128", v, name + " " + fam)
            assert_unreachable("ifft128", taps)

def sts_input():
    f = np.zeros((64, 2), np.int16); A = 10000                                           # build_sts (oracle/tables.cpp)
    for k, s in ((4, -1), (8, -1), (12, 1), (16, 1), (20, 1), (24, 1), (40, 1), (44, -1), (48, 1), (52, -1), (56, -1), (60, 1)):
        f[k] = (s * A, s * A)
    return f

def test_sts_patterns():
    """The STS input of build_sts through IFFT<64>, and the oracle's 16 cyclic patterns built from the reference's output."""
    f = sts_input()
    r = oracle_py.ref_ifft64(f[None])[0]
    assert (oracle_py.ifft64(f[None])[0] == r).all()
    pat = np.ctypeslib.as_array(oracle_py.lib().sbo_sts_pattern(), (16 * 16 * 2,)).reshape(16, 16, 2)
    want = np.stack([r[i:i + 16] for i in range(16)])
    assert (pat == want).all()

# ---- the host-compiled device sources against the reference --------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None: pytest.skip("no host compiler")
    so = str(tmp_path_factory.mktemp("fft_emu") / "fft_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-DSB_HOST_EMU", "-I", os.path.join(ROOT, "sora_b200", "csrc"),
                           "-o", so, os.path.join(ROOT, "tests", "cpp", "fft_emu.cpp")])
    L = C.CDLL(so)
    L.emu_fft64.argtypes = [C.c_int, C.c_uint64, C.c_void_p, C.c_void_p]; L.emu_ifft64.argtypes = [C.c_uint64, C.c_void_p, C.c_void_p]
    L.emu_sts.argtypes = [C.c_void_p]
    return L

def run_emu(emu, kind, x):
    x = np.ascontiguousarray(x, np.int16); o = np.zeros_like(x); n = len(x)
    if kind == "ifft64": emu.emu_ifft64(n, x.ctypes.data, o.ctypes.data)
    else: emu.emu_fft64(1 if kind == "packed" else 0, n, x.ctypes.data, o.ctypes.data)
    return o

def device_corpus(N, seed):
    fams = [("random", np.random.default_rng(seed).integers(-32768, 32768, (200_000, N, 2)).astype(np.int16))] + structured(N)
    return fams

@pytest.mark.parametrize("kind", ("scalar", "packed", "ifft64"))
def test_device_sources_equal_reference(emu, kind):
    """k_front11n's (scalar) and k_front11a's (packed) FFT<64> chains, and host_ifft64: random full-scale vectors, the structured edge
    families, the searched corpus and the 802.11a front-end domain."""
    name = "ifft64" if kind == "ifft64" else "fft64"
    fams = device_corpus(64, 77) + [("corpus", np.array(corpus()[name]))]
    if name == "fft64":
        rng = np.random.default_rng(5); fc = rng.integers(-32767, 32768, (50_000, 64, 2)).astype(np.int16)
        fams.append(("rx11a domain", cmul_q15(rng.integers(-32768, 32768, (50_000, 64, 2)).astype(np.int16) >> 1, fc)))
    else:
        fams.append(("sts", sts_input()[None]))
    for fam, x in fams:
        r = XFORMS[name][2](x); g = run_emu(emu, kind, x)
        bad = np.flatnonzero((g != r).reshape(len(x), -1).any(1))
        assert bad.size == 0, "%s %s: %d of %d vectors differ, first: x=%s ref=%s device=%s" % (kind, fam, bad.size, len(x), x[bad[0]].tolist(), r[bad[0]].tolist(), g[bad[0]].tolist())

def test_device_sts_table(emu):
    """HostTables::sts (uploaded for the device's carrier sense) equals the 16 cyclic patterns cut from the reference's IFFT<64>."""
    r = oracle_py.ref_ifft64(sts_input()[None])[0]
    got = np.zeros(256, np.uint32); emu.emu_sts(got.ctypes.data)
    got = got.view(np.int16).reshape(16, 16, 2)
    assert (got == np.stack([r[i:i + 16] for i in range(16)])).all()
