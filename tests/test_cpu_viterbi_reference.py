"""The K=7 Viterbi against the reference's OWN code: T11aViterbi<...>::Filter, TViterbiCore and Viterbi_sig11 compiled from
kernel/bb/Brick11/src where they lie (oracle/build_ref_viterbi.sh -> oracle/_ref/libviterbi_ref.so).  Every other Viterbi test compares
with oracle/viterbi.cpp, a restatement of those headers; here the restatement and the host-compiled device source of both kernels
(tests/cpp/lane_emu.cpp, re_emu.cpp) must equal the compiled reference byte for byte: every code rate, each of the three instantiations
the reference ships (802.11a 48 / 256 / 24, 802.11n 312 / 192 / 36, the short 48 / 24 / 24 window), frame lengths from 1 to 4095 and
every position of the flush point in a 6-step chunk and a puncture group, clean, noisy and adversarial soft values, and the SIGNAL
decoder on random and real SIGNAL words.  The GPU side of the same comparison is tests/test_gpu_zz_viterbi_reference.py."""
import ctypes as C, shutil
import numpy as np, pytest
import oracle_py
from sora_b200 import synth

CR_12, CR_23, CR_34 = 0, 1, 2
GROUPS = {CR_12: (2, 1), CR_23: (3, 2), CR_34: (4, 3)}          # soft values and trellis steps per puncture group
RATES = {CR_12: (1, 2), CR_23: (2, 3), CR_34: (3, 4)}
INSTS = oracle_py.REF_VITERBI_INSTS                              # inst -> (N_INPUT, depth, lookahead)
LENGTHS = (1, 2, 3, 100, 1500, 4095)
FLUSH_LENGTHS = tuple(range(4, 16))                              # 8 L + 22 at every even offset of a 6-step chunk, every offset of a group
# One period of 32 soft values (a rate-3/4 normalisation period: 8 groups, 24 steps), found by hill-climbing the largest metric the
# reference's Normalize sees: tiled, it keeps every path metric near 200 at each normalisation, far above 127 (a signed byte or 16-bit
# compare would go wrong there) though below 256: with 3-bit soft values the best path grows by at most 29 per group, and the measured
# largest metric at a normalisation, over all searches, is 204.
HIGH_METRIC = np.array([int(c) for c in "43333343444344434344334343433433"], np.uint8)

pytestmark = pytest.mark.skipif(not oracle_py.ref_viterbi_available(), reason="oracle/_ref/libviterbi_ref.so not built (needs the reference tree)")

def nsoft_for(inst, cr, L, extra_groups=0):
    """Soft values for a frame of L bytes: enough whole groups to reach the flush point 8 L + 22, plus extra_groups, rounded up to whole
    N_INPUT bursts (so every decoder sees the same groups)."""
    ni = INSTS[inst][0]; per, st = GROUPS[cr]
    ns = (-(-(8 * L + 22) // st) + extra_groups) * per
    ns = -(-ns // ni) * ni
    assert ns // per * st < oracle_py.REF_TRELLIS_MAX
    return ns

def families(rng, cr, L, ns, nflip=(0.02, 0.08, 0.2)):
    """(name, soft row of ns values): a clean code word, the same word at several flip rates, uniform noise over 0..7, all 0, all 7,
    0 / 7 alternating per coded bit, and the tiled high-metric period."""
    per, st = GROUPS[cr]
    nbits = ns // per * st
    bits = rng.integers(0, 2, nbits).astype(np.uint8); bits[8 * L + 16:] = 0
    A, B = synth.conv_encode(bits)
    coded = synth.puncture(A, B, RATES[cr])[:ns]
    clean = np.where(coded > 0, rng.integers(5, 8, ns), rng.integers(0, 3, ns)).astype(np.uint8)
    out = [("clean", clean)]
    for f in nflip:
        out.append(("flip%g" % f, np.where(rng.random(ns) < f, 7 - clean, clean).astype(np.uint8)))
    out += [("noise", rng.integers(0, 8, ns).astype(np.uint8)), ("zeros", np.zeros(ns, np.uint8)), ("sevens", np.full(ns, 7, np.uint8)),
            ("alt07", np.tile(np.array([0, 7], np.uint8), ns)[:ns]), ("high", np.tile(HIGH_METRIC, ns // 32 + 1)[:ns])]
    return out, bits

def oracle_block(inst, soft, cr, L):
    _, depth, look = INSTS[inst]
    return oracle_py.viterbi_block(soft, cr, L, depth, look)

@pytest.mark.parametrize("inst", sorted(INSTS))
@pytest.mark.parametrize("cr", (CR_12, CR_23, CR_34))
def test_blocks_equal_oracle(inst, cr):
    """oracle viterbi_decode_block == the compiled T11aViterbi Filter, byte for byte, on every input family and frame length."""
    rng = np.random.default_rng(100 * inst + cr)
    for L in LENGTHS + FLUSH_LENGTHS:
        ns = nsoft_for(inst, cr, L, extra_groups=int(rng.integers(0, 9)))
        rows, bits = families(rng, cr, L, ns, nflip=(0.05,) if L >= 1500 else (0.02, 0.08, 0.2))
        for name, soft in rows:
            ref = oracle_py.ref_viterbi_block(inst, soft, cr, L)
            assert len(ref) == L + 2, (inst, cr, L, name, len(ref))
            o = oracle_block(inst, soft, cr, L)
            assert len(o) == len(ref) and (o == ref).all(), (inst, cr, L, name, np.argwhere(o != ref)[:4] if len(o) == len(ref) else len(o))
            if name == "clean":
                assert (np.unpackbits(ref, bitorder="little")[:8 * L + 16] == bits[:8 * L + 16]).all(), (inst, cr, L)

@pytest.mark.parametrize("cr", (CR_12, CR_23, CR_34))
def test_short_input_and_partial_bursts(cr):
    """Soft values that end before the flush point (a truncated frame): the Filter emits only the windows it could trace back, and the
    oracle fed the same whole bursts emits the same bytes."""
    rng = np.random.default_rng(7 + cr)
    for inst in sorted(INSTS):
        ni = INSTS[inst][0]
        for L in (100, 1500):
            full = nsoft_for(inst, cr, L)
            for ns in sorted({ni, full // 2 // ni * ni, full - ni}):
                soft = rng.integers(0, 8, ns).astype(np.uint8)
                ref = oracle_py.ref_viterbi_block(inst, soft, cr, L)
                o = oracle_block(inst, soft, cr, L)
                assert len(o) == len(ref) and (o == ref).all(), (inst, cr, L, ns, len(o), len(ref))

def test_high_metric_pattern_reaches_the_top_byte_range():
    """The high-metric period really drives the reference's path metrics above 127 at rate 3/4 (what the harness's Normalize tap saw,
    unwrapped), and, as 3-bit soft values allow, no further than 255; uniform noise stays far lower."""
    for inst in sorted(INSTS):
        ns = nsoft_for(inst, CR_34, 300)
        soft = np.tile(HIGH_METRIC, ns // 32 + 1)[:ns]
        ref, (max_min, max_any) = oracle_py.ref_viterbi_block(inst, soft, CR_34, 300, debug=True)
        assert 192 <= max_min <= max_any < 256, (inst, max_min, max_any)
        assert (oracle_block(inst, soft, CR_34, 300) == ref).all()
        _, (nmin, nany) = oracle_py.ref_viterbi_block(inst, np.random.default_rng(1).integers(0, 8, ns).astype(np.uint8), CR_34, 300, debug=True)
        assert nany < 180, (inst, nmin, nany)

def _signal_soft(rng, word, flips):
    bits = np.array([(word >> i) & 1 for i in range(24)], np.uint8)
    A, B = synth.conv_encode(bits)
    coded = synth.puncture(A, B, (1, 2))
    soft = np.where(coded > 0, rng.integers(5, 8, 48), rng.integers(0, 3, 48)).astype(np.uint8)
    idx = rng.choice(48, flips, replace=False); soft[idx] = 7 - soft[idx]
    return soft

def test_signal_equals_oracle():
    """Viterbi_sig11 (with T11aViterbiSig's >> 6) == the oracle's viterbi_signal on 20 000 random 48-value vectors, all 0, all 7, and
    the SIGNAL words of all eight rates at several lengths with 0..6 flipped soft values; clean words decode to themselves."""
    rng = np.random.default_rng(48)
    L = oracle_py.lib(); L.sbo_viterbi_signal.argtypes = [C.c_void_p]
    vecs = list(rng.integers(0, 8, (20000, 48)).astype(np.uint8)) + [np.zeros(48, np.uint8), np.full(48, 7, np.uint8)]
    words = []
    for code in (0xB, 0xF, 0xA, 0xE, 0x9, 0xD, 0x8, 0xC):
        for length in (1, 14, 100, 1500, 2304, 4095):
            w = code | (length << 5); w |= (bin(w).count("1") & 1) << 17
            words.append(w)
            for flips in range(7):
                vecs.append(_signal_soft(rng, w, flips))
            clean = _signal_soft(rng, w, 0)
            assert oracle_py.ref_viterbi_sig11(clean) == w, hex(w)
    for v in vecs:
        v = np.ascontiguousarray(v)
        assert oracle_py.ref_viterbi_sig11(v) == L.sbo_viterbi_signal(v.ctypes.data), v

# ---- the host-compiled device source of both kernels against the compiled reference ------------------------------------------------
@pytest.fixture(scope="module")
def emus(tmp_path_factory):
    if shutil.which("g++") is None: pytest.skip("no host compiler")
    import test_cpu_lane_emu, test_cpu_re_emu
    return {"lane": test_cpu_lane_emu.build_emu(tmp_path_factory), "re": test_cpu_re_emu.build_emu(tmp_path_factory)}

@pytest.mark.parametrize("kernel", ("lane", "re"))
@pytest.mark.parametrize("cr", (CR_12, CR_23, CR_34))
def test_kernel_emulations_equal_reference(emus, kernel, cr):
    """Every input family, as one batch of code blocks per frame length, through the emulated kernel at each instantiation's window."""
    rng = np.random.default_rng(200 + cr)
    for inst in sorted(INSTS):
        _, depth, look = INSTS[inst]
        for L in (1, 3, 100, 7, 10, 13) if inst != 1 else (2, 100, 9, 14):
            ns = nsoft_for(inst, cr, L, extra_groups=int(rng.integers(0, 5)))
            rows, _ = families(rng, cr, L, ns)
            soft = np.stack([r for _, r in rows])
            g, nraw = emus[kernel](soft, cr, L, depth, look)
            for i, (name, r) in enumerate(rows):
                ref = oracle_py.ref_viterbi_block(inst, r, cr, L)
                assert nraw[i] == len(ref) == L + 2 and (g[i] == ref).all(), (kernel, inst, cr, L, name, np.argwhere(g[i] != ref)[:4])
