"""The 802.11a transmit oracle (oracle/tx11a.cpp) against the reference's own compiled modulator bricks and graphs (oracle/build_ref_mod.sh):
the scrambler, the three convolutional encoders, the four interleavers, the four mappers, the pilot inserter, TIFFTx and the 16 -> 8 bit
pack one by one, then whole frames through CreatePreamble11a_40M and CreateModGraph11a_40M driven as Test11A_FB_Mod drives them.  Bit for
bit.  No GPU.  The library's debug tap shows that the corpus reaches the edges: pack saturation, the 9 Mbps symbol-pair padding and the
frames whose padding adds a symbol beyond the standard's N_SYM."""
import numpy as np, pytest
import oracle_py

pytestmark = pytest.mark.skipif(not oracle_py.ref_mod_available(), reason="oracle/_ref/libmod_ref.so not built (oracle/build_ref_mod.sh)")

RATES_11A = (6000, 9000, 12000, 18000, 24000, 36000, 48000, 54000)
SEEDS = (0x01, 0x5D, 0x7F, 0xFF)
# every length 1-64, then a sweep to the largest frame (LENGTH = 4091 + 4 FCS bytes = 4095)
LENGTHS = tuple(range(1, 65)) + tuple(range(65, 4091, 331)) + (1500, 2304, 4090, 4091)

def _bits(b):
    return np.unpackbits(np.ascontiguousarray(b, np.uint8), bitorder="little")
def _bytes(bits):
    return np.packbits(np.ascontiguousarray(bits, np.uint8), bitorder="little")

def _std_nsym(length, rate):
    ndbps = rate // 250
    return -(-(16 + 8 * (length + 4) + 6) // ndbps)
def _nsym_over_standard(rate):
    """The lengths 1 .. 4091 whose transmitted symbol count exceeds the standard's N_SYM at this rate (the tail counted as a whole byte;
    at 9 Mbps also the symbol pair), as the oracle counts symbols."""
    L = oracle_py.lib()
    return [n for n in range(1, 4092) if L.sbo_tx11a_nsym(n, rate) > _std_nsym(n, rate)]

# ---- stages ----
def test_scrambler_equals_the_reference_at_every_seed():
    data = np.tile(np.arange(256, dtype=np.uint8), 3)
    rng = np.random.default_rng(1)
    ctrls = (np.ones(data.size, np.uint8), rng.integers(0, 3, data.size).astype(np.uint8),
             np.r_[np.zeros(3, np.uint8), np.ones(data.size - 5, np.uint8), 2, 1].astype(np.uint8))     # SIGNAL, DATA, tail, pad
    for seed in range(256):
        for ctrl in ctrls:
            a = oracle_py.tx11a_scramble(data, ctrl, seed); b = oracle_py.ref_mod11a_scramble(data, ctrl, seed)
            assert (a == b).all(), (seed, np.nonzero(a != b)[0][:8])

def _all_pairs():
    """Every (previous byte, byte) pair as consecutive bytes: each byte is encoded from every encoder state (the state after a byte is
    its top six bits), and the stream's length is a multiple of 6 so that every puncturing burst is whole."""
    a, b = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8), indexing="ij")
    return np.stack([a.ravel(), b.ravel()], 1).ravel()[:131070]

@pytest.mark.parametrize("cr", (0, 1, 2))
def test_encoders_equal_the_reference_on_every_state_and_byte(cr):
    x = _all_pairs()
    got = _bytes(oracle_py.tx11a_encode_bits(x, cr)); want = oracle_py.ref_mod11a_encode(cr, x)
    assert got.size == want.size and (got == want).all(), (cr, np.nonzero(got != want)[0][:8])
    y = np.random.default_rng(2).integers(0, 256, 6000).astype(np.uint8)
    assert (_bytes(oracle_py.tx11a_encode_bits(y, cr)) == oracle_py.ref_mod11a_encode(cr, y)).all()

@pytest.mark.parametrize("nbpsc", (1, 2, 4, 6))
def test_interleavers_equal_the_reference_on_every_row(nbpsc):
    n = 48 * nbpsc
    onehot = np.eye(n, dtype=np.uint8)                                      # every input bit on its own: where each row goes
    rnd = np.random.default_rng(3).integers(0, 2, (500, n)).astype(np.uint8)
    for bits in (onehot, rnd, np.ones((1, n), np.uint8)):
        got = oracle_py.tx11a_interleave(bits, nbpsc)
        want = _bits(oracle_py.ref_mod11a_interleave(nbpsc, _bytes(bits.ravel()).reshape(len(bits), -1))).reshape(len(bits), n)
        assert (got == want).all(), (nbpsc, np.argwhere(got != want)[:8])

@pytest.mark.parametrize("nbpsc", (1, 2, 4, 6))
def test_mappers_equal_the_reference_at_every_index(nbpsc):
    if nbpsc == 6:                                                            # 12-bit indices, two per 3-byte burst: all 4096 of each slot
        i = np.arange(4096); j = 4095 - i
        raw = np.stack([i & 0xFF, (i >> 8) | ((j & 0xF) << 4), j >> 4], 1).astype(np.uint8).ravel()
    else:
        raw = np.arange(256, dtype=np.uint8)
    per = 6 * nbpsc
    raw = np.r_[raw, np.zeros(-raw.size % per, np.uint8)].astype(np.uint8)
    got = oracle_py.tx11a_map(_bits(raw).reshape(-1, 48 * nbpsc), nbpsc).reshape(-1, 2)
    want = oracle_py.ref_mod11a_map(nbpsc, raw)
    assert got.shape == want.shape and (got == want).all(), (nbpsc, np.argwhere(got != want)[:8])

def test_pilot_inserter_equals_the_reference():
    rng = np.random.default_rng(4)
    d = rng.integers(-32768, 32768, (300, 48, 2)).astype(np.int16)           # 300 symbols: the pilot index wraps twice
    assert (oracle_py.tx11a_add_pilot(d) == oracle_py.ref_mod11a_add_pilot(d)).all()

def _spectra():
    rng = np.random.default_rng(5)
    yield rng.integers(-32768, 32768, (400, 64, 2)).astype(np.int16)         # random, full range
    yield rng.integers(-12000, 12000, (400, 64, 2)).astype(np.int16)
    lv = np.array([10720, -10720, 7581, -7581, 3390 * 3, -3390 * 3, 1654 * 7, -1654 * 7], np.int16)   # the mappers' corner levels
    yield rng.choice(lv, (400, 64, 2)).astype(np.int16)
    rails = np.where(rng.random((200, 64, 2)) < 0.5, -32768, 32767).astype(np.int16)
    yield rails                                                               # rails: the IFFT and the pack saturate
    yield np.stack([np.full((64, 2), v, np.int16) for v in (32767, -32768, 10720, -1, 0)])
    e = np.zeros((64, 64, 2), np.int16); e[np.arange(64), np.arange(64), 0] = 32767; yield e   # one carrier at a time

def test_ifftx_equals_the_reference():
    for x in _spectra():
        a = oracle_py.tx11a_ifftx(x); b = oracle_py.ref_mod11a_ifftx(x)
        assert (a == b).all(), np.argwhere(a != b)[:8]

def test_pack_equals_the_reference():
    rng = np.random.default_rng(6)
    edges = np.array([-32768, -32767, -129, -128, -127, -1, 0, 1, 126, 127, 128, 255, 256, 32767], np.int16)
    for x in (rng.integers(-32768, 32768, (8000, 2)), rng.integers(-300, 300, (8000, 2)), np.tile(edges, 8).reshape(-1, 2),
              oracle_py.tx11a_ifftx(next(_spectra())).reshape(-1, 2)):
        x = np.ascontiguousarray(x, np.int16)
        assert (oracle_py.tx11a_pack8(x) == oracle_py.ref_pack16to8(x)).all()

# ---- whole frames ----
def _frame_equal(p, rate, seed):
    want = oracle_py.ref_mod11a_frame(p, rate, seed)
    got = oracle_py.tx11a_modulate(p, rate, seed, tail_zeros=0)
    assert got.shape == want.shape, (rate, len(p), seed, got.shape, want.shape)
    assert (got == want).all(), (rate, len(p), seed, np.argwhere(got != want)[:4])

@pytest.mark.parametrize("rate", RATES_11A)
def test_frames_equal_the_reference(rate):
    rng = np.random.default_rng(rate)
    for i, n in enumerate(LENGTHS):
        _frame_equal(rng.integers(0, 256, n).astype(np.uint8), rate, SEEDS[i % len(SEEDS)])

def _boundary_lengths(rate):
    """Lengths on both sides of the standard's symbol boundaries, the lengths whose symbol count exceeds the standard's N_SYM (none at
    the rates whose N_DBPS is a whole number of bytes: the tail byte then never crosses a boundary), and at 9 Mbps both parities of N_SYM."""
    over = _nsym_over_standard(rate)
    edge = [n for n in range(2, 4092) if _std_nsym(n, rate) != _std_nsym(n - 1, rate)]
    pick = over[:6] + over[len(over) // 2:len(over) // 2 + 3] + over[-3:]
    for n in edge[:4] + edge[len(edge) // 2:len(edge) // 2 + 2] + edge[-2:]:
        pick += [n - 1, n]
    if rate == 9000:
        assert over
        pick += [n for n in range(1, 200) if _std_nsym(n, rate) % 2 == 0][:5] + [n for n in range(1, 200) if _std_nsym(n, rate) % 2][:5]
    return pick

@pytest.mark.parametrize("rate", RATES_11A)
def test_frames_at_symbol_boundaries(rate):
    rng = np.random.default_rng(rate + 1)
    for n in _boundary_lengths(rate):
        _frame_equal(rng.integers(0, 256, n).astype(np.uint8), rate, 0x5D)

def test_frames_at_every_seed_and_constant_payloads():
    for seed in range(0, 256, 17):
        _frame_equal(np.full(100, 0xFF, np.uint8), 54000, seed)
        _frame_equal(np.zeros(37, np.uint8), 6000, seed)

def test_preamble_table_equals_the_reference():
    """The oracle's TTS11aSrc table through the pack equals the compiled preamble graph's 640 samples (the first 640 of any frame)."""
    want = oracle_py.ref_mod11a_frame(np.zeros(1, np.uint8), 6000)[:640]
    assert (oracle_py.tx11a_modulate(np.zeros(1, np.uint8), 6000, 0xFF, 0)[:640] == want).all()

def test_counters_reached():
    """The corpus above reaches each edge the tap counts: the spectra of test_ifftx through the compiled TIFFTx and pack (pack lanes that
    saturate), and the lengths of test_frames_at_symbol_boundaries through the compiled graphs (the 9 Mbps symbol
    pair and symbols beyond N_SYM, both read from what the graph wrote)."""
    oracle_py.ref_mod_debug_reset()
    for x in _spectra():
        oracle_py.ref_pack16to8(oracle_py.ref_mod11a_ifftx(x).reshape(-1, 2))
    for rate in RATES_11A:
        rng = np.random.default_rng(rate + 1)
        for n in _boundary_lengths(rate):
            oracle_py.ref_mod11a_frame(rng.integers(0, 256, n).astype(np.uint8), rate, 0x5D)
    d = oracle_py.ref_mod_debug()
    assert all(v > 0 for v in d.values()), d
