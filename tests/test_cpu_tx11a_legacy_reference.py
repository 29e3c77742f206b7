"""The legacy 802.11a transmitter of the oracle (sbo_tx11a_legacy_modulate_ex, oracle/tx11a_legacy44.cpp) against the reference's own
BB11ATxFrameMod and BB11AModulateACK, compiled from atx_*.c where they lie (oracle/build_ref_tx11a_legacy.sh -> oracle/_ref/libtx11a_legacy_ref.so),
at 40 and 44 Msps.  Every check is bit for bit: samples, the RCB zero padding and SignalLength.  No GPU; skipped without the compiled library.

The device (k_tx11a_legacy) equals the oracle on the same frames (test_gpu_tx11a_legacy_tx.py) and the compiled transmitter directly
(test_gpu_tx11a_legacy_reference.py); the committed vectors under tests/golden/legacy_tx/ and legacy_tx44/ are checked against it here."""
import os, zlib
import numpy as np, pytest
import oracle_tx11a_legacy as O

pytestmark = pytest.mark.skipif(not O.ref_tx_available(), reason="oracle/_ref/libtx11a_legacy_ref.so not built (needs the reference tree)")
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
E_FAIL = -2147467259                                                    # 0x80004005 as int32


def scrambler(n):
    """The 802.11a scrambler sequence from the all-ones state (bReg = 0xFF, atx_tpl.h:19), bytes LSB first: byte i XORs SERVICE/PSDU byte i."""
    s, out = [1] * 7, []
    for _ in range(n):
        v = 0
        for k in range(8):
            b = s[6] ^ s[3]; s = [b] + s[:6]; v |= b << k
        out.append(v)
    return np.array(out, np.uint8)


SCR = scrambler(4200)


def payload(kind, n, rng):
    """MPDU + FCS of n bytes.  'corner0' / 'corner1' scramble to all zeros / all ones, so the encoder emits constant bits and every data
    carrier sits on the same outermost constellation point: the symbol peaks that drive Copy_NT into saturation."""
    if kind == "random": return rng.integers(0, 256, n).astype(np.uint8)
    if kind == "zeros": return np.zeros(n, np.uint8)
    if kind == "ones": return np.full(n, 0xFF, np.uint8)
    if kind == "corner0": return SCR[2:2 + n].copy()
    if kind == "corner1": return SCR[2:2 + n] ^ np.uint8(0xFF)
    raise ValueError(kind)


KINDS = ("random", "zeros", "ones", "corner0", "corner1")


def boundary_lengths(kbps):
    """MPDU lengths on both sides of symbol boundaries: the last length of n symbols and the first of n + 1, for n over the whole range
    (both parities of the 9 Mbps symbol count among them)."""
    nd = O.NDBPS[kbps]; out = set()
    for s in list(range(1, 40)) + list(range(40, O.nsym(4096, kbps) + 1, 17)):
        last = (s * nd - 22) // 8 - 4                                   # the largest MPDU (FCS excluded) that fits s symbols
        for n in (last, last + 1):
            if 0 <= n <= 4092: out.add(n)
    return sorted(out)


def check(psdu, kbps, sr, ctx=None):
    got = O.ref_modulate(psdu, kbps, sr, ctx)
    want = O.modulate(psdu, kbps, sr, append_crc=False)
    assert got.shape == want.shape, (kbps, sr, len(psdu), got.shape, want.shape)
    bad = np.flatnonzero((got != want).any(axis=1))
    assert bad.size == 0, (kbps, sr, len(psdu), bad[:8])
    return len(got)


FRAMES = {}


@pytest.mark.parametrize("sr", [40, 44])
@pytest.mark.parametrize("kbps", O.RATES)
def test_whole_frames(kbps, sr):
    """Every PacketSize 0..64, a sweep to 4092 (LENGTH 4096, the parity-bit case), both sides of symbol boundaries, frames of more than 127
    data symbols (the pilot index wraps), random / 0x00 / 0xFF / corner payloads, and an FCS that is not the frame's CRC."""
    rng = np.random.default_rng(kbps * 7 + sr)
    lens = sorted(set(range(65)) | set(range(65, 4093, 97)) | {4092, 4091} | set(boundary_lengths(kbps)))
    assert O.nsym(4096, kbps) > 127
    n = 0
    for i, m in enumerate(lens):
        psdu = payload(KINDS[i % len(KINDS)], m + 4, rng)
        if i % 3 == 0: psdu[-4:] = np.frombuffer(zlib.crc32(bytes(psdu[:-4])).to_bytes(4, "little"), np.uint8)
        check(psdu, kbps, sr); n += 1
    for m in (3429, 4092):                                              # every kind at lengths past the pilot wrap
        for k in KINDS:
            check(payload(k, m + 4, rng), kbps, sr); n += 1
    FRAMES[(kbps, sr)] = n


def test_golden_vectors_are_the_compiled_transmitter():
    """tests/golden/legacy_tx/legacy_tx_<kbps>.i8 (MPDU .bin + CRC-32, 40 Msps), ofdm.bin (the reference's own capture: 200 bytes of 0x31
    at 24 Mbps) and, where committed, the 44 Msps vectors of tests/golden/legacy_tx44/."""
    for kbps in O.RATES:
        body = np.fromfile(os.path.join(GOLD, "legacy_tx", f"legacy_tx_{kbps}.bin"), np.uint8)
        want = np.fromfile(os.path.join(GOLD, "legacy_tx", f"legacy_tx_{kbps}.i8"), np.int8).reshape(-1, 2)
        psdu = np.concatenate([body, np.frombuffer(zlib.crc32(bytes(body)).to_bytes(4, "little"), np.uint8)])
        got = O.ref_modulate(psdu, kbps, 40)
        assert len(want) <= len(got) and (got[:len(want)] == want).all(), kbps
        p44 = os.path.join(GOLD, "legacy_tx44", f"legacy_tx44_{kbps}.i8")
        if os.path.exists(p44):
            b44 = np.fromfile(os.path.join(GOLD, "legacy_tx44", f"legacy_tx44_{kbps}.bin"), np.uint8)
            w44 = np.fromfile(p44, np.int8).reshape(-1, 2)
            assert (O.ref_modulate(b44, kbps, 44) == w44).all(), kbps
    ref = np.fromfile(os.path.join(GOLD, "ofdm.bin"), np.int8).reshape(-1, 2)
    body = np.full(200, 0x31, np.uint8)
    psdu = np.concatenate([body, np.frombuffer(zlib.crc32(bytes(body)).to_bytes(4, "little"), np.uint8)])
    assert (O.ref_modulate(psdu, 24000, 40)[:3680] == ref[:3680]).all()


def test_preamble_fixture_is_the_compiled_table():
    """tests/golden/preamble40_11a.i16, what callers hand BB11ATxSetPreamble, is lutst/preamble40_11a.c's PREAMBLE40_11A_LUT."""
    assert (O.preamble() == O.ref_preamble()).all()


@pytest.mark.parametrize("sr", [40, 44])
def test_mdl_chains(sr):
    """Scramble11a walks the MDL chain (StartVa + ByteOffset, ByteCount, Next): one PSDU split over 1-4 MDLs, with non-zero ByteOffsets
    and a zero-length MDL, is the frame of one MDL."""
    rng = np.random.default_rng(sr)
    for m in (0, 1, 30, 777, 4092):
        psdu = rng.integers(0, 256, m + 4).astype(np.uint8); mpdu, fcs = psdu[:-4], int.from_bytes(bytes(psdu[-4:]), "little")
        want = O.modulate(psdu, 18000, sr, append_crc=False)
        a, b = sorted(rng.integers(0, m + 1, 2))
        empty = mpdu[:0]
        for parts in ([mpdu], [mpdu[:a], mpdu[a:]], [mpdu[:a], empty, mpdu[a:]], [mpdu[:a], mpdu[a:b], empty, mpdu[b:]]):
            assert sum(p.size for p in parts) == m
            hr, out, sl = O.ref_frame_mod_raw(parts, fcs, O.CODE[18000], sr, offsets=[3 + 5 * i for i in range(len(parts))])
            assert hr == 0 and sl == 2 * len(want) and (out[:sl].view(np.int8).reshape(-1, 2) == want).all(), (m, [p.size for p in parts])


def test_context_reuse():
    """Back-to-back frames on one BB11A_TX_VECTOR, at changing rates and sample rates, equal frames made on fresh contexts: nothing a frame
    leaves in the context (the window, the encoder register, cSymbol44M, the scrambled bytes) reaches the next."""
    rng = np.random.default_rng(11)
    ctx = O.RefContext()
    for i in range(60):
        kbps = O.RATES[rng.integers(0, 8)]; sr = (40, 44)[rng.integers(0, 2)]
        psdu = payload(KINDS[i % len(KINDS)], int(rng.integers(4, 1600)), rng)
        assert (O.ref_modulate(psdu, kbps, sr, ctx) == O.ref_modulate(psdu, kbps, sr)).all(), (i, kbps, sr)
        check(psdu, kbps, sr, ctx)


@pytest.mark.parametrize("sr", [40, 44])
def test_ack(sr):
    """BB11AModulateACK: a 14-byte ACK (FC 0xD4 0x00, Duration 0, RA, CRC-32) through BB11ATxBufferMod6M at 6 Mbps, although it sets
    ti_uiDataRate to 24 Mbps; it returns the padded signal length in bytes."""
    rng = np.random.default_rng(sr)
    for ra in ([0] * 6, [0xFF] * 6, list(range(0x10, 0x16)), list(rng.integers(0, 256, 6)), list(rng.integers(0, 256, 6))):
        n, buf = O.ref_ack(np.array(ra, np.uint8), sr)
        want = O.modulate(O.ack_frame(ra), 6000, sr, append_crc=False)
        assert n == 2 * len(want) == 2 * O.padded_samples(14, 6000, sr)
        assert (buf[:n].view(np.int8).reshape(-1, 2) == want).all() and (buf[n:] == 0x55).all()
        assert (O.ref_modulate(O.ack_frame(ra), 6000, sr) == want).all()


def test_preamble_over_read_reaches_one_output():
    """At 44 Msps CopyPreamble16_NT's fourth chunk loads one vector past PREAMBLE40_11A_LUT; the library reads zeros there (DESIGN.md §1).
    With anything else behind the table exactly one output changes, output 175 of that chunk (sample 703), and nothing at 40 Msps."""
    rng = np.random.default_rng(4)
    psdu = rng.integers(0, 256, 300).astype(np.uint8)
    base = {sr: O.ref_modulate(psdu, 54000, sr) for sr in (40, 44)}
    try:
        for pad in (np.full((8, 2), 20000, np.int16), rng.integers(-32768, 32768, (8, 2)).astype(np.int16)):
            O.ref_set_pad(pad)
            got = O.ref_modulate(psdu, 54000, 44)
            assert list(np.flatnonzero((got != base[44]).any(axis=1))) == [3 * 176 + 175]
            assert (O.ref_modulate(psdu, 54000, 40) == base[40]).all()
            pad4 = np.concatenate([O.preamble()[480:], pad[:4]])       # the chunk with that vector behind it, by the upsampler readings
            assert got[703, 0] == np.clip(O.up160_numpy(pad4)[175] >> 6, -128, 127)[0]
    finally:
        O.ref_set_pad(np.zeros((8, 2), np.int16))
    assert (O.ref_modulate(psdu, 54000, 44) == base[44]).all()


def test_refusals():
    """E_FAIL and nothing written for a rate code that is not an 802.11a rate and for PacketSize + 4 > INPUT_MAX (atx_fe.c:20-27, :56-60)."""
    for parts, code in (([np.zeros(10, np.uint8)], 0x7), ([np.zeros(4093, np.uint8)], O.CODE[6000])):
        hr, out, sl = O.ref_frame_mod_raw(parts, 0, code, 40)
        assert hr == E_FAIL and sl == 0 and (out == 0x55).all()


def test_counters_reached():
    """The debug tap over a corpus of every rate, both sample rates and every payload kind: Copy_NT's int8 pack saturates (corner payloads
    put every data carrier on one outermost point); IFFT64x's << 2 never loses bits (DESIGN.md §7 (f) rank 4: IFFT peak below 6480 < 8192)
    and Window's saturating add never clips (|x| <= 4 * 6480 per sample, and the window's weights sum to one per output)."""
    rng = np.random.default_rng(21)
    O.ref_debug_reset()
    for kbps in O.RATES:
        for sr in (40, 44):
            for k in KINDS:
                for m in (1, 100, 1500):
                    O.ref_modulate(payload(k, m + 4, rng), kbps, sr)
    d = O.ref_debug()
    print("tap:", d, "frames per (rate, sample rate):", FRAMES)
    assert d["pack_sat"] > 0
    assert d["ifft_shl_loss"] == 0 and d["window_sat"] == 0
