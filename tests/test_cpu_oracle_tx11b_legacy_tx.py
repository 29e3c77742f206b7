"""The legacy 802.11b transmitter (BB11BPMDBufferTx4XWith{Long,Short}Header, kernel/bb/dot11b/bbb_tx.c) — the restatement in
oracle_tx11b_legacy.py against the reference's own compiled encoder (oracle/_ref/libtx11b_legacy_ref.so, built by oracle/build_ref_tx11b.sh;
skipped where it is absent), against the known answers the reference ships (TestModAck, kernel/bb/demod11/modulate11b.cpp:100-165), and
through the 802.11b receive oracle."""
import os, sys, zlib, numpy as np, pytest
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import oracle_py
import oracle_tx11b_legacy as O
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RATES = [1000, 2000, 5500, 11000]
needs_ref = pytest.mark.skipif(not O.ref_available(), reason="oracle/_ref/libtx11b_legacy_ref.so not built (needs the reference tree)")


def ack_psdu():
    """TestModAck's frame: an ACK (frame control 0xD4) to 00:14:6c:e2:00:e5, duration 0, and its FCS."""
    ack = bytes([0xD4, 0x00, 0x00, 0x00, 0x00, 0x14, 0x6C, 0xE2, 0x00, 0xE5])
    return np.frombuffer(ack + zlib.crc32(ack).to_bytes(4, "little"), np.uint8)


def test_reference_known_answer_for_the_encoder():
    """modulate11b.cpp:145-150: the 2 Mbps short-preamble ACK's encoder output has CRC-32 0xaca87240 (6 784 COMPLEX8 samples)."""
    enc, _ = O.encode(ack_psdu(), 2000, short_preamble=True)
    assert len(enc) == 6784 and zlib.crc32(enc.tobytes()) == 0xACA87240


def test_reference_known_answer_for_the_filter_is_the_assembly_body():
    """modulate11b.cpp:151-163 checks the filtered ACK against CRC-32 0xfdf0c0fc and its last 512 bytes against temp[] (tests/golden/
    tx11b_legacy/ack_fir_tail.bin).  Those constants were made by the inline-assembly body (BB11BPMDSpreadFIR4ASM, variant 1); the intrinsic
    body that BB11BPMDSpreadFIR4SSE compiles to on x64 (variant 0) gives 0x81583a77 and differs in the tail."""
    enc, _ = O.encode(ack_psdu(), 2000, short_preamble=True)
    tail = np.fromfile(os.path.join(GOLD, "tx11b_legacy", "ack_fir_tail.bin"), np.uint8)
    asm = oracle_py.fir37_legacy(enc, 1).tobytes()
    assert zlib.crc32(asm) == 0xFDF0C0FC and asm[-512:] == tail.tobytes()
    sse = oracle_py.fir37_legacy(enc, 0).tobytes()
    assert zlib.crc32(sse) == 0x81583A77 and sse[-512:] != tail.tobytes()


@needs_ref
def test_regenerated_tables_equal_the_compiled_tables():
    T = O.tables()
    def packed(v, nr):                                    # the LUT_ELEMENT_* layout: Values[] then bNewRef, byte-packed
        vv = v.reshape(*nr.shape, -1)
        return np.concatenate([vv.view(np.uint8), nr[..., None]], axis=-1).ravel()
    assert (O.ref_table(0) == T["scr"].ravel()).all()
    assert (O.ref_table(5).view(np.uint16) == T["crc16"]).all()
    assert (O.ref_table(1) == packed(*T["dbpsk"])).all()
    assert (O.ref_table(2) == packed(*T["dqpsk"])).all()
    assert (O.ref_table(3) == packed(*T["cck5"])).all()
    assert (O.ref_table(4) == packed(*T["cck11"])).all()


def cases(seed):
    rng = np.random.default_rng(seed)
    for n in range(0, 65):
        yield rng.integers(0, 256, n + 4).astype(np.uint8)
    for n in (1499, 1500, 2047, 4090, 4091):             # odd and even CCK-11 byte counts up to the largest PSDU
        yield rng.integers(0, 256, n + 4).astype(np.uint8)
    for n in rng.integers(65, 4092, 6):
        yield rng.integers(0, 256, int(n) + 4).astype(np.uint8)


@needs_ref
@pytest.mark.parametrize("short", [False, True])
@pytest.mark.parametrize("rate", RATES)
def test_restatement_equals_the_compiled_encoder(rate, short):
    for psdu in cases(rate + short):
        a, sa = O.encode(psdu, rate, short)
        b, sb = O.ref_encode(psdu, rate, short)
        assert a.shape == b.shape and (a == b).all(), (rate, short, len(psdu))
        assert (sa == sb).all()                            # the bytes the reference leaves scrambled in the caller's buffer


@pytest.mark.parametrize("short", [False, True])
@pytest.mark.parametrize("rate", RATES)
def test_frame_layout(rate, short):
    """Length = 4 x chips + 37 zeros rounded up to 128; every fourth sample carries a chip; short preamble at 1 Mbps stops after the header."""
    psdu = np.arange(104, dtype=np.uint8)
    enc, scr = O.encode(psdu, rate, short)
    cpb = {1000: 0 if short else 88, 2000: 44, 5500: 16, 11000: 8}[rate]
    chips = (9 * 88 + 6 * 44 if short else 24 * 88) + len(psdu) * cpb
    assert len(enc) % 128 == 0 and len(enc) >= 4 * chips + 37 and len(enc) - 128 < 4 * chips + 37
    assert (enc[1:4 * chips:4] == 0).all() and (enc[2:4 * chips:4] == 0).all() and (enc[3:4 * chips:4] == 0).all() and (enc[4 * chips:] == 0).all()
    assert (np.abs(enc[:4 * chips:4].astype(int)).max(axis=1) >= 127).all()
    assert len(scr) == len(psdu) and (scr != psdu).any()


@pytest.mark.parametrize("rate", RATES)
def test_long_preamble_round_trip_through_the_receive_oracle(rate):
    """Legacy long-preamble TX with the SSE filter -> COMPLEX16 -> the 802.11b receive oracle returns the payload (the receiver delivers
    frame_length - 1 bytes, the FCS's last byte is never delivered).  The short preamble has no receiver in the reference."""
    rng = np.random.default_rng(rate)
    for n in (1, 77, 300):
        pay = rng.integers(0, 256, n).astype(np.uint8)
        y = O.modulate(pay, rate, short_preamble=False, filt=1)
        iq = np.ascontiguousarray(np.concatenate([np.zeros((280, 2), np.int16), y.astype(np.int16) << 8, np.zeros(((-len(y) - 280) % 28 + 56, 2), np.int16)]))
        res, out = oracle_py.rx11b_batch(iq, np.zeros(1, np.uint64), np.array([len(iq)], np.uint32))
        assert res[0]["status"] == 1 and res[0]["rate_kbps"] == rate and res[0]["length"] == n + 4, (rate, n, res[0])
        assert (out[0, :n] == pay).all()
