"""The legacy 802.11a transmitter at 40 and 44 Msps in the oracle (sbo_tx11a_legacy_modulate_ex, oracle/tx11a_legacy44.cpp): the 40 Msps path
against the pinned entry point, the 40 -> 44 Msps upsampler against a second reading and the reference's compiled body, 44 Msps frames
through the receive oracle, the ACK path, and LENGTH 4096."""
import os, zlib
import numpy as np, pytest
import oracle_py
import oracle_tx11a_legacy as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("kbps", O.RATES)
def test_40msps_is_the_pinned_transmitter_then_zeros(kbps):
    rng = np.random.default_rng(kbps)
    for n in (0, 1, 13, 100, 1500):
        body = rng.integers(0, 256, n).astype(np.uint8)
        old = oracle_py.tx11a_legacy_modulate(body, kbps)
        new = O.modulate(body, kbps, 40)
        assert len(new) == O.padded_samples(n + 4, kbps, 40) and len(new) % 64 == 0 and len(old) == O.signal_samples(n + 4, kbps, 40)
        assert (new[:len(old)] == old).all() and (new[len(old):] == 0).all()


def test_40msps_reproduces_ofdm_bin_and_the_table_vectors():
    ref = np.fromfile(os.path.join(GOLD, "ofdm.bin"), np.int8).reshape(-1, 2)
    got = O.modulate(np.full(200, 0x31, np.uint8), 24000, 40)
    assert (got[:3680] == ref[:3680]).all()
    for kbps in O.RATES:
        body = np.fromfile(os.path.join(GOLD, "legacy_tx", f"legacy_tx_{kbps}.bin"), np.uint8)
        want = np.fromfile(os.path.join(GOLD, "legacy_tx", f"legacy_tx_{kbps}.i8"), np.int8).reshape(-1, 2)
        assert (O.modulate(body, kbps, 40)[:len(want)] == want).all(), kbps


def test_44msps_reproduces_the_compiled_transmitter_vectors():
    """tests/golden/legacy_tx44/: one frame per rate that the reference's own BB11ATxFrameMod, compiled from atx_*.c, made at 44 Msps
    (make_legacy_tx44_vectors.py); the .bin is the MPDU + FCS as sent.  Padding included, sample for sample."""
    for kbps in O.RATES:
        psdu = np.fromfile(os.path.join(GOLD, "legacy_tx44", f"legacy_tx44_{kbps}.bin"), np.uint8)
        want = np.fromfile(os.path.join(GOLD, "legacy_tx44", f"legacy_tx44_{kbps}.i8"), np.int8).reshape(-1, 2)
        got = O.modulate(psdu, kbps, 44, append_crc=False)
        assert got.shape == want.shape and (got == want).all(), kbps


def _chunks():
    rng = np.random.default_rng(5)
    yield rng.integers(-32768, 32768, (164, 2)).astype(np.int16)                  # full range
    yield rng.integers(-2000, 2000, (164, 2)).astype(np.int16)                    # signal level
    yield rng.choice(np.array([-32768, 32767], np.int16), (164, 2))               # the rails
    yield np.full((164, 2), -32768, np.int16)
    yield np.full((164, 2), 32767, np.int16)
    yield rng.integers(16384, 32768, (164, 2)).astype(np.int16)                   # where SONE * x != x


def test_upsampler_sse_equals_scalar_reading():
    for x in _chunks():
        assert (O.up160(x) == O.up160_numpy(x)).all()
        w = x[:4].copy(); w[3] = 0
        assert (O.up3(w) == O.up3_numpy(w)).all()
    x = np.full((164, 2), 30000, np.int16)
    assert (O.up160(x)[0] != 30000).any()                                         # pmulhrsw by 0x7fff rounds: not the identity


def test_upsampler_over_read_reaches_output_175_only():
    x = np.random.default_rng(7).integers(-20000, 20000, (164, 2)).astype(np.int16)
    y = x.copy(); y[160] = 0
    a, b = O.up160(x), O.up160(y)
    assert (a[:175] == b[:175]).all() and (a[175] != b[175]).any()


@pytest.mark.skipif(not O.ref_available(), reason="oracle/_ref/libupsample44_ref.so not built (needs the reference tree)")
def test_upsampler_equals_the_reference_body():
    for x in _chunks():
        assert (O.up160(x) == O.ref_up160(x[:160], in_place_tail=False, behind=x[160:])).all()
        # in place, as UpsampleAndCopyNT runs it: the over-read sees the call's own first output
        y = x.copy(); y[160:] = O.up160(np.concatenate([x[:160], np.zeros((4, 2), np.int16)]))[:4]
        assert (O.up160(y) == O.ref_up160(x[:160], in_place_tail=True)).all()
        w = x[:4].copy(); w[3] = 0
        assert (O.up3(w) == O.ref_up3(w)).all()


@pytest.mark.parametrize("kbps", O.RATES)
def test_44msps_preamble_and_tail_by_the_scalar_reading(kbps):
    pre = O.preamble()
    got = O.modulate(np.arange(60, dtype=np.uint8), kbps, 44)
    p = np.concatenate([pre, np.zeros((4, 2), np.int16)])
    for c in range(4):
        want = O.up160_numpy(p[160 * c: 160 * c + 164])
        assert (got[176 * c: 176 * (c + 1)] == np.clip(want >> 6, -128, 127)).all(), c
    sig = O.signal_samples(64, kbps, 44)
    assert (got[sig - 4: sig] == 0).all() and (got[sig:] == 0).all()


@pytest.mark.parametrize("kbps", O.RATES)
def test_44msps_frames_decode_through_the_receive_oracle(kbps):
    rng = np.random.default_rng(kbps + 44)
    for n in (1, 333):
        body = rng.integers(0, 256, n).astype(np.uint8)
        w = O.modulate(body, kbps, 44)
        iq = np.zeros((len(w) + 4000, 2), np.int16); iq[1000:1000 + len(w)] = w.astype(np.int16) << 8
        res, out = oracle_py.rx11a_run(oracle_py.resample_44_40(iq), max_frames=1, out_stride=4096)
        assert len(res) == 1 and res[0]["status"] == oracle_py.E_FRAME_OK and res[0]["rate_kbps"] == kbps and res[0]["length"] == n + 4, res
        assert (out[0, :n] == body).all()


@pytest.mark.parametrize("sr", [40, 44])
def test_ack_path_equals_frame_path(sr):
    """Test11AACK: BB11AModulateACK (14 bytes through BB11ATxBufferMod6M) == BB11ATxFrameMod of FC + Duration + RA with the ACK's CRC as FCS."""
    ack = O.ack_frame([0x00, 0x11, 0x22, 0x33, 0x44, 0x55])
    assert list(ack[:4]) == [0xD4, 0, 0, 0] and int.from_bytes(bytes(ack[10:]), "little") == zlib.crc32(bytes(ack[:10]))
    a = O.modulate(ack, 6000, sr, append_crc=False)
    b = O.modulate(ack[:10], 6000, sr, append_crc=True)
    assert len(a) == O.padded_samples(14, 6000, sr) and (a == b).all()


@pytest.mark.parametrize("kbps", [6000, 18000, 36000, 48000])
@pytest.mark.parametrize("sr", [40, 44])
def test_length_4096_goes_into_the_parity_bit(kbps, sr):
    """GetSignal(code, 4096) = code | 1 << 17.  For the rate codes of odd parity that is GetSignal(code, 0), so the SIGNAL symbol of a
    4096-byte PSDU equals that of an empty one; the data symbols still carry all 4096 bytes."""
    assert bin(O.CODE[kbps]).count("1") % 2 == 1
    body = np.random.default_rng(1).integers(0, 256, 4092).astype(np.uint8)
    big = O.modulate(body, kbps, sr)
    empty = O.modulate(np.zeros(0, np.uint8), kbps, sr, append_crc=False)
    ch = 176 if sr == 44 else 160
    assert (big[4 * ch: 5 * ch] == empty[4 * ch: 5 * ch]).all()
    assert len(big) == O.padded_samples(4096, kbps, sr)
    small = O.modulate(body[:-1], kbps, sr)                                        # LENGTH 4095: another SIGNAL
    assert (small[4 * ch: 5 * ch] != big[4 * ch: 5 * ch]).any()
