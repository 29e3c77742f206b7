"""The 802.11b receiver oracle (oracle/rx11b.cpp) against the reference's own compiled bricks and graph (oracle/build_ref_rx11b.sh):
the CCK-11 and CCK-5.5 decoders, the differential demappers, the Barker despreader, the PLCP parser, the descrambler and frame sink, and
the whole CreateDemodGraph driven as MAC11b_Receive drives it.  No GPU.  The library's debug tap shows that the inputs reach the edges:
CCK correlations of INT_MIN, arg-max ties, DQPSK sums that wrap, every SFD / sync / PLCP / FCS outcome.  About 15 s on one core: the whole-chain cases run the scalar graph one capture at a
time."""
import itertools, numpy as np, pytest
import oracle_py, plcp_inputs, rail_inputs
from sora_b200 import synth
from test_cpu_oracle_11b import _fixture
from test_gpu_rx11b import _capture_11b

pytestmark = pytest.mark.skipif(not oracle_py.ref_rx11b_available(), reason="oracle/_ref/librx11b_ref.so not built (oracle/build_ref_rx11b.sh)")

_PH = np.array([[1, 1], [-1, 1], [-1, -1], [1, -1]])
def _qpsk_patterns(amp):
    """Every QPSK chip pattern of 8 chips (4^8), at amplitude amp; at amp 32767 the negative rail is -32768, so every CCK butterfly B
    reaches +-32768 and the L products INT_MIN."""
    x = (_PH[np.array(list(itertools.product(range(4), repeat=8)))] * amp).astype(np.int64)
    if amp == 32767: x = np.where(x < 0, -32768, x)
    return x.astype(np.int16)

_LASTS = ((0, 0), (1, -1), (32767, 32767), (-32768, -32768), (32767, -32768))

def _cck_inputs():
    rng = np.random.default_rng(11)
    yield from (_qpsk_patterns(a) for a in (37, 1 << 13, 32767))
    yield rng.integers(-32768, 32768, (20000, 8, 2)).astype(np.int16)                    # random full range
    yield np.zeros((16, 8, 2), np.int16)                                                   # all zero: every comparison ties
    yield np.stack([np.full((8, 2), v, np.int16) for v in (1, -1, 32767, -32768, 12345, -4096, 3)] * 2)   # constant chips
    yield np.where(rng.random((4000, 8, 2)) < 0.5, -32768, 32767).astype(np.int16)        # the rails at random

def test_cck_decoders_equal_the_reference():
    oracle_py.ref_rx11b_debug_reset()
    for x in _cck_inputs():
        for last in _LASTS:
            a, la = oracle_py.cck11_decode_n(x, last); b, lb = oracle_py.ref_cck11_decode(x, last)
            assert (a == b).all() and (la == lb).all(), ("CCK-11", last, np.nonzero(a != b)[0][:8])
            # both parities: the same symbols again after one more symbol, so each meets the other is_even
            a, _ = oracle_py.cck11_decode_n(x[1:], last); b, _ = oracle_py.ref_cck11_decode(x[1:], last)
            assert (a == b).all(), ("CCK-11 odd start", last)
            x5 = x[: len(x) // 2 * 2].reshape(-1, 16, 2)
            a, la = oracle_py.cck5_decode_n(x5, last); b, lb = oracle_py.ref_cck5_decode(x5, last)
            assert (a == b).all() and (la == lb).all(), ("CCK-5.5", last, np.nonzero(a != b)[0][:8])
    d = oracle_py.ref_rx11b_debug()
    assert d["cck_int_min"] > 0 and d["cck_tie"] > 0, d

def _dq(ref, s, halve):
    """The two DQPSK phase decisions on one chip pair, in int64 with 32-bit wrapping: soradsp.h:190-199 (halve) and
    barkerspread.hpp:432-439 (not)."""
    w = lambda v: ((v + (1 << 31)) % (1 << 32)) - (1 << 31)
    re = w(ref[..., 0] * s[..., 0] + ref[..., 1] * s[..., 1]); im = w(ref[..., 0] * s[..., 1] - ref[..., 1] * s[..., 0])
    if halve: re >>= 1; im >>= 1
    return (w(re + im) < 0).astype(np.uint8) | ((w(re - im) < 0).astype(np.uint8) << 1)

def test_cck_rails_halve_before_the_dqpsk_sum():
    """TCCK11Decoder takes the phase of each symbol's last chip against the last chip before it with soradsp.h's demap_dqpsk_bits, which
    halves re and im before re + im, not with TDQPSKDemap's.  The two bits it puts in 0..1 (then XORed with the odd-symbol rotation)
    follow the halved form on every rail pattern, and the unhalved form, which wraps there, disagrees on a large share of them."""
    x = _qpsk_patterns(32767).astype(np.int64)
    for last in _LASTS:
        b, _ = oracle_py.ref_cck11_decode(x.astype(np.int16), last)
        ref = np.concatenate([np.array([last], np.int64), x[:-1, 7]]); s = x[:, 7]
        got = (b & 3) ^ (np.arange(len(b)) % 2 * 3).astype(np.uint8)
        assert (got == _dq(ref, s, True)).all(), last
        assert (_dq(ref, s, False) != got).mean() > 0.2, last

def test_differential_demappers_equal_the_reference():
    """The oracle's DQPSK and DBPSK demappers (the functions its chain calls) against TDQPSKDemap and TDBPSKDemap, on the rails, at random
    and over the range of despread symbols.  At the rails TDQPSKDemap's re + im wraps in MSVC's 32-bit long (barkerspread.hpp:434-438)."""
    rng = np.random.default_rng(5)
    oracle_py.ref_rx11b_debug_reset()
    rails = np.where(rng.random((3000, 8, 2)) < 0.5, -32768, 32767).astype(np.int16)
    rnd = rng.integers(-32768, 32768, (3000, 8, 2)).astype(np.int16)
    small = rng.integers(-22528, 22529, (3000, 8, 2)).astype(np.int16)       # the range of despread symbols
    cck_ref = _qpsk_patterns(32767)[:4000, 7].reshape(-1, 8, 2)               # raw CCK chips, as the reference after a CCK symbol
    for x in (rails, rnd, small, cck_ref):
        for last in _LASTS:
            a, la = oracle_py.dqpsk_demap_n(x.reshape(-1, 4, 2), last); b, lb = oracle_py.ref_dqpsk_demap(x.reshape(-1, 4, 2), last)
            assert (a == b).all() and (la == lb).all(), ("DQPSK", last, np.nonzero(a != b)[0][:8])
            a, la = oracle_py.dbpsk_demap_n(x, last); b, lb = oracle_py.ref_dbpsk_demap(x, last)
            assert (a == b).all() and (la == lb).all(), ("DBPSK", last, np.nonzero(a != b)[0][:8])
    d = oracle_py.ref_rx11b_debug()
    assert d["dqpsk_re_wrap"] > 0 and d["dqpsk_sum_wrap"] > 0, d

def test_barker_despread_equals_the_reference():
    """The oracle's Barker despreader against QuickBarkerDespread (barkerspread.hpp:276-304), at random and on the rails."""
    rng = np.random.default_rng(6)
    x = np.concatenate([rng.integers(-32768, 32768, (5000, 11, 2)), np.where(rng.random((2000, 11, 2)) < 0.5, -32768, 32767),
                        rng.integers(-40, 40, (2000, 11, 2)), np.full((1, 11, 2), -32768), np.full((1, 11, 2), 32767)]).astype(np.int16)
    assert (oracle_py.despread_n(x) == oracle_py.ref_despread(x)).all()

def _hdr(signal, service, length, crc_flip=0):
    h = np.zeros((len(signal), 6), np.uint8)
    h[:, 0] = signal; h[:, 1] = service; h[:, 2] = length & 0xFF; h[:, 3] = length >> 8
    for i in range(len(h)):
        c = _crc16(h[i, :4]) ^ crc_flip
        h[i, 4] = c & 0xFF; h[i, 5] = c >> 8
    return h

def _crc16(b):
    c = 0xFFFF
    for x in b:
        c ^= int(x)
        for _ in range(8): c = (c >> 1) ^ 0x8408 if c & 1 else c >> 1
    return (~c) & 0xFFFF

def test_plcp_parser_equals_the_reference_and_the_restatement():
    oracle_py.ref_rx11b_debug_reset()
    sig, srv = np.meshgrid(np.arange(256), np.arange(256), indexing="ij"); sig = sig.ravel(); srv = srv.ravel()
    # every SIGNAL x SERVICE at a few lengths; then the four rates at lengths around each limit and zero, with every single-bit CRC error
    for length in (0, 1, 33, 12000, 65535):
        h = _hdr(sig, srv, np.full(len(sig), length))
        got = oracle_py.ref_plcp11b_parse(h)
        want = np.array([plcp_inputs.parse_11b(int(a), int(b), length, True) for a, b in zip(sig, srv)], np.int64)
        assert (want[:, 0] == 1).all() and (got[:, 0] == 0).all() and (got[:, 3] == want[:, 1]).all() and (got[:, 4] == want[:, 2]).all(), length
    rates = np.array([0x0A, 0x14, 0x37, 0x6E]); lens = np.array([0, 1, 2, 3, 4, 5, 8, 16, 11998, 12000, 12008, 12032, 65535])
    for flip in [0] + [1 << k for k in range(16)]:
        s = np.repeat(rates, len(lens) * 4); L = np.tile(np.repeat(lens, 4), len(rates)); sv = np.tile(np.array([0, 0x04, 0x08, 0x88]), len(rates) * len(lens))
        got = oracle_py.ref_plcp11b_parse(_hdr(s, sv, L, flip), prev=(1, 2000, 777))
        prev = (2000, 777)
        for i in range(len(s)):
            ok, rate, n = plcp_inputs.parse_11b(int(s[i]), int(sv[i]), int(L[i]), flip == 0, prev)
            assert got[i, 0] == (0 if ok else oracle_py.E_PLCP_FAIL) and got[i, 3] == rate and got[i, 4] == n, (flip, i, got[i], ok, rate, n)
            prev = (rate, n)
    d = oracle_py.ref_rx11b_debug()
    assert d["plcp_crc16"] > 0 and d["plcp_unknown_rate"] > 0 and d["plcp_short_length"] > 0, d

def test_descrambler_and_sink_equal_the_reference():
    """TDesc741 -> TBB11bFrameSink at every frame length 1..1500 and every seed (the seed runs with the length), good and bad FCS: the
    frame buffer holds the descrambled bytes and the verdict compares the CRC-32 of all but the FCS with the FCS's first three bytes.
    Below 4 bytes `frame_length - 4` wraps (PHY_11b.hpp:714): the sink keeps every byte and never reaches a verdict."""
    rng = np.random.default_rng(8)
    oracle_py.ref_rx11b_debug_reset()
    # the scrambler that TDesc741 (x^7 + x^4 + 1, scramble.hpp:93-162) undoes, one byte at a time from each register state
    lut_out = np.zeros((128, 256), np.uint8); lut_reg = np.zeros((128, 256), np.uint8)
    for reg0 in range(128):
        for byte in range(256):
            reg = reg0; o = 0
            for k in range(8):
                b = ((byte >> k) & 1) ^ (reg & 1) ^ ((reg >> 3) & 1)
                reg = (reg >> 1) | (b << 6); o |= b << k
            lut_out[reg0, byte] = o; lut_reg[reg0, byte] = reg
    for n in range(1, 1501):
        seed = n % 128; body = rng.integers(0, 256, max(n - 4, 0)).astype(np.uint8)
        fcs = np.frombuffer(np.uint32(oracle_py.crc32(body)).tobytes(), np.uint8)
        plain = np.concatenate([body, fcs])[:n] if n >= 4 else rng.integers(0, 256, n).astype(np.uint8)
        if n >= 4 and n % 3 == 0: plain[rng.integers(0, n - 1)] ^= 0x10
        reg = seed; out = np.zeros(n, np.uint8)
        for i, byte in enumerate(plain): out[i] = lut_out[reg, byte]; reg = int(lut_reg[reg, byte])
        e, crc, fb = oracle_py.ref_desc_sink11b(out, seed, n)
        if n < 4:
            assert e == 0 and (fb == plain).all(), (n, e)
            continue
        assert (fb[:n - 1] == plain[:n - 1]).all(), n
        fcs3 = int.from_bytes(plain[n - 4:n - 1].tobytes(), "little")
        good = (oracle_py.crc32(plain[:n - 4]) & 0xFFFFFF) == fcs3
        assert e == (1 if good else oracle_py.E_CRC32_FAIL) and crc == fcs3, (n, e, good)
    d = oracle_py.ref_rx11b_debug()
    assert d["fcs_ok"] > 0 and d["fcs_fail"] > 0, d

def _resample(x, ppm):
    """x at a sampling clock off by ppm (linear interpolation)."""
    t = np.arange(int(len(x) / (1 + ppm * 1e-6)) - 1) * (1 + ppm * 1e-6)
    return np.stack([np.interp(t, np.arange(len(x)), x[:, k]) for k in (0, 1)], -1).round().astype(np.int16)

def _sfd_bit_errors():
    """A 1 Mbps frame with each of the 16 SFD bits flipped on the air: every symbol from that bit on negated (DBPSK)."""
    iq, _ = synth.make_frames_11b(1, psdu_len=40, rate_kbps=1000, snr_db=None, gain=0.3, seed0=91)
    for j in range(16):
        x = iq[0].copy(); k = 400 + (128 + j) * 44
        x[k:] = -x[k:].astype(np.int32).clip(-32767, 32767)
        yield f"sfd-bit/{j}", x, 2

def _chain_cases():
    for name in ("1long44.mf.bin", "2long44.mf.bin"):
        yield name, _fixture(name), 4
    for rate in (5500, 11000):                                                             # CCK chips on the rails (rail_inputs)
        for i, x in enumerate(rail_inputs.cck_rail_frames_11b(rate)): yield f"cck-rails/{rate}/{i}", x, 1
    for rate in (1000, 2000, 5500, 11000):                                                 # every 44 Msps phase offset of the frame start
        iq, _ = synth.make_frames_11b(1, psdu_len=30, rate_kbps=rate, snr_db=30, gain=0.3, seed0=rate + 3)
        for ph in range(44): yield f"phase/{rate}/{ph}", np.concatenate([np.zeros((ph, 2), np.int16), iq[0]]), 1
        for ppm in (-80, -20, 20, 80):                                                     # sampling-clock offsets
            iq, _ = synth.make_frames_11b(1, psdu_len=200, rate_kbps=rate, snr_db=35, gain=0.3, seed0=rate + 5)
            yield f"clock/{rate}/{ppm}", _resample(iq[0], ppm), 2
    yield from _sfd_bit_errors()
    rng = np.random.default_rng(12)
    alt = np.where(np.arange(28 * 200) % 2 == 0, 1, -1)                                    # zero DC, |x|^2 >> 5 summed over 32 samples:
    for a in (1000, 999):                                                                  # exactly cca_pwr_threshold at 1000, below at 999
        yield f"cca-exact/{a}", np.stack([alt * a, np.zeros_like(alt)], -1).astype(np.int16), 4
    for sd in (690, 707, 725):                                                             # noise around the threshold
        yield f"cca-noise/{sd}", rng.normal(0, sd, (28 * 400, 2)).round().astype(np.int16), 8
    for dc in ((32767, -32768), (-32768, -32768)):                                         # DC on the rails, with noise
        yield f"dc-rails/{dc}", (np.array(dc) + rng.normal(0, 300, (28 * 300, 2))).clip(-32768, 32767).astype(np.int16), 8
    for rate in (1000, 2000, 5500, 11000):
        for snr, gain in ((None, 1.0), (40, 0.3), (28, 0.25), (18, 0.2)):
            iq, _ = synth.make_frames_11b(5, psdu_len=96, rate_kbps=rate, snr_db=snr, gain=gain, seed0=rate + 7)
            for i in range(len(iq)): yield f"{rate}/{snr}/{gain}/{i}", iq[i], 1
        for k, (label, x) in enumerate(rail_inputs.cases_11b(rate)): yield f"rails/{rate}/{label}", x, 2
        iq, _ = synth.make_frames_11b(2, psdu_len=120, rate_kbps=rate, snr_db=30, gain=0.3, seed0=rate + 99, cfo_hz=60e3)
        for i in range(len(iq)): yield f"cfo/{rate}/{i}", iq[i], 2
    iq, _ = synth.make_frames_11b(1, psdu_len=200, rate_kbps=11000, snr_db=40, gain=0.3)
    for n in (len(iq[0]), len(iq[0]) // 2, 3001, 3000, 27, 28, 29, 1):                     # truncated and tiny slots
        yield f"trunc/{n}", iq[0][:n], 4
    rng = np.random.default_rng(4)
    yield "noise", rng.normal(0, 2500, (28 * 300, 2)).astype(np.int16), 8
    yield "noise-loud", rng.normal(0, 9000, (28 * 900, 2)).clip(-32768, 32767).astype(np.int16), 8
    yield "zeros", np.zeros((5600, 2), np.int16), 8
    for s, specs, nz in ((1, [(11000, 300, False), (2000, 60, False), (5500, 200, True), (11000, 1000, False), (1000, 40, False)], 60.0),
                         (2, [(5500, 500, False), (11000, 77, False)], 0.0),
                         (3, [(2000, 100, True), (1000, 30, False), (11000, 1496, False)], 120.0)):
        yield f"capture/{s}", _capture_11b(s, specs, noise=nz)[0], 8

def test_whole_chain_equals_the_reference():
    """oracle rx11b_run == CreateDemodGraph under MAC11b_Receive: every event, its position, detection vector, CRC and bytes."""
    oracle_py.ref_rx11b_debug_reset()
    for name, iq, maxf in _chain_cases():
        a, ab = oracle_py.rx11b_run(iq, max_frames=maxf, out_stride=2048)
        b, bb = oracle_py.ref_rx11b_run(iq, max_frames=maxf, out_stride=2048)
        assert len(a) == len(b), (name, a, b)
        for k in a.dtype.names: assert (a[k] == b[k]).all(), (name, k, a, b)
        for i in range(len(a)):
            if a["status"][i] in (1, oracle_py.E_CRC32_FAIL):
                L = min(int(a["length"][i]) - 1, 2048)
                assert (ab[i, :L] == bb[i, :L]).all(), (name, i)
    d = oracle_py.ref_rx11b_debug()
    for k in ("sfd_fail", "sfd_timeout", "sync_timeout", "plcp_crc16", "fcs_ok", "fcs_fail", "cs_timeout"):
        assert d[k] > 0, (k, d)

def test_batch_equals_the_reference():
    iq, _ = synth.make_frames_11b(6, psdu_len=80, rate_kbps=5500, snr_db=25, gain=0.3, seed0=77)
    F, slot, _ = iq.shape
    off = np.arange(F, dtype=np.uint64) * slot; ln = np.array([slot, slot, slot // 3, 100, slot, 28], np.uint32)
    a, ab = oracle_py.rx11b_batch(iq.reshape(-1, 2), off, ln, out_stride=512)
    b, bb = oracle_py.ref_rx11b_batch(iq.reshape(-1, 2), off, ln, out_stride=512)
    for k in a.dtype.names: assert (a[k] == b[k]).all(), (k, a, b)
