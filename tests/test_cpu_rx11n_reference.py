"""The PLCP header parsers and the descrambler / frame sink of the OFDM receivers against the reference's own compiled bricks
(oracle/build_ref_rx11n.sh -> oracle/_ref/librx11n_ref.so): T11aPLCPParser, T11nSigParser, and T11aDesc into TBB11aFrameSink.

Until now these stages were checked only against their restatement in oracle/ (and, for the parsers, tests/plcp_inputs.py, a second
restatement): a wrong limit, a CRC-8 compared at the wrong width or a descrambler seeded from the wrong bits would have passed as long
as both restatements made it.  Here the oracle must equal the compiled bricks on every field they leave:
  - every one of the 2^24 SIGNAL words through T11aPLCPParser, and every one as the L-SIG of T11nSigParser;
  - HT-SIG blocks with every MCS 0-127, lengths at and around the 1500-byte limit, a bad CRC-8 in each bit, bits set past the CRC,
    and sequences whose L-SIG refusals report the MCS of the block before (CF_HTRxVector is never reset);
  - the descrambler and sink of both receivers at every scrambler seed 0-127, every frame length 1-1500, good and bad FCS.
Every word the SIGNAL decoders can hand over (bits 18-23 clear, the decoder's >> 6: 2^18 of them) is also compared with the restatement
in tests/plcp_inputs.py, through both parsers.
The 802.11n front end (carrier sense, CFO, channel estimates and 2x2 inverse, pilot tracker, demappers, de-interleavers, stream
de-parser) is not compiled or compared here.
Runs in about 7 s on one CPU core.  Skips when the library is not built (no reference tree)."""
import numpy as np
import pytest

import oracle_py as O
import plcp_inputs as P
from sora_b200 import synth

pytestmark = pytest.mark.skipif(not O.ref_rx11n_available(), reason="oracle/_ref/librx11n_ref.so not built (needs the reference tree)")

CHUNK = 1 << 21


def _sig9(lsig, ht48):
    """9 bytes as T11nViterbiSig hands them: the L-SIG's 24 bits, then the HT-SIG's 48 (the first 34, the CRC-8, the tail)."""
    lsig = np.asarray(lsig, np.uint64).reshape(-1); ht48 = np.broadcast_to(np.asarray(ht48, np.uint64), lsig.shape)
    w = np.empty((len(lsig), 9), np.uint8)
    for i in range(3): w[:, i] = (lsig >> np.uint64(8 * i)) & np.uint64(0xFF)
    for i in range(6): w[:, 3 + i] = (ht48 >> np.uint64(8 * i)) & np.uint64(0xFF)
    return w


def _ht48(h34, crc_xor=0):
    return (h34 & ((1 << 34) - 1)) | (P.crc8_htsig(h34) ^ crc_xor) << 34


def _diff(a, b, fields, what):
    bad = np.nonzero((a != b).any(1))[0]
    if len(bad):
        i = bad[0]
        raise AssertionError(f"{what}: {len(bad)} differ, first #{i}: oracle {dict(zip(fields, a[i]))} reference {dict(zip(fields, b[i]))}")


def test_plcp11a_every_signal_word():
    for lo in range(0, 1 << 24, CHUNK):
        w = np.arange(lo, lo + CHUNK, dtype=np.uint32)
        _diff(O.plcp11a_parse(w), O.ref_plcp11a_parse(w), O.PLCP11A_FIELDS, f"SIGNAL words {lo:#x}..")


def test_plcp11a_decodable_words_match_restatement():
    w = np.arange(1 << 18, dtype=np.uint32)
    ref = O.ref_plcp11a_parse(w)
    for i in range(1 << 18):                            # every word the decoder can hand over
        acc, rate, length, nsym = P.parse_11a(i)
        got = ref[i]
        assert (bool(got[0]), got[1] == P.E_PLCP) == (acc, not acc), hex(i)
        if acc:
            assert (got[2], got[3], got[4]) == (rate, length, nsym), hex(i)
        elif rate == 0:
            assert got[2] == 0, hex(i)


def test_lsig11n_every_word():
    ht = _ht48(9 | 100 << 8 | 0x07 << 24)
    for lo in range(0, 1 << 24, CHUNK):
        s = _sig9(np.arange(lo, lo + CHUNK, dtype=np.uint64), ht)
        _diff(O.sig11n_parse(s), O.ref_sig11n_parse(s), O.SIG11N_FIELDS, f"L-SIG words {lo:#x}..")


def test_lsig11n_decodable_words_match_restatement():
    ht = 9 | 100 << 8 | 0x07 << 24
    w = np.arange(1 << 18, dtype=np.uint64)             # every word the decoder can hand over
    ref = O.ref_sig11n_parse(_sig9(w, _ht48(ht)))
    prev = 0
    for i, word in enumerate(w):
        acc, mcs, length, nsym, _ = P.parse_11n(int(word), ht, P.crc8_htsig(ht), prev_mcs=prev)
        got = ref[i]
        assert (bool(got[0]), got[6]) == (acc, mcs), hex(int(word))
        if acc:
            assert (got[3], got[4]) == (length, nsym), hex(int(word))
        prev = mcs


def _htsig_corpus():
    """(name, sig9) blocks: every MCS with a good CRC at several lengths, a bad CRC in each bit, bits past the CRC, flags."""
    lw = synth.signal_word_11a(6000, 300)
    blocks, names = [], []
    def add(name, h34, crc_xor=0, tail=0, lsig=lw):
        blocks.append(_sig9(lsig, _ht48(h34, crc_xor) | tail << 42)[0]); names.append(name)
    for mcs in range(128):
        for L in (0, 1, 4, 1499, 1500, 1501, 4095, 65535):
            add(f"mcs{mcs}_len{L}", mcs | L << 8 | 0x07 << 24)
    h = 9 | 200 << 8 | 0x07 << 24
    for bit in range(8):
        add(f"crc8_bit{bit}", h, 1 << bit)
    for bit in range(34):
        add(f"data_bit{bit}_crc_kept", h ^ 1 << bit, P.crc8_htsig(h) ^ P.crc8_htsig(h ^ 1 << bit))
    # bits past the CRC: PHY_11n.hpp:488 compares the CRC byte with an int, so any of them fails the check (the oracle once cast
    # to 8 bits there and accepted these).  The SIG decoder's >> 6 keeps them clear in a receiver.
    for t in range(6):
        add(f"htsig_tail_bit{t}_set", h, 0, 1 << t)
    for flags in range(0, 256, 7):
        add(f"flags_{flags:02x}", 9 | 200 << 8 | flags << 24)
    # L-SIG refusals between HT-SIGs: the MCS of the block before is what a refusal reports
    for k, lsig in enumerate((lw ^ 1 << 17, lw | 1 << 4 ^ 1 << 17, synth.signal_word_11a(6000, 751), (lw & ~0xF) | 0x7)):
        add(f"mcs10_before_lsig_refusal{k}", 10 | 100 << 8 | 0x07 << 24)
        add(f"lsig_refusal{k}", h, lsig=lsig)
        add(f"crc_fail_before_lsig_refusal{k}", h, 0x40)
        add(f"lsig_refusal{k}_after_crc_fail", h, lsig=lsig)
    return names, np.array(blocks, np.uint8)


def test_htsig_corpus():
    names, s = _htsig_corpus()
    a, b = O.sig11n_parse(s), O.ref_sig11n_parse(s)
    bad = np.nonzero((a != b).any(1))[0]
    assert not len(bad), [(names[i], a[i].tolist(), b[i].tolist()) for i in bad[:5]]
    prev = 0
    for i, name in enumerate(names):                   # and the restatement, on the blocks a decoder can hand over
        lsig = int.from_bytes(s[i, :3].tobytes(), "little"); ht = int.from_bytes(s[i, 3:].tobytes(), "little")
        if ht >> 42:
            assert b[i, 0] == 0 and b[i, 6] == 0, name
        else:
            acc, mcs, length, nsym, _ = P.parse_11n(lsig, ht & ((1 << 34) - 1), ht >> 34, prev_mcs=prev)
            assert (bool(b[i, 0]), b[i, 6]) == (acc, mcs), name
            if acc:
                assert (b[i, 3], b[i, 4]) == (length, nsym), name
        prev = int(b[i, 6])
    assert set(b[:, 6]) >= set(range(8, 11)) and b[:, 0].sum() > 0


def _decoded(psdu, seed):
    """What T11aViterbi hands the descrambler for PSDU bytes `psdu` scrambled from `seed`: SERVICE then the PSDU, scrambled."""
    bits = np.zeros(16 + 8 * len(psdu), np.uint8)
    bits[16:] = np.unpackbits(np.asarray(psdu, np.uint8), bitorder="little")
    bits ^= synth.scrambler_seq(seed, len(bits))
    return np.packbits(bits, bitorder="little")


def _sink_cases():
    rng = np.random.default_rng(11)
    for seed in range(128):
        yield f"seed{seed}", seed, P.psdu(100, seed), 100
    for L in range(1, 1501):
        body = P.psdu(L, L)
        yield f"len{L}", 1 + L % 127, body, L
        if L >= 4 and L % 7 == 0:
            bad = body.copy(); bad[rng.integers(0, L)] ^= 1 << int(rng.integers(0, 8))
            yield f"len{L}_bad_fcs", 1 + L % 127, bad, L
    body = P.psdu(300, 5)
    yield "claim_shorter", 33, body, 200
    yield "claim_longer", 34, body[:250], 300


def test_descrambler_and_sink():
    n_ok = n_fail = 0
    for name, seed, body, L in _sink_cases():
        d = _decoded(body, seed)
        want = O.ref_desc_sink(d, L)
        m = min(L, len(d) - 2)                          # the bytes the sink stored; the rest of its buffer is whatever was there
        for chain in (0, 1):
            got = O.desc_sink(chain, d, L)
            assert got[0] == want[0] and got[1] == want[1] and (got[2][:m] == want[2][:m]).all(), (name, chain, got[:2], want[:2])
        if L >= 4 and len(body) >= L:
            assert (want[2] == body[:L]).all(), name
        n_ok += want[0] == O.E_FRAME_OK; n_fail += want[0] == O.E_CRC32_FAIL
    assert n_ok > 1000 and n_fail > 100


def test_counters_reached():
    O.ref_rx11n_debug_reset()
    O.ref_plcp11a_parse(np.arange(1 << 18, dtype=np.uint32))
    _, s = _htsig_corpus()
    O.ref_sig11n_parse(s)
    O.ref_sig11n_parse(_sig9(np.arange(1 << 16, dtype=np.uint64), _ht48(9 | 100 << 8)))
    for name, seed, body, L in list(_sink_cases())[:200]:
        O.ref_desc_sink(_decoded(body, seed), L)
    O.ref_desc_sink(_decoded(P.psdu(50, 1)[::-1], 3), 50)
    d = O.ref_rx11n_debug()
    assert all(v > 0 for v in d.values()), d
