"""PLCP header cases for the 802.11a / b / n receivers: ready-made captures whose headers are whatever a case asks for, and a plain
restatement of the three header parsers that says what a receiver reports for each of them.

The restatement is the reference for the header arithmetic only.  What follows an accepted header (demodulation, Viterbi, sink) is
the C++ oracle's to say, so a case also names the verdict its body leads to:
  "ok"    the body is a valid PSDU of the claimed length;
  "crc"   the claim and the body disagree, the FCS check fails;
  "none"  the sink never reaches a verdict inside the slot: no event (LENGTH < 4 has no verdict, `(int)L - 4` is negative);
  "failed" every symbol went through without a verdict (802.11a / n LENGTH < 4: E_FAILED once the symbols run out).

What the parsers see of a header is what the SIGNAL decoders hand them: the Viterbi SIGNAL decoders return their traceback `>> 6`
(viterbi.hpp:39), so the six tail bits of the 802.11a SIGNAL and of the L-SIG, and the HT-SIG tail, never reach a parser.
"""
import numpy as np
from sora_b200 import synth

E_OK, E_CRC32, E_PLCP, E_NONE, E_FAILED = 1, 0x80000006, 0x80000005, 0x8000F001, 0x8000FFFF
VERDICT = {"ok": E_OK, "crc": E_CRC32, "none": E_NONE, "failed": E_FAILED}

RATE11A = {0xB: 6000, 0xF: 9000, 0xA: 12000, 0xE: 18000, 0x9: 24000, 0xD: 36000, 0x8: 48000, 0xC: 54000}   # ieee80211a_cmn.h:97-112
NDBPS11A = {6000: 24, 9000: 36, 12000: 48, 18000: 72, 24000: 96, 36000: 144, 48000: 192, 54000: 216}
NDBPS11N = {8: 52, 9: 104, 10: 156, 11: 208, 12: 312, 13: 416, 14: 468}                                     # ieee80211n_cmn.h:7-26


def _odd_parity(w):
    return bin(w).count("1") & 1


def parse_11a(sig):
    """T11aPLCPParser::_parse_plcp (PHY_11a.hpp:549-580) on a CF_11aRxVector just Reset() (ieee80211facade.hpp:235-242).
    sig: the 24 SIGNAL bits as sent.  Returns (accepted, rate_kbps, length, nsym) as the receiver reports them."""
    u = sig & 0x3FFFF                                   # the decoder hands over bits 0..17 (viterbi.hpp:39)
    rate, length, nsym = 6000, 0, 0
    if u & 0xFC0010 or _odd_parity(u):                  # :553-562 reserved bit / tail, even parity
        return False, rate, length, nsym
    rate = RATE11A.get(u & 0xF, 0)                      # :564-566 BB11aParseDataRate: 0 is stored, then refused
    if rate == 0:
        return False, 0, length, nsym
    length = (u >> 5) & 0xFFF                           # :570-572
    if length > 2500:
        return False, rate, length, nsym
    nsym = -(-(length * 8 + 16 + 6) // NDBPS11A[rate]) + 1   # :574-576, this SIGNAL symbol counted
    return True, rate, length, nsym


_SIGNAL11B = {0x0A: 1000, 0x14: 2000, 0x37: 5500, 0x6E: 11000}

def parse_11b(signal, service, length, crc_ok, prev=(0, 0)):
    """TBB11bPlcpParser (PHY_11b.hpp:556-651).  CF_11bRxVector has no Reset() (ieee80211facade.hpp:72-76): `prev` = (rate, length) the
    context holds from the event before (batch slots start from (0, 0)).  Returns (accepted, rate_kbps, length)."""
    if not crc_ok:                                      # :562-566
        return False, prev[0], prev[1]
    rate = _SIGNAL11B.get(signal, 0)                    # :608-629
    if signal == 0x0A: L = length >> 3                  # :631-651, ushort arithmetic: 5.5 / 11 Mbps LENGTH 0 with a correction wraps to 0xFFFF
    elif signal == 0x14: L = length >> 2
    elif signal == 0x37: L = ((length * 11) >> 4) - (service >> 7) - ((service >> 3) & 1)
    elif signal == 0x6E: L = ((length * 11) >> 3) - (service >> 7) - ((service >> 3) & 1)
    else: L = 0                                         # unknown rate: rxrate_state unchanged, demodulation goes on as DBPSK
    return True, rate, L & 0xFFFF


def crc8_htsig(h34):
    """CRC-8 of the first 34 HT-SIG bits (core/inc/CRC8.h:29-50)."""
    return synth._crc8_htsig(np.frombuffer((h34 & ((1 << 34) - 1)).to_bytes(6, "little"), np.uint8))


def parse_11n(lsig, h34, crc8, mcs_limit=11, prev_mcs=0):
    """T11nSigParser (PHY_11n.hpp:432-513) after CF_11aRxVector::Reset().  lsig: the 24 L-SIG bits as sent; h34: the first 34 HT-SIG bits;
    crc8: the CRC-8 sent with them.  CF_HTRxVector has no Reset() (ieee80211facade.hpp:269-272): when _parse_plcp refuses the L-SIG,
    ht_frame_mcs is still `prev_mcs`, the value of the event before (0 in a fresh context).
    Returns (accepted, mcs, length, nsym, lsig_length)."""
    u = lsig & 0x3FFFF                                  # the decoder hands over bits 0..17 (viterbi.hpp:39)
    if u & 0xFC0010 or _odd_parity(u) or not (u & 8):  # :458-475 _parse_plcp; the eight legal rate codes all have bit 3 set
        return False, prev_mcs, 0, 0, 0
    length = ((u >> 5) & 0xFFF) * 2                     # :477-479
    if length > 1500:
        return False, prev_mcs, length, 0, length
    if crc8_htsig(h34) != crc8:                         # :486-494 _parse_htsig
        return False, 0, length, 0, length
    mcs = h34 & 0x7F                                    # :496-501 (11 as shipped; 15 with the 16-/64-QAM branches)
    if mcs < 8 or mcs >= mcs_limit:
        return False, mcs, length, 0, length
    hl = (h34 >> 8) & 0xFFFF                            # :503-506
    if hl > 1500:
        return False, mcs, length, 0, length
    return True, mcs, hl, -(-(hl * 8 + 16 + 6) // NDBPS11N[mcs]) + 4, length    # :508-510, :447 frame_length = ht_frame_length


# ---- case builders --------------------------------------------------------------------------------------------------------------
def psdu(n, seed):
    """n >= 4 bytes: random MPDU + its CRC-32; n < 4: zeros (no FCS fits)."""
    if n < 4:
        return np.zeros(n, np.uint8)
    return synth.psdu_with_fcs(np.random.RandomState(seed).randint(0, 256, n - 4).astype(np.uint8))


def pack(slots):
    """list of int16 [n, 2] captures -> (iq, off, len) with every slot starting on a 16-byte boundary."""
    off = np.cumsum([0] + [(len(s) + 3) // 4 * 4 for s in slots[:-1]]).astype(np.uint64)
    iq = np.zeros((int(off[-1]) + len(slots[-1]), 2), np.int16)
    for o, s in zip(off, slots):
        iq[int(o):int(o) + len(s)] = s
    return iq, off, np.array([len(s) for s in slots], np.uint32)


def case_11a(name, rate, body, signal_word=None, verdict=None, trail=400, slot=None):
    """One 802.11a frame at 40 Msps: SIGNAL `signal_word` (default: the one `body` calls for), DATA = `body` at `rate`."""
    sw = synth.signal_word_11a(rate, len(body)) if signal_word is None else signal_word
    iq = synth.to_iq16(synth.modulate(body, rate, signal_word=sw), lead=200, trail=trail)[0]
    if slot is not None:
        iq = iq[:slot]
    acc, r, L, ns = parse_11a(sw)
    if not acc:
        verdict = "plcp"
    elif verdict is None:
        verdict = "ok" if L == len(body) and L >= 4 else "failed" if L < 4 else "crc"
    return dict(name=name, iq=iq, word=sw, body=body, verdict=verdict, expect=dict(rate_kbps=r, length=L, nsym=ns))


def cases_11a():
    C = []
    b100 = psdu(100, 1)
    for nib in range(16):                               # every rate nibble, correct parity
        rate = RATE11A.get(nib, 6000)
        w = nib | 100 << 5; w |= _odd_parity(w) << 17
        C.append(case_11a(f"rate_nibble_{nib:x}", rate, b100, w))
    w = synth.signal_word_11a(24000, 100)
    C.append(case_11a("parity_flipped", 24000, b100, w ^ 1 << 17))
    C.append(case_11a("reserved_bit", 24000, b100, w ^ 1 << 4 ^ 1 << 17))          # parity kept even
    for t in range(6):
        C.append(case_11a(f"tail_bit_{t}", 24000, b100, w | 1 << (18 + t)))
    for L in range(4):
        C.append(case_11a(f"length_{L}", 12000, np.zeros(L, np.uint8)))
    C.append(case_11a("length_4_empty_mpdu", 12000, psdu(4, 0)))
    for rate in sorted(NDBPS11A):
        C.append(case_11a(f"length_5_{rate}", rate, psdu(5, rate)))
        C.append(case_11a(f"length_2500_{rate}", rate, psdu(2500, rate + 1), trail=64))
    for L in (2501, 4095):
        C.append(case_11a(f"length_{L}", 54000, b100, synth.signal_word_11a(54000, L)))
    C.append(case_11a("claim_longer_than_body", 36000, b100, synth.signal_word_11a(36000, 160), trail=1200))
    C.append(case_11a("claim_shorter_than_body", 36000, b100, synth.signal_word_11a(36000, 60)))
    C.append(case_11a("claim_past_slot_end", 36000, b100, synth.signal_word_11a(36000, 1000), verdict="none"))
    return C


def case_11b(name, rate, body, plcp=None, verdict=None, trail=400, prev=(0, 0)):
    """One long-preamble 802.11b frame at 44 Msps; plcp = (SIGNAL, SERVICE, LENGTH, CRC-16 xor mask) or None for the right one."""
    hdr = synth.plcp_11b(len(body), rate) + (0,) if plcp is None else plcp
    td = synth.modulate_11b(body, rate, shape=False, plcp=hdr)               # rectangular chips: every clean 11 Mbps body decodes
    n = 400 + len(td) + trail; trail += (-n) % 28
    iq = synth.to_iq16(td, lead=400, trail=trail)[0]
    acc, r, L = parse_11b(hdr[0], hdr[1], hdr[2], hdr[3] == 0, prev)
    if not acc:
        verdict = "plcp"
    elif verdict is None:
        verdict = "ok" if L == len(body) and L >= 4 else "none" if L < 4 or r == 0 else "crc"
    return dict(name=name, iq=iq, word=hdr, body=body, verdict=verdict, expect=dict(rate_kbps=r, length=L))


def cases_11b():
    C = []
    b60 = psdu(60, 2)
    for sig in (0x0A, 0x14, 0x37, 0x6E, 0x00, 0xFF, 0x0B, 0x6F):
        rate = _SIGNAL11B.get(sig, 1000)
        hdr = synth.plcp_11b(60, rate)
        C.append(case_11b(f"signal_{sig:02x}", rate, b60, (sig, hdr[1], hdr[2], 0)))
    hdr = synth.plcp_11b(60, 2000) + (0,)
    for bit in range(16):
        C.append(case_11b(f"crc16_bit_{bit}", 2000, b60, hdr[:3] + (1 << bit,)))
    for L in range(200, 211):                           # all 11 residues of 8L mod 11
        s, sv, ln = synth.plcp_11b(L, 11000)
        body = psdu(L, L)
        C.append(case_11b(f"cck11_len_{L}_ext_right", 11000, body, (s, sv, ln, 0)))
        C.append(case_11b(f"cck11_len_{L}_ext_wrong", 11000, body, (s, sv ^ 0x80, ln, 0)))
    for rate in (5500, 11000):
        s, sv, ln = synth.plcp_11b(90, rate)
        C.append(case_11b(f"service_bit3_clear_{rate}", rate, psdu(90, 3), (s, sv & ~0x08, ln, 0)))
        C.append(case_11b(f"service_bit3_set_{rate}", rate, psdu(90, 3), (s, sv | 0x08, ln, 0)))
    for L in range(6):                                  # frame lengths 0..5 at 1 Mbps: LENGTH 8 L microseconds
        C.append(case_11b(f"frame_length_{L}", 1000, psdu(L, 5), (0x0A, 0x04, 8 * L, 0)))
    for rate, s in ((5500, 0x37), (11000, 0x6E)):
        C.append(case_11b(f"length_0_ext_{rate}", rate, psdu(8, 6), (s, 0x84, 0, 0), trail=65536 * (64 if rate == 5500 else 32)))   # ((0 * 11) >> n) - 1 wraps to 0xFFFF
    C.append(case_11b("length_4095_11m", 11000, psdu(4095, 7), trail=200))
    C.append(case_11b("length_2000_1m", 1000, psdu(2000, 8), trail=200))
    # a claim beyond 4096 bytes: the sink wraps its frame buffer in the oracle, clips at out_stride on the device; fields only
    C.append(case_11b("claim_beyond_4096", 11000, b60, (0x6E, 0x04, 3700, 0), trail=170000))
    return C


CHAN = ((1.0, 0.3j), (-0.2, 0.9))

def case_11n(name, mcs, body, lsig_word=None, htsig=None, verdict=None, mcs_limit=11, prev_mcs=0, trail=200):
    """One HT-MF 2x2 frame at 40 Msps through CHAN; lsig_word / htsig = (first 34 bits, CRC-8 xor mask) override the header."""
    L = len(body)
    nt = -(-(16 + 8 * L + 6) // NDBPS11N[mcs]) + 5
    lw = synth.signal_word_11a(6000, (nt * 24 - 22) // 8) if lsig_word is None else lsig_word
    h34, cx = (mcs | L << 8 | 0x07 << 24, 0) if htsig is None else htsig
    tx = synth.modulate_11n(body, mcs, lsig_word=lw, htsig=(h34, cx))
    rx = np.einsum("ab,fbn->fan", np.asarray(CHAN, np.complex128), tx)
    iq0 = synth.to_iq16(rx[:, 0], lead=400, trail=trail)[0]; iq1 = synth.to_iq16(rx[:, 1], lead=400, trail=trail)[0]
    acc, m, ln, ns, lsl = parse_11n(lw, h34, crc8_htsig(h34) ^ cx, mcs_limit, prev_mcs)
    if not acc:
        verdict = "plcp"
    elif verdict is None:
        verdict = "ok" if ln == L and ln >= 4 else "failed" if ln < 4 else "crc"
    return dict(name=name, iq0=iq0, iq1=iq1, word=(lw, h34, cx), body=body, verdict=verdict,
                expect=dict(mcs=m, length=ln, nsym=ns, lsig_length=lsl))


def cases_11n(mcs_limit=11):
    C = []
    b = psdu(120, 9)
    base = lambda m, body: (m | len(body) << 8 | 0x07 << 24, 0)
    k = lambda name, *a, **kw: C.append(case_11n(name, *a, mcs_limit=mcs_limit, **kw))
    nt = -(-(16 + 8 * 120 + 6) // 104) + 5
    lw = synth.signal_word_11a(6000, (nt * 24 - 22) // 8)
    k("lsig_parity", 9, b, lsig_word=lw ^ 1 << 17)
    k("lsig_reserved", 9, b, lsig_word=lw ^ 1 << 4 ^ 1 << 17)
    for t in (0, 5):
        k(f"lsig_tail_{t}", 9, b, lsig_word=lw | 1 << (18 + t))
    k("lsig_rate_54m", 9, b, lsig_word=synth.signal_word_11a(54000, (lw >> 5) & 0xFFF))
    w = (lw & ~0xF) | 0x7; k("lsig_rate_illegal", 9, b, lsig_word=w ^ (_odd_parity(w) ^ _odd_parity(lw)) << 17)
    for L in (750, 751):
        k(f"lsig_length_{L}", 9, b, lsig_word=synth.signal_word_11a(6000, L))
    h = base(9, b)
    for bit in (0, 3, 7):
        k(f"crc8_bit_{bit}", 9, b, htsig=(h[0], 1 << bit))
    for m in list(range(0, 17)) + [127]:
        body_mcs = m if 8 <= m <= 14 else 9
        k(f"mcs_{m}", body_mcs, b, htsig=base(m, b))
    k("cbw40", 9, b, htsig=(h[0] | 1 << 7, 0))
    for L in (0, 1, 3, 4, 1500):
        body = psdu(L, 10 + L)
        k(f"ht_length_{L}", 8, body)
    for L in (1501, 65535):
        k(f"ht_length_{L}", 9, b, htsig=((h[0] & ~(0xFFFF << 8)) | L << 8, 0))
    # bits the parser ignores, set with a valid CRC: smoothing 24, not sounding 25 (0x07 already sets 24..26), aggregation 27,
    # STBC 28-29, LDPC 30, short GI 31, Ness 32-33
    for name, bits in (("smoothing_off", 0x07 & ~1), ("not_sounding_off", 0x07 & ~2), ("aggregation", 0x07 | 8), ("stbc", 0x07 | 0x30),
                       ("ldpc", 0x07 | 0x40), ("short_gi", 0x07 | 0x80), ("ness", 0x07 | 0x300)):
        k(f"flag_{name}", 9, b, htsig=((h[0] & ~(0xFF << 24)) | bits << 24, 0))
    return C


def slots_of(cases, key="iq"):
    return pack([c[key] for c in cases])


def expected_status(c):
    return E_PLCP if c["verdict"] == "plcp" else VERDICT[c["verdict"]]


# ---- continuous captures: refused headers between decoded frames, for what a context carries from one event to the next -------------
def _chain(cases, keys):
    return tuple(np.concatenate([c[k] for c in cases]) for k in keys)

def _expect(c, status_fields):
    e = dict(c["expect"]); e["status"] = expected_status(c)
    return {k: e[k] for k in status_fields}

def stream_11a():
    """Decoded, parity refused, illegal rate, LENGTH 2501, decoded: CF_11aRxVector::Reset() after every event, nothing carried."""
    b = psdu(300, 21)
    cs = [case_11a("dec54", 54000, b), case_11a("parity", 24000, b, synth.signal_word_11a(24000, 300) ^ 1 << 17),
          case_11a("nibble3", 6000, b, 3 | 300 << 5 | _odd_parity(3 | 300 << 5) << 17), case_11a("len2501", 54000, b, synth.signal_word_11a(54000, 2501)),
          case_11a("dec12", 12000, psdu(77, 22))]
    return _chain(cs, ("iq",))[0], [_expect(c, ("status", "rate_kbps", "length", "nsym")) for c in cs]

def stream_11b():
    """Decoded, CRC-16 failure, decoded, SERVICE bit 3 set, CRC-16 failure, decoded: CF_11bRxVector has no Reset(), so a refused header
    reports the rate and length of the event before it."""
    b100, b60 = psdu(100, 31), psdu(60, 32)
    h11, h2 = synth.plcp_11b(100, 11000), synth.plcp_11b(60, 2000)
    s55 = synth.plcp_11b(90, 5500)
    specs = [(11000, b100, None), (2000, b60, h2 + (0x0100,)), (2000, b60, None), (5500, psdu(90, 33), (s55[0], s55[1] | 8, s55[2], 0)),
             (11000, b100, h11 + (0x8000,)), (1000, psdu(30, 34), None)]
    cs, prev = [], (0, 0)
    for rate, body, hdr in specs:
        c = case_11b("s", rate, body, hdr, prev=prev); cs.append(c); prev = (c["expect"]["rate_kbps"], c["expect"]["length"])
    return _chain(cs, ("iq",))[0], [_expect(c, ("status", "rate_kbps", "length")) for c in cs]

def stream_11n(mcs_limit=11):
    """Decoded MCS 9, L-SIG refused (parity), HT-SIG CRC-8 failure, L-SIG refused (rate), MCS refused, L-SIG refused (LENGTH), decoded
    MCS 8.  ht_frame_mcs is never reset: an L-SIG refusal reports the MCS of the event before; lsig_length is zero again."""
    b = psdu(200, 41)
    nt = -(-(16 + 8 * 200 + 6) // 104) + 5; lw = synth.signal_word_11a(6000, (nt * 24 - 22) // 8)
    h9 = 9 | 200 << 8 | 0x07 << 24
    refused = 11 if mcs_limit <= 11 else 15
    bad_rate = (lw & ~0xF) | 0x7; bad_rate ^= (_odd_parity(bad_rate) ^ _odd_parity(lw)) << 17
    specs = [dict(mcs=9, body=b), dict(mcs=9, body=b, lsig_word=lw ^ 1 << 17), dict(mcs=9, body=b, htsig=(h9, 0x10)),
             dict(mcs=9, body=b, lsig_word=bad_rate), dict(mcs=9, body=b, htsig=(h9 & ~0x7F | refused, 0)),
             dict(mcs=9, body=b, lsig_word=synth.signal_word_11a(6000, 751)), dict(mcs=8, body=psdu(150, 42))]
    cs, prev = [], 0
    for sp in specs:
        c = case_11n("s", sp.pop("mcs"), sp.pop("body"), mcs_limit=mcs_limit, prev_mcs=prev, **sp); cs.append(c); prev = c["expect"]["mcs"]
    iq0, iq1 = _chain(cs, ("iq0", "iq1"))
    return iq0, iq1, [_expect(c, ("status", "mcs", "length", "nsym", "lsig_length")) for c in cs]
