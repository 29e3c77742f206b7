"""Restatement of the reference's legacy 802.11b encoder — TEST INFRASTRUCTURE (checker only, never the product path).

BB11BPMDBufferTx4XWith{Long,Short}Header (kernel/bb/dot11b/bbb_tx.c:508-758) over the look-up tables of bbb_scramble.c, bbb_dbpsk.c,
bbb_dqpsk.c, bbb_cck5.c and bbb_cck11.c and CalcCRC16 (kernel/core/inc/CRC16.h).  The tables are regenerated here from closed forms and
checked entry for entry against the compiled ones (oracle/_ref/libtx11b_legacy_ref.so, oracle/build_ref_tx11b.sh):

  * scrambler  LUT[x][reg]: x^-4 + x^-7 self-synchronising, bit-serial LSB first, reg bit 6 = newest output; the caller sets reg = out >> 1;
  * CRC-16     reflected CCITT (0x8408), LUT[i] = CRC of byte i from 0; CalcCRC16 starts at 0xFFFF and inverts;
  * DBPSK      [byte][ref 0|1] 88 chips: per bit (LSB first) ref ^= bit, then 11 chips ref ? +Barker : -Barker; +1 -> +127, -1 -> -128;
  * DQPSK      [byte][ref 0..3] 44 chips: phase in quarter turns, ref 0 -> 2 (-1), 1 -> 3 (-j), 2 -> 1 (+j), 3 -> 0 (+1); per dibit
               (LSB first) phase += {0, 3, 1, 2}[dibit], then 11 chips j^phase * Barker, amplitude 127 (DQPSK_POSITIVE_SQRT_TWO = 90 is
               defined in bbb_dqpsk.c but no entry uses it);
  * CCK 5.5    [byte][ref] 16 chips, two 4-bit symbols, the second with an extra pi: phi1 = ref + {0, 3, 1, 2}[d0 d1], phi2 = 1 + 2 d2,
               phi3 = 0, phi4 = 2 d3 (quarter turns); chips j^(phi1+phi2+phi3+phi4), j^(phi1+phi3+phi4), j^(phi1+phi2+phi4), -j^(phi1+phi4),
               j^(phi1+phi2+phi3), j^(phi1+phi3), -j^(phi1+phi2), j^phi1, amplitude 127;
  * CCK 11     [byte][ref][even 0 | odd 1] 8 chips: phi1 = ref + {0, 3, 1, 2}[d0 d1] (+ pi when odd), phi2..4 = {0, 2, 1, 3}[d2 d3 | d4 d5 | d6 d7];
  * every table's bNewRef is the ref code of the last phase (DBPSK: the last bit's ref).

The frame (bbb_tx.c:508-758): long = SYNC 0xFF x 16, SFD 0xF3A0; short = SYNC 0x00 x 7, SFD 0x05CF; then SIGNAL (rate code), SERVICE (bit 7
= length extension), LENGTH (PLCPGetLength, bbb_tx.c:39-65), CRC-16 over SIGNAL .. LENGTH.  PLCP frame, PSDU and FCS are scrambled as one
stream (seed 0x6C long, 0x1B short), rewriting the caller's buffer.  Long: the 24 PLCP bytes DBPSK; short: 9 preamble bytes DBPSK, the 6
header bytes DQPSK; ref is turned from BPSK into QPSK form with ref |= ref << 1 before any DQPSK / CCK section (1 Mbps long keeps it).  The
short-preamble code has no 1 Mbps data case (bbb_tx.c:563-605): such a frame is preamble and header only.  Each chip is followed by three
zero samples, then TX_FIR_DEPTH = 37 zero samples, rounded up so that the total is a multiple of 128.
"""
import numpy as np

BARKER = np.array([1, -1, 1, 1, -1, 1, 1, 1, -1, -1, -1])
RATE_CODE = {1000: 0x0A, 2000: 0x14, 5500: 0x37, 11000: 0x6E}         # bb/bbb.h:47-50
Q_OF_REF = [2, 3, 1, 0]                                                  # ref code -> quarter turns of the phase it stands for
REF_OF_Q = [3, 2, 0, 1]
DQPSK_ROT = [0, 3, 1, 2]
CCK11_PHI = [0, 2, 1, 3]
UNIT = [(1, 0), (0, 1), (-1, 0), (0, -1)]


def _c8(q, amp_pos=127, amp_neg=-127):
    re, im = UNIT[q % 4]
    f = lambda v: amp_pos if v > 0 else amp_neg if v < 0 else 0
    return f(re), f(im)


def scrambler_lut():
    t = np.zeros((256, 128), np.uint8)
    for x in range(256):
        for reg in range(128):
            s, o, b = reg, 0, x
            for k in range(8):
                bit = (b ^ s ^ (s >> 3)) & 1
                s = (s >> 1) | (bit << 6); o |= bit << k; b >>= 1
            t[x, reg] = o
    return t


def crc16_lut():
    t = np.zeros(256, np.uint16)
    for i in range(256):
        c = i
        for _ in range(8): c = (c >> 1) ^ 0x8408 if c & 1 else c >> 1
        t[i] = c
    return t


def dbpsk_lut():
    """-> values int8 [256, 2, 88, 2], new ref uint8 [256, 2]"""
    v = np.zeros((256, 2, 88, 2), np.int8); nr = np.zeros((256, 2), np.uint8)
    for x in range(256):
        for r in range(2):
            p = r
            for b in range(8):
                p ^= (x >> b) & 1
                for k in range(11): v[x, r, 11 * b + k] = _c8((0 if p else 2) + (2 if BARKER[k] < 0 else 0), 127, -128)
            nr[x, r] = p
    return v, nr


def dqpsk_lut():
    v = np.zeros((256, 4, 44, 2), np.int8); nr = np.zeros((256, 4), np.uint8)
    for x in range(256):
        for r in range(4):
            q = Q_OF_REF[r]
            for s in range(4):
                q = (q + DQPSK_ROT[(x >> (2 * s)) & 3]) % 4
                for k in range(11): v[x, r, 11 * s + k] = _c8(q + (2 if BARKER[k] < 0 else 0))
            nr[x, r] = REF_OF_Q[q]
    return v, nr


def _cck8(p1, p2, p3, p4):
    return [_c8(q) for q in (p1 + p2 + p3 + p4, p1 + p3 + p4, p1 + p2 + p4, p1 + p4 + 2, p1 + p2 + p3, p1 + p3, p1 + p2 + 2, p1)]


def cck5_lut():
    v = np.zeros((256, 4, 16, 2), np.int8); nr = np.zeros((256, 4), np.uint8)
    for x in range(256):
        for r in range(4):
            q = Q_OF_REF[r]
            for s in range(2):
                n = (x >> (4 * s)) & 15
                q = (q + DQPSK_ROT[n & 3] + (2 if s else 0)) % 4
                v[x, r, 8 * s: 8 * s + 8] = _cck8(q, 1 + 2 * ((n >> 2) & 1), 0, 2 * ((n >> 3) & 1))
            nr[x, r] = REF_OF_Q[q]
    return v, nr


def cck11_lut():
    v = np.zeros((256, 4, 2, 8, 2), np.int8); nr = np.zeros((256, 4, 2), np.uint8)
    for x in range(256):
        for r in range(4):
            for e in range(2):
                q = (Q_OF_REF[r] + DQPSK_ROT[x & 3] + 2 * e) % 4
                v[x, r, e] = _cck8(q, CCK11_PHI[(x >> 2) & 3], CCK11_PHI[(x >> 4) & 3], CCK11_PHI[(x >> 6) & 3])
                nr[x, r, e] = REF_OF_Q[q]
    return v, nr


_T = None
def tables():
    global _T
    if _T is None:
        _T = dict(scr=scrambler_lut(), crc16=crc16_lut(), dbpsk=dbpsk_lut(), dqpsk=dqpsk_lut(), cck5=cck5_lut(), cck11=cck11_lut())
    return _T


def plcp_length(size_with_fcs, rate_kbps):
    """PLCPGetLength (bbb_tx.c:39-65) for CCK: (LENGTH in microseconds, length-extension bit)"""
    s = size_with_fcs
    if rate_kbps == 1000: return s << 3, 0
    if rate_kbps == 2000: return s << 2, 0
    if rate_kbps == 5500: return ((s << 4) - 1) // 11 + 1, 0
    ret = ((s << 3) - 1) // 11 + 1
    return ret, 1 if ret * 11 - (s << 3) >= 8 else 0


def encode(psdu_with_fcs, rate_kbps, short_preamble=False):
    """BB11BPMDBufferTx4XWith{Short,Long}Header.  psdu_with_fcs: MPDU + FCS (>= 4 bytes).  Returns (int8 [n, 2] at 44 Msps, n % 128 == 0;
    the scrambled bytes the reference leaves in the caller's buffer)."""
    T = tables()
    d = bytes(np.asarray(psdu_with_fcs, np.uint8))
    code = RATE_CODE[rate_kbps]
    ln, ext = plcp_length(len(d), rate_kbps)
    hdr = [code, ext << 7, ln & 0xFF, (ln >> 8) & 0xFF]
    c = 0xFFFF
    for b in hdr: c = (c >> 8) ^ int(T["crc16"][(c & 0xFF) ^ b])
    c = ~c & 0xFFFF
    hdr += [c & 0xFF, c >> 8]
    pre = [0x00] * 7 + [0xCF, 0x05] if short_preamble else [0xFF] * 16 + [0xA0, 0xF3]
    stream = pre + hdr + list(d)
    reg = 0x1B if short_preamble else 0x6C
    scr = []
    for b in stream:
        o = int(T["scr"][b, reg]); scr.append(o); reg = o >> 1
    plcp = len(pre) + 6
    chips = []
    dbv, dbr = T["dbpsk"]; dqv, dqr = T["dqpsk"]
    ref = 0
    n_dbpsk = len(pre) if short_preamble else plcp
    for b in scr[:n_dbpsk]:
        chips.append(dbv[b, ref]); ref = int(dbr[b, ref])
    data = scr[plcp:]
    if short_preamble:
        ref |= ref << 1
        for b in scr[n_dbpsk:plcp]:
            chips.append(dqv[b, ref]); ref = int(dqr[b, ref])
        if rate_kbps == 1000: data = []                      # no 1 Mbps case in the short-preamble switch
    elif rate_kbps != 1000:
        ref |= ref << 1
    even = 0
    for b in data:
        if rate_kbps == 1000: chips.append(dbv[b, ref]); ref = int(dbr[b, ref])
        elif rate_kbps == 2000: chips.append(dqv[b, ref]); ref = int(dqr[b, ref])
        elif rate_kbps == 5500: v, r = T["cck5"]; chips.append(v[b, ref]); ref = int(r[b, ref])
        else: v, r = T["cck11"]; chips.append(v[b, ref, even]); ref = int(r[b, ref, even]); even ^= 1
    ch = np.concatenate(chips) if chips else np.zeros((0, 2), np.int8)
    n = 4 * len(ch)
    pad = 37
    if (pad + n) & 127: pad += 128 - ((pad + n) & 127)
    out = np.zeros((n + pad, 2), np.int8)
    out[0:n:4] = ch
    return out, np.array(scr[plcp:], np.uint8)


def crc32(b):
    import zlib
    return zlib.crc32(bytes(np.asarray(b, np.uint8)))


def modulate(payload, rate_kbps, short_preamble=False, filt=0, fcs_in_payload=False):
    """What sb200_tx11b_legacy_batch writes for one frame: payload = MPDU (the FCS is appended) or, with fcs_in_payload, MPDU + FCS sent
    verbatim; filt 0 = encoder output, 1 = BB11BPMDSpreadFIR4SSE over it, 2 = BB11BPMDSpreadFIR4ASM (oracle/tx11b_legacy.cpp)."""
    p = np.asarray(payload, np.uint8)
    psdu = p if fcs_in_payload else np.concatenate([p, np.frombuffer(crc32(p).to_bytes(4, "little"), np.uint8)])
    enc, _ = encode(psdu, rate_kbps, short_preamble)
    if filt == 0: return enc
    import oracle_py
    return oracle_py.fir37_legacy(enc, filt - 1)


# ---- the compiled reference (oracle/_ref, built by oracle/build_ref_tx11b.sh where the reference tree exists) ----------------------------
import os, ctypes as C
_REF_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libtx11b_legacy_ref.so")
_REF = None
def ref_available():
    return os.path.exists(_REF_SO)

def _ref():
    global _REF
    if _REF is None:
        _REF = C.CDLL(_REF_SO); _REF.ref_tx11b_table.restype = C.c_void_p
    return _REF

def ref_encode(psdu_with_fcs, rate_kbps, short_preamble=False):
    """The reference's own compiled BB11BPMDBufferTx4XWith{Short,Long}Header: (int8 [n, 2], scrambled PSDU + FCS)."""
    d = np.ascontiguousarray(psdu_with_fcs, np.uint8)
    cap = 4 * (24 * 88 + len(d) * 88) + 256
    out = np.zeros((cap, 2), np.int8); scr = np.zeros(max(len(d), 1), np.uint8); n = C.c_uint(0)
    r = _ref().ref_tx11b_legacy(C.c_void_p(d.ctypes.data), C.c_uint(len(d)), C.c_uint(RATE_CODE[rate_kbps]), C.c_uint(1 if short_preamble else 0),
                                C.c_void_p(out.ctypes.data), C.byref(n), C.c_void_p(scr.ctypes.data))
    assert r == 0
    return out[:n.value].copy(), scr[:len(d)].copy()

def ref_table(which):
    """Raw bytes of compiled table `which`: 0 scrambler, 1 DBPSK, 2 DQPSK, 3 CCK 5.5, 4 CCK 11, 5 CRC-16."""
    n = C.c_uint(0); p = _ref().ref_tx11b_table(C.c_int(which), C.byref(n))
    return np.frombuffer((C.c_uint8 * n.value).from_address(p), np.uint8).copy()
