"""Synthetic 802.11a PPDU generator (numpy, float IFFT) in the reference's amplitude convention.

Test/bench infrastructure: produces int16 interleaved IQ at 40 Msps exactly shaped like the output of the
reference's offline modulator after `ConvertModFile2DumpFile_8b`:
  * pre-IFFT BPSK amplitude 10720, QPSK/16/64-QAM scaled by 1/sqrt(2,10,42)   (Brick11/src/mapper11a.hpp:8-11)
  * 128-point IFFT (2x oversampled), result / 16                                (Brick11/src/fft.hpp:51-58)
  * saturate to int8, then << 8 into COMPLEX16                                  (brick/inc/stdbrick.hpp:437, demod11/modulate11a.cpp:178-179)
  * STS amplitude 1.472 x BPSK, LTS = BPSK amplitude                            (Brick11/src/preamble11a.hpp:15-16)
The bit pipeline is 802.11a-1999 clause 17 (scramble x^7+x^4+1, K=7 133/171, puncture, interleave, Gray map, pilots).
It is a float modulator, not a restatement of the reference's fixed-point TX, so it never serves as a parity oracle —
only as an input source; parity is always GPU-vs-oracle on the same IQ.
"""
import numpy as np
import zlib

RATES = {  # kbps: (rate bits R1-R4 as SIGNAL[3:0] value, N_BPSC, coding 'num/den', N_DBPS)
    6000: (0xB, 1, (1, 2), 24), 9000: (0xF, 1, (3, 4), 36), 12000: (0xA, 2, (1, 2), 48), 18000: (0xE, 2, (3, 4), 72),
    24000: (0x9, 4, (1, 2), 96), 36000: (0xD, 4, (3, 4), 144), 48000: (0x8, 6, (2, 3), 192), 54000: (0xC, 6, (3, 4), 216),
}
BPSK_MOD = 10720
KMOD = {1: 10720, 2: int(10720 / 1.414), 4: int(10720 / 3.162), 6: int(10720 / 6.481)}
_LTS = np.array([1,1,-1,-1,1,1,-1,1,-1,1,1,1,1,1,1,-1,-1,1,1,-1,1,-1,1,1,1,1,0,
                 1,-1,-1,1,1,-1,1,-1,1,-1,-1,-1,-1,-1,1,1,-1,-1,1,-1,1,-1,1,1,1,1], dtype=np.float64)

_SCR_CACHE = {}
def scrambler_seq(seed, n):
    """seed: 7-bit initial state, bit6 = x7 ... bit0 = x1.  Returns n output bits."""
    seed &= 0x7F
    out = _SCR_CACHE.get(seed)
    if out is None:
        st = seed
        out = np.zeros(127, np.uint8)
        for i in range(127):
            b = ((st >> 6) ^ (st >> 3)) & 1
            st = ((st << 1) | b) & 0x7F
            out[i] = b
        _SCR_CACHE[seed] = out
    return np.resize(out, n)

_PILOT_POL = 1 - 2 * scrambler_seq(0x7F, 127).astype(np.int64)   # p_0..p_126

def interleave_map(ncbps, nbpsc):
    s = max(nbpsc // 2, 1)
    k = np.arange(ncbps)
    i = (ncbps // 16) * (k % 16) + k // 16
    return s * (i // s) + (i + ncbps - (16 * i) // ncbps) % s      # j = position on air of coded bit k

def conv_encode(bits):
    """bits [..., n] uint8 -> (A, B) each [..., n]; encoder starts from the all-zero state."""
    pad = np.zeros(bits.shape[:-1] + (6,), np.uint8)
    x = np.concatenate([pad, bits], -1)
    n = bits.shape[-1]
    d = lambda k: x[..., 6 - k: 6 - k + n]
    A = d(0) ^ d(2) ^ d(3) ^ d(5) ^ d(6)
    B = d(0) ^ d(1) ^ d(2) ^ d(3) ^ d(6)
    return A, B

def puncture(A, B, rate):
    n = A.shape[-1]
    if rate == (1, 2):
        return np.stack([A, B], -1).reshape(A.shape[:-1] + (2 * n,))
    if rate == (3, 4):
        a = A.reshape(A.shape[:-1] + (n // 3, 3)); b = B.reshape(B.shape[:-1] + (n // 3, 3))
        return np.stack([a[..., 0], b[..., 0], a[..., 1], b[..., 2]], -1).reshape(A.shape[:-1] + (n // 3 * 4,))
    a = A.reshape(A.shape[:-1] + (n // 2, 2)); b = B.reshape(B.shape[:-1] + (n // 2, 2))
    return np.stack([a[..., 0], b[..., 0], a[..., 1]], -1).reshape(A.shape[:-1] + (n // 2 * 3,))

_GRAY = {1: np.array([-1, 1.]), 2: np.array([-3, 3, -1, 1.]),  # index = b0 | b1<<1 ... (first bit in LSB)
         3: np.array([-7, 7, -1, 1, -5, 5, -3, 3.])}
# 16-QAM: b0b1 = 00->-3, 01->-1, 11->+1, 10->+3 ; index b0|b1<<1: 0:-3, 1(b0=1,b1=0):+3, 2(b0=0,b1=1):-1, 3:+1
# 64-QAM: b0b1b2: 000:-7 001:-5 011:-3 010:-1 110:+1 111:+3 101:+5 100:+7 ; index b0|b1<<1|b2<<2:
#   0:-7, 1(100):+7, 2(010):-1, 3(110):+1, 4(001):-5, 5(101):+5, 6(011):-3, 7(111):+3

def map_symbols(bits_air, nbpsc):
    """bits_air [..., nsym, 48*nbpsc] -> complex [..., nsym, 48] (unscaled levels x kmod)."""
    sh = bits_air.shape[:-1]
    b = bits_air.reshape(sh + (48, nbpsc)).astype(np.int64)
    if nbpsc == 1:
        return (_GRAY[1][b[..., 0]] + 0j) * KMOD[1]
    h = nbpsc // 2
    w = (1 << np.arange(h))
    ii = (b[..., :h] * w).sum(-1); qq = (b[..., h:] * w).sum(-1)
    return (_GRAY[h][ii] + 1j * _GRAY[h][qq]) * KMOD[nbpsc]

def _ofdm_td(freq64):
    """freq64 [..., 64] complex in FFT order -> [..., 160] time samples at 40 Msps incl. 32-sample GI."""
    X = np.zeros(freq64.shape[:-1] + (128,), np.complex128)
    X[..., :32] = freq64[..., :32]; X[..., 96:] = freq64[..., 32:]
    td = np.fft.ifft(X, axis=-1) / 16.0          # ifft already divides by 128 (3 radix stages of the fixed-point IFFT<128>)
    out = np.concatenate([td[..., 96:], td], -1)
    return out

def _place(data48, pilot_pol):
    """data48 [..., nsym, 48] complex, pilot_pol [nsym] (+1/-1) -> [..., nsym, 64] FFT-order."""
    f = np.zeros(data48.shape[:-1] + (64,), np.complex128)
    neg = [k for k in range(-26, 0) if k not in (-21, -7)]
    pos = [k for k in range(1, 27) if k not in (7, 21)]
    idx = np.array([k % 64 for k in neg + pos])
    f[..., idx] = data48
    pp = pilot_pol.reshape((1,) * (data48.ndim - 2) + (-1,))
    f[..., 7] = BPSK_MOD * pp; f[..., 21] = -BPSK_MOD * pp; f[..., 64 - 7] = BPSK_MOD * pp; f[..., 64 - 21] = BPSK_MOD * pp
    return f

def preamble_td():
    S = np.zeros(64, np.complex128)
    a = BPSK_MOD * 1.472 * (1 + 1j)
    for k, s in ((4, -1), (8, -1), (12, 1), (16, 1), (20, 1), (24, 1), (-24, 1), (-20, -1), (-16, 1), (-12, -1), (-8, -1), (-4, 1)):
        S[k % 64] = s * a
    X = np.zeros(128, np.complex128); X[:32] = S[:32]; X[96:] = S[32:]
    sts = np.fft.ifft(X) / 16.0
    sts = np.tile(sts, 3)[:320]
    L = np.zeros(64, np.complex128)
    for k in range(-26, 27):
        L[k % 64] = _LTS[k + 26] * BPSK_MOD
    X = np.zeros(128, np.complex128); X[:32] = L[:32]; X[96:] = L[32:]
    lt = np.fft.ifft(X) / 16.0
    lts = np.concatenate([lt[64:], lt, lt])
    return np.concatenate([sts, lts])               # 640 samples @ 40 Msps

def psdu_with_fcs(payload):
    payload = np.asarray(payload, np.uint8)
    fcs = zlib.crc32(payload.tobytes()) & 0xFFFFFFFF
    return np.concatenate([payload, np.frombuffer(fcs.to_bytes(4, "little"), np.uint8)])

def signal_word_11a(rate_kbps, length):
    """The 24-bit SIGNAL field (bit i = i-th bit on air) of a frame of `length` PSDU bytes: RATE, reserved 0, LENGTH, even parity, tail 0."""
    w = RATES[rate_kbps][0] | (length & 0xFFF) << 5
    return w | (bin(w).count("1") & 1) << 17

def modulate(psdus, rate_kbps=54000, scramble_seeds=None, window=True, signal_word=None):
    """psdus: uint8 [F, L] (L >= 0 bytes each, FCS already included).  Returns complex128 [F, nsamp] time signal in
    int8-LSB units (i.e. what TPackSample16to8 would saturate), 640 + 160*(1+Nsym) samples at 40 Msps.
    signal_word: the 24 SIGNAL bits to send instead of signal_word_11a(rate_kbps, L); the DATA field is still the PSDU at rate_kbps."""
    psdus = np.atleast_2d(np.asarray(psdus, np.uint8))
    F, L = psdus.shape
    rbits, nbpsc, cr, ndbps = RATES[rate_kbps]
    nsym = -(-(16 + 8 * L + 6) // ndbps)
    ndata = nsym * ndbps
    if scramble_seeds is None:
        scramble_seeds = 1 + (np.arange(F) % 127)
    bits = np.zeros((F, ndata), np.uint8)
    bits[:, 16:16 + 8 * L] = np.unpackbits(psdus, axis=1, bitorder="little")
    seq = np.stack([scrambler_seq(int(s), ndata) for s in np.asarray(scramble_seeds).reshape(-1)])
    bits ^= seq
    bits[:, 16 + 8 * L: 16 + 8 * L + 6] = 0            # tail bits forced to zero after scrambling
    A, B = conv_encode(bits)
    coded = puncture(A, B, cr).reshape(F, nsym, 48 * nbpsc)
    jmap = interleave_map(48 * nbpsc, nbpsc)
    air = np.zeros_like(coded); air[..., jmap] = coded
    data = map_symbols(air, nbpsc)
    pol = _PILOT_POL[(np.arange(nsym) + 1) % 127]
    td_data = _ofdm_td(_place(data, pol))               # [F, nsym, 160]
    # SIGNAL
    sw = signal_word_11a(rate_kbps, L) if signal_word is None else int(signal_word)
    sig = np.array([(sw >> i) & 1 for i in range(24)], np.uint8)
    As, Bs = conv_encode(sig)
    cs = puncture(As, Bs, (1, 2))
    j48 = interleave_map(48, 1)
    airs = np.zeros(48, np.uint8); airs[j48] = cs
    td_sig = _ofdm_td(_place(map_symbols(airs[None, :], 1), _PILOT_POL[:1]))[0]   # [160]
    syms = np.concatenate([np.broadcast_to(td_sig, (F, 1, 160)), td_data], 1)
    if window:
        syms = syms.copy(); syms[..., :2] *= 0.5; syms[..., 158:] *= 0.5
    pre = preamble_td()
    return np.concatenate([np.broadcast_to(pre, (F, 640)), syms.reshape(F, -1)], 1)

def to_iq16(td, gain=1.0, lead=32, trail=32, snr_db=None, cfo_hz=0.0, rng=None, phase=0.0):
    """complex time signal (int8 units) -> int16 IQ [F, lead+n+trail, 2]: saturate to int8, << 8, plus optional
    CFO (Hz at 40 Msps), AWGN at snr_db relative to the signal power, a constant gain and silent gaps."""
    td = np.atleast_2d(td)
    F, n = td.shape
    x = td * gain
    if cfo_hz or phase:
        x = x * np.exp(1j * (2 * np.pi * cfo_hz * np.arange(n) / 40e6 + phase))
    re = np.clip(np.round(x.real), -128, 127) * 256.0
    im = np.clip(np.round(x.imag), -128, 127) * 256.0
    out = np.zeros((F, lead + n + trail, 2), np.float64)
    out[:, lead:lead + n, 0] = re; out[:, lead:lead + n, 1] = im
    if snr_db is not None:
        rng = rng or np.random.default_rng(0)
        p = (re ** 2 + im ** 2).mean()
        sigma = np.sqrt(p / (10 ** (snr_db / 10)) / 2)
        out += rng.normal(0, sigma, out.shape)
    return np.clip(np.round(out), -32768, 32767).astype(np.int16)

def make_frames(nframes, psdu_len=1500, rate_kbps=54000, seed0=0x5EED0000, snr_db=None, lead=32, trail=32, cfo_hz=0.0, gain=1.0):
    """BASELINE config #2 shaped frames: PSDU = (psdu_len-4) random bytes from mt19937(seed0+i) + CRC-32,
    scrambler seed 1 + i % 127.  Returns (iq int16 [F, slot, 2], psdus uint8 [F, psdu_len])."""
    ps = np.zeros((nframes, psdu_len), np.uint8)
    for i in range(nframes):
        r = np.random.RandomState(seed=(seed0 + i) & 0xFFFFFFFF)
        ps[i] = psdu_with_fcs(r.randint(0, 256, psdu_len - 4).astype(np.uint8))
    td = modulate(ps, rate_kbps)
    rng = np.random.default_rng(seed0 & 0xFFFFFFFF)
    return to_iq16(td, gain=gain, lead=lead, trail=trail, snr_db=snr_db, cfo_hz=cfo_hz, rng=rng), ps


# =====================================================================================================================
# 802.11b (DSSS / CCK) PPDUs at 44 Msps (4 samples per chip), long preamble — IEEE 802.11b-1999 clause 18.
# Float modulator for test input only (same role as the 11a generator above).
# =====================================================================================================================
_BARKER = np.array([1, -1, 1, 1, -1, 1, 1, 1, -1, -1, -1], dtype=np.float64)
_SIGNAL_11B = {1000: 0x0A, 2000: 0x14, 5500: 0x37, 11000: 0x6E}

def _crc16_ccitt_reflected(data):
    c = 0xFFFF
    for b in data:
        c ^= b
        for _ in range(8):
            c = (c >> 1) ^ 0x8408 if c & 1 else c >> 1
    return (~c) & 0xFFFF

def _scramble_11b(bits, state=0x1B):
    """Self-synchronising scrambler s[k] = b[k] ^ s[k-4] ^ s[k-7]; `state` bit i = s[k-1-i]."""
    out = np.zeros_like(bits)
    st = state
    for k, b in enumerate(bits):
        s = int(b) ^ ((st >> 3) & 1) ^ ((st >> 6) & 1)
        out[k] = s
        st = ((st << 1) | s) & 0x7F
    return out

_DQPSK = {(0, 0): 0, (0, 1): 1, (1, 1): 2, (1, 0): 3}          # (d0, d1) -> quarter turns, counter-clockwise
_QPSK = {(0, 0): 0, (0, 1): 1, (1, 0): 2, (1, 1): 3}           # CCK phi2..phi4 encoding (Table 18-?): 00,01,10,11 -> 0, pi/2, pi, 3pi/2

def plcp_11b(L, rate_kbps):
    """(SIGNAL, SERVICE, LENGTH) of a long-preamble PLCP header for L PSDU bytes at rate_kbps."""
    service = 0x04                                      # locked clocks
    if rate_kbps == 11000:
        lp = L * 8 / 11.0; length = int(np.ceil(lp))
        if length - lp >= 8 / 11.0 - 1e-12: service |= 0x80
    elif rate_kbps == 5500:
        length = int(np.ceil(L * 8 / 5.5))
    else:
        length = L * 8 * 1000 // rate_kbps
    return _SIGNAL_11B[rate_kbps], service, length

def modulate_11b(psdu, rate_kbps=11000, amp=90.0, shape=True, plcp=None):
    """psdu: uint8 [L] (FCS included).  Returns complex chips-domain waveform at 44 Msps in int8 units.
    plcp: (SIGNAL, SERVICE, LENGTH, CRC-16 xor mask) to send instead of plcp_11b(L, rate_kbps) with a correct CRC-16;
    the PSDU is still modulated at rate_kbps."""
    psdu = np.asarray(psdu, np.uint8)
    signal, service, length, crc_xor = plcp_11b(len(psdu), rate_kbps) + (0,) if plcp is None else plcp
    hdr = bytes([signal & 0xFF, service & 0xFF, length & 0xFF, (length >> 8) & 0xFF])
    crc = _crc16_ccitt_reflected(hdr) ^ (crc_xor & 0xFFFF)
    hdr = hdr + bytes([crc & 0xFF, crc >> 8])
    bits = np.concatenate([np.ones(128, np.uint8),
                           np.unpackbits(np.frombuffer((0xF3A0).to_bytes(2, "little"), np.uint8), bitorder="little"),
                           np.unpackbits(np.frombuffer(hdr, np.uint8), bitorder="little"),
                           np.unpackbits(psdu, bitorder="little")])
    sb = _scramble_11b(bits)
    npre = 128 + 16 + 48
    chips = []
    ph = 0                                              # current phase in quarter turns
    for b in sb[:npre]:                                 # DBPSK 1 Mbps preamble + header
        ph = (ph + 2 * int(b)) & 3
        chips.append(_BARKER * np.exp(1j * np.pi / 2 * ph))
    d = sb[npre:]
    if rate_kbps == 1000:
        for b in d:
            ph = (ph + 2 * int(b)) & 3; chips.append(_BARKER * np.exp(1j * np.pi / 2 * ph))
    elif rate_kbps == 2000:
        for i in range(0, len(d), 2):
            ph = (ph + _DQPSK[(int(d[i]), int(d[i + 1]))]) & 3; chips.append(_BARKER * np.exp(1j * np.pi / 2 * ph))
    else:
        nb = 4 if rate_kbps == 5500 else 8
        for k, i in enumerate(range(0, len(d), nb)):
            w = [int(x) for x in d[i:i + nb]]
            ph = (ph + _DQPSK[(w[0], w[1])] + (2 if (k & 1) else 0)) & 3
            if nb == 4:
                p2 = 2 * w[2] + 1; p3 = 0; p4 = 2 * w[3]
            else:
                p2 = _QPSK[(w[2], w[3])]; p3 = _QPSK[(w[4], w[5])]; p4 = _QPSK[(w[6], w[7])]
            e = lambda q: np.exp(1j * np.pi / 2 * (q & 3))
            p1 = ph
            chips.append(np.array([e(p1 + p2 + p3 + p4), e(p1 + p3 + p4), e(p1 + p2 + p4), -e(p1 + p4),
                                   e(p1 + p2 + p3), e(p1 + p3), -e(p1 + p2), e(p1)]))
    c = np.concatenate(chips)
    x = np.repeat(c, 4)                                 # 4 samples per chip
    if shape:                                           # raised cosine, beta 0.5, +-3 chips: zero ISI at the chip centres
        n = np.arange(-12, 13); t = n / 4.0; beta = 0.5
        den = 1.0 - (2 * beta * t) ** 2
        h = np.sinc(t) * np.cos(np.pi * beta * t) / np.where(np.abs(den) < 1e-9, 1.0, den)
        h[np.abs(den) < 1e-9] = np.pi / 4 * np.sinc(1 / (2 * beta))
        imp = np.zeros(len(c) * 4, np.complex128); imp[::4] = c            # impulses at chip centres
        x = np.convolve(imp, h, mode="same")
    return x * amp

def make_frames_11b(nframes, psdu_len=1500, rate_kbps=11000, seed0=0xB11B0000, snr_db=None, lead=400, trail=200, gain=1.0, cfo_hz=0.0):
    """Returns (iq int16 [F, slot, 2], psdus uint8 [F, psdu_len]); slot length is a multiple of 28."""
    ps = np.zeros((nframes, psdu_len), np.uint8); tds = []
    for i in range(nframes):
        r = np.random.RandomState(seed=(seed0 + i) & 0xFFFFFFFF)
        ps[i] = psdu_with_fcs(r.randint(0, 256, psdu_len - 4).astype(np.uint8))
        tds.append(modulate_11b(ps[i], rate_kbps))
    n = len(tds[0])
    tot = lead + n + trail; trail += (-tot) % 28
    rng = np.random.default_rng(seed0 & 0xFFFFFFFF)
    td = np.stack(tds)
    if cfo_hz:
        td = td * np.exp(2j * np.pi * cfo_hz * np.arange(n) / 44e6)
    return to_iq16(td, gain=gain, lead=lead, trail=trail, snr_db=snr_db, rng=rng), ps


# =====================================================================================================================
# 802.11n HT mixed format, 20 MHz, 2 spatial streams, direct mapping onto 2 transmit chains (IEEE 802.11n-2009 clause 20),
# MCS 8..10 — the ones the reference's HT-SIG parser admits (Brick11/src/PHY_11n.hpp:496-501) — and MCS 11..14 (16-QAM / 64-QAM), which its
# graphs carry and the engine decodes with option ht_mcs_limit = 15.  Float modulator, test input only.
# =====================================================================================================================
HT_MCS = {8: (1, (1, 2), 52), 9: (2, (1, 2), 104), 10: (2, (3, 4), 156),       # mcs: (N_BPSC per stream, code rate, N_DBPS)
          11: (4, (1, 2), 208), 12: (4, (3, 4), 312), 13: (6, (2, 3), 416), 14: (6, (3, 4), 468)}

def _crc8_htsig(b, nbytes=4, tail_bits=2):
    """CRC-8 x^8+x^2+x+1 as the reference computes it (core/inc/CRC8.h:29-50): reflected, init 0xFF, inverted."""
    crc = 0xFF
    def step(c, nb):
        for _ in range(nb): c = (c >> 1) ^ 0xE0 if c & 1 else c >> 1
        return c
    for i in range(nbytes): crc = step(crc ^ int(b[i]), 8)
    crc = step(crc ^ (int(b[nbytes]) & ((1 << tail_bits) - 1)), tail_bits)
    return (~crc) & 0xFF

def ht_interleave_map(nbpsc, iss):
    """position on air of coded bit k of spatial stream iss (0-based), 20 MHz: N_COL 13, N_ROW 4*N_BPSC, N_ROT 11."""
    ncbpss = 52 * nbpsc; s = max(nbpsc // 2, 1); k = np.arange(ncbpss)
    i = 4 * nbpsc * (k % 13) + k // 13
    j = s * (i // s) + (i + ncbpss - (13 * i) // ncbpss) % s
    return (j - ((iss * 2) % 3 + 3 * (iss // 3)) * 11 * nbpsc) % ncbpss

def _csd(freq64, shift20):
    """cyclic shift by -shift20 samples at 20 Msps (advance), applied per carrier in FFT order."""
    k = np.fft.fftfreq(64, 1 / 64.0)
    return freq64 * np.exp(2j * np.pi * k * shift20 / 64.0)

def _td_plain(freq64, n):
    """n-sample periodic extension (40 Msps) of one 128-sample IFFT period, ending at the period end."""
    X = np.zeros(128, np.complex128); X[:32] = freq64[:32]; X[96:] = freq64[32:]
    p = np.fft.ifft(X) / 16.0
    reps = -(-n // 128) + 1
    return np.tile(p, reps)[-n:]

def modulate_11n(psdus, mcs=8, scramble_seeds=None, lsig_word=None, htsig=None):
    """psdus uint8 [F, L] (FCS included) -> complex128 [F, 2, nsamp]: the two transmit chains at 40 Msps, int8 units.
    lsig_word: the 24 L-SIG bits to send instead of 6 Mbps with the spoofed length; htsig: (first 34 HT-SIG bits, CRC-8 xor mask)
    instead of (MCS | L << 8 | 0x07 << 24, 0).  The data field is still the PSDU at `mcs`."""
    psdus = np.atleast_2d(np.asarray(psdus, np.uint8)); F, L = psdus.shape
    nbpsc, cr, ndbps = HT_MCS[mcs]
    nsym = -(-(16 + 8 * L + 6) // ndbps); ndata = nsym * ndbps
    if scramble_seeds is None: scramble_seeds = 1 + (np.arange(F) % 127)
    A0 = BPSK_MOD / np.sqrt(2.0)                                    # per-chain tone amplitude
    # ---- legacy preamble + L-SIG + HT-SIG (chain 2: 200 ns = 4-sample cyclic shift) ----
    S = np.zeros(64, np.complex128)
    for k, s in ((4, -1), (8, -1), (12, 1), (16, 1), (20, 1), (24, 1), (-24, 1), (-20, -1), (-16, 1), (-12, -1), (-8, -1), (-4, 1)):
        S[k % 64] = s * 1.472 * (1 + 1j)
    Lf = np.zeros(64, np.complex128)
    for k in range(-26, 27): Lf[k % 64] = _LTS[k + 26]
    nt = nsym + 5
    lsig_len = (nt * 24 - 22) // 8
    lw = signal_word_11a(6000, lsig_len) if lsig_word is None else int(lsig_word)
    sig = np.array([(lw >> i) & 1 for i in range(24)], np.uint8)
    j48 = interleave_map(48, 1)
    def bpsk48(bits24_or_48):
        a, b = conv_encode(bits24_or_48); c = puncture(a, b, (1, 2)).reshape(-1, 48)
        air = np.zeros_like(c); air[:, j48] = c
        return 2.0 * air - 1.0
    lsig_f = _place(bpsk48(sig)[None, :, :] * BPSK_MOD, _PILOT_POL[:1])[0, 0] / BPSK_MOD
    td = np.zeros((F, 2, 640 + 160 * (nt + 1)), np.complex128)
    for fidx in range(F):
        h34, c8x = (mcs | L << 8 | 0x07 << 24, 0) if htsig is None else htsig
        hb = np.frombuffer((int(h34) & ((1 << 34) - 1)).to_bytes(6, "little"), np.uint8).copy()
        c8 = _crc8_htsig(hb) ^ (c8x & 0xFF); hb[4] |= (c8 << 2) & 0xFF; hb[5] |= c8 >> 6
        hbits = np.unpackbits(hb, bitorder="little")
        hs = _place(bpsk48(hbits)[None, :, :] * BPSK_MOD, _PILOT_POL[1:3])[0] / BPSK_MOD          # [2, 64]
        hs = np.where(np.abs(hs) > 0, hs, 0); data_mask = np.ones(64, bool); data_mask[[7, 21, 57, 43]] = False
        hs[:, data_mask] = hs[:, data_mask] * 1j                                                   # QBPSK on the data tones
        # ---- data field ----
        bits = np.zeros(ndata, np.uint8); bits[16:16 + 8 * L] = np.unpackbits(psdus[fidx], bitorder="little")
        bits ^= scrambler_seq(int(np.asarray(scramble_seeds).reshape(-1)[fidx]), ndata); bits[16 + 8 * L:16 + 8 * L + 6] = 0
        a, b = conv_encode(bits); coded = puncture(a, b, cr).reshape(nsym, 2 * 52 * nbpsc)
        for ch in range(2):
            sh_leg, sh_ht = (0, 0) if ch == 0 else (4, 8)
            parts = [_td_plain(_csd(S, sh_leg) * A0, 320), _td_plain(_csd(Lf, sh_leg) * A0, 320)]
            for f in (lsig_f, hs[0], hs[1]): parts.append(_ofdm_td(_csd(f, sh_leg) * A0))
            parts.append(_ofdm_td(_csd(S, sh_ht) * A0))                                            # HT-STF
            H = Lf.copy(); H[27] = H[28] = -1; H[64 - 28] = H[64 - 27] = 1
            P = ((1, -1), (1, 1))[ch]
            for n in range(2): parts.append(_ofdm_td(_csd(H, sh_ht) * A0 * P[n]))
            sblk = max(nbpsc // 2, 1)                                                               # stream parser: s = max(N_BPSC / 2, 1) bits per stream in turn
            sb = coded.reshape(nsym, -1, 2, sblk)[:, :, ch, :].reshape(nsym, 52 * nbpsc)
            jm = ht_interleave_map(nbpsc, ch)
            air = np.zeros_like(sb); air[:, jm] = sb
            if nbpsc == 1: pts = 2.0 * air - 1.0 + 0j
            elif nbpsc == 2: q = air.reshape(nsym, 52, 2); pts = ((2.0 * q[..., 0] - 1) + 1j * (2.0 * q[..., 1] - 1)) / np.sqrt(2.0)
            else:                                                                                   # Gray-coded 16-QAM / 64-QAM, unit average power (clause 17.3.5.7 levels)
                h = nbpsc // 2; q = air.reshape(nsym, 52, nbpsc).astype(np.int64); w = (1 << np.arange(h))
                ii = (q[..., :h] * w).sum(-1); qq = (q[..., h:] * w).sum(-1)
                pts = (_GRAY[h][ii] + 1j * _GRAY[h][qq]) / np.sqrt(10.0 if h == 2 else 42.0)
            fr = np.zeros((nsym, 64), np.complex128)
            idx = np.array([k % 64 for k in list(range(-28, 0)) + list(range(1, 29)) if k not in (-21, -7, 7, 21)])
            fr[:, idx] = pts
            psi = ((1, 1, -1, -1), (1, -1, -1, 1))[ch]
            for n in range(nsym):
                pol = _PILOT_POL[(n + 3) % 127]
                for m, k in enumerate((-21, -7, 7, 21)): fr[n, k % 64] = pol * psi[(n + m) % 4]
            parts.append(_ofdm_td(_csd(fr, sh_ht) * A0).reshape(-1))
            sig_td = np.concatenate(parts)
            td[fidx, ch, :len(sig_td)] = sig_td
    return td

def make_frames_11n(nframes, psdu_len=1500, mcs=8, seed0=0x11A0000, snr_db=None, lead=64, trail=64, cfo_hz=0.0, gain=1.0,
                    chan=((1.0, 0.3j), (-0.2, 0.9))):
    """2x2 frames through a flat channel `chan` (rx = chan @ tx).  Returns (iq0, iq1 int16 [F, slot, 2], psdus [F, L])."""
    ps = np.zeros((nframes, psdu_len), np.uint8)
    for i in range(nframes):
        r = np.random.RandomState(seed=(seed0 + i) & 0xFFFFFFFF)
        ps[i] = psdu_with_fcs(r.randint(0, 256, psdu_len - 4).astype(np.uint8))
    tx = modulate_11n(ps, mcs)
    Hm = np.asarray(chan, np.complex128)
    rx = np.einsum("ab,fbn->fan", Hm, tx)
    rng = np.random.default_rng(seed0 & 0xFFFFFFFF)
    iq0 = to_iq16(rx[:, 0], gain=gain, lead=lead, trail=trail, snr_db=snr_db, cfo_hz=cfo_hz, rng=rng)
    iq1 = to_iq16(rx[:, 1], gain=gain, lead=lead, trail=trail, snr_db=snr_db, cfo_hz=cfo_hz, rng=rng)
    return iq0, iq1, ps
