"""Receive batches at the scale where k_viterbi_re's persistent CTAs loop (test input only): seeded unique captures of every rate, length,
noise level and kind of damage, and tile(), which lays n slots over them in a seeded, non-periodic order.

At 65 536 slots every code rate's work list of the 802.11a receiver holds more code blocks than one round of the four-lane kernel's CTAs,
so a CTA decodes many groups of 8 one after the other, and every group mixes lengths and verdicts.  The IQ of the uniques exists once;
the slot table points into it (bench.py does the same with --unique).

  * uniques_11a(): about 1 500 single-frame captures over all eight rates, weighted so that each code rate (1/2: 6, 12, 24 Mbps; 2/3: 48;
    3/4: 9, 18, 36, 54) carries about a third of the decoded frames.  PSDU lengths 1 .. 1 500 B (as far as a slot holds them), leads of
    every phase mod 4, carrier offsets up to +-150 kHz, and clean, comfortable and near-threshold SNR, so the oracle returns FRAME_OK and
    CRC32_FAIL at every code rate.  Plus payload hits (CRC fail), SIGNAL hits (PLCP fail: the frame never reaches a work list),
    noise-only and all-zero slots, and slots cut inside the DATA field (a truncated code block).  Every slot is at most SLOT_CAP samples:
    the receiver sizes its soft workspace from the longest slot, nframes x ((max_len / 2) / 80 + 1) x 288 B, about 3.9 GB at 65 536.
  * uniques_11n(): about 600 2x2 captures at MCS 8 .. 14 (decoded with ht_mcs_limit 15, so all three code rates occur), PSDUs of at most
    400 B, the same kinds of damage.
  * uniques_streams(): 256 continuous captures of 3 .. 5 frames each, at least 85 % of them at rate 3/4.

Every generator returns a Uniques: the IQ (one flat int16 [n, 2] buffer, per antenna for 802.11n), each unique's offset and length in it,
and per unique the rate (kbps; the MCS for 802.11n; a list per capture for streams), the PSDU length and the kind of capture.
"""
import functools
from dataclasses import dataclass
import numpy as np
from sora_b200 import synth

SLOT_CAP = 32768                                        # samples per slot at most
RATES_11A = {0: (6000, 12000, 24000), 1: (48000,), 2: (9000, 18000, 36000, 54000)}      # code rate -> rates
CODE_RATE_11A = {r: cr for cr, rs in RATES_11A.items() for r in rs}
MCS_11N = {0: (8, 9, 11), 1: (13,), 2: (10, 12, 14)}
CODE_RATE_11N = {m: cr for cr, ms in MCS_11N.items() for m in ms}
NDBPS_11A = {6000: 24, 9000: 36, 12000: 48, 18000: 72, 24000: 96, 36000: 144, 48000: 192, 54000: 216}
# SNR (dB, synth.to_iq16's definition) about where the payload of a 1 000 B frame starts to fail, per rate: "edge" captures sit around it
EDGE_11A = {6000: 3.0, 9000: 5.0, 12000: 6.0, 18000: 9.0, 24000: 11.5, 36000: 15.5, 48000: 19.5, 54000: 21.0}
EDGE_11N = {8: 3.0, 9: 6.0, 10: 9.0, 11: 12.0, 12: 15.5, 13: 19.5, 14: 21.5}
CFO_11N = 40e3                                          # Hz: beyond about this the 802.11n receiver rejects many HT-SIGs (PLCP fail)
# share of the frames per code rate: rate 1/2 loses more of its frames before the work list (SIGNAL at the 6 Mbps edge, PSDUs too short
# for a verdict), so it gets more, and every code rate ends with about a third of the decoded frames
CR_WEIGHT_11A = (0.36, 0.32, 0.32)
# kinds of capture and their share: frames that reach a work list, and the rest
KINDS = (("clean", 0.20), ("snr", 0.40), ("edge", 0.22), ("payload", 0.08), ("trunc", 0.04), ("signal", 0.02), ("noise", 0.02), ("zero", 0.02))


@dataclass
class Uniques:
    iq: object                  # int16 [n, 2]; 802.11n: (antenna 0, antenna 1)
    off: np.ndarray             # uint64 [U]: first sample of each unique
    length: np.ndarray          # uint32 [U]: its samples
    rate: list                  # kbps (802.11a), MCS (802.11n), a list per capture (streams); 0 for a slot without a frame
    psdu_len: list              # PSDU bytes, a list per capture for streams; 0 without a frame
    kind: list                  # one of KINDS


def _kind(rng):
    return KINDS[int(rng.choice(len(KINDS), p=[p for _, p in KINDS]))][0]

def _max_psdu_11a(rate, lead):
    """The longest PSDU at `rate` whose frame (640 preamble + 160 SIGNAL + 160 per data symbol) and a 64-sample trail fit SLOT_CAP."""
    nsym = (SLOT_CAP - lead - 64 - 800) // 160
    return min(1500, (nsym * NDBPS_11A[rate] - 22) // 8)

def _frame_11a(rate, L, seed, snr, cfo, lead, trail, gain=0.5):
    """One 802.11a capture int16 [lead + frame + trail, 2]: a PSDU of L bytes (with FCS when L >= 4) through synth.make_frames."""
    if L >= 4:
        iq, _ = synth.make_frames(1, psdu_len=L, rate_kbps=rate, seed0=seed, snr_db=snr, lead=lead, trail=trail, cfo_hz=cfo, gain=gain)
        return iq[0]
    ps = np.random.RandomState(seed & 0xFFFFFFFF).randint(0, 256, (1, L)).astype(np.uint8)    # too short for an FCS: no verdict
    return synth.to_iq16(synth.modulate(ps, rate), gain=gain, lead=lead, trail=trail, snr_db=snr, cfo_hz=cfo, rng=np.random.default_rng(seed))[0]

def _damage(x, kind, lead, rng, nsym_data, sig_at=640):
    """Payload hit: a burst of strong noise over two data symbols.  SIGNAL hit: noise over the SIGNAL symbol.  Truncation: the slot ends
    inside the DATA field (at least one data symbol in, at least one short)."""
    x = x.copy()
    if kind == "payload":
        s = lead + sig_at + 160 + 160 * int(rng.integers(0, max(nsym_data - 1, 1)))
        x[s:s + 320] = rng.integers(-6000, 6000, x[s:s + 320].shape)
    elif kind == "signal":
        x[lead + sig_at:lead + sig_at + 160] = rng.integers(-6000, 6000, (160,) + x.shape[1:])
    elif kind == "trunc":
        keep = lead + sig_at + 160 + 160 * int(rng.integers(1, max(nsym_data, 2))) - int(rng.integers(0, 120))
        x = x[:keep]
    return x

def _pack(parts):
    """Captures -> one flat buffer, every capture starting at a multiple of 4 samples (lengths as they are)."""
    off = np.zeros(len(parts), np.uint64); n = 0
    for i, p in enumerate(parts): off[i] = n; n += (len(p) + 3) // 4 * 4
    buf = np.zeros((n, 2), np.int16)
    for o, p in zip(off, parts): buf[int(o):int(o) + len(p)] = p
    return buf, off, np.array([len(p) for p in parts], np.uint32)


@functools.lru_cache(maxsize=None)
def uniques_11a(n=1500, seed=0x5CA1E11A):
    rng = np.random.default_rng(seed)
    parts, rate, plen, kinds = [], [], [], []
    for i in range(n):
        kind = _kind(rng)
        lead = 32 + 4 * int(rng.integers(0, 64)) + i % 4                # every phase mod 4
        if kind in ("noise", "zero"):
            m = int(rng.integers(2000, SLOT_CAP + 1))
            x = np.zeros((m, 2), np.int16) if kind == "zero" else np.clip(np.round(rng.normal(0, 1500, (m, 2))), -32768, 32767).astype(np.int16)
            parts.append(x); rate.append(0); plen.append(0); kinds.append(kind)
            continue
        cr = int(rng.choice(3, p=CR_WEIGHT_11A))
        r = RATES_11A[cr][int(rng.integers(0, len(RATES_11A[cr])))]
        Lmax = _max_psdu_11a(r, lead)
        L = int(rng.integers(1, 40)) if rng.random() < 0.1 else int(rng.integers(1, Lmax + 1))
        snr = {"clean": None, "snr": EDGE_11A[r] + float(rng.uniform(8, 20)), "edge": EDGE_11A[r] + float(rng.uniform(-1.0, 3.0))}.get(kind, EDGE_11A[r] + 12)
        cfo = float(rng.uniform(-150e3, 150e3)) if rng.random() < 0.6 else 0.0
        x = _frame_11a(r, L, 0x5CA10000 + i, snr, cfo, lead, 64)
        nsym_data = -(-(8 * L + 22) // NDBPS_11A[r])
        if kind in ("payload", "trunc") and nsym_data < 2: kind = "snr"
        parts.append(_damage(x, kind, lead, rng, nsym_data)); rate.append(r); plen.append(L); kinds.append(kind)
    iq, off, ln = _pack(parts)
    assert ln.max() <= SLOT_CAP
    return Uniques(iq, off, ln, rate, plen, kinds)


@functools.lru_cache(maxsize=None)
def uniques_11n(n=600, seed=0x5CA1E11B):
    rng = np.random.default_rng(seed)
    p0, p1, rate, plen, kinds = [], [], [], [], []
    for i in range(n):
        kind = _kind(rng)
        lead = 64 + 4 * int(rng.integers(0, 48)) + i % 4
        if kind in ("noise", "zero"):
            m = int(rng.integers(2000, 12000))
            for p in (p0, p1):
                p.append(np.zeros((m, 2), np.int16) if kind == "zero" else np.clip(np.round(rng.normal(0, 1500, (m, 2))), -32768, 32767).astype(np.int16))
            rate.append(0); plen.append(0); kinds.append(kind)
            continue
        cr = i % 3
        mcs = MCS_11N[cr][int(rng.integers(0, len(MCS_11N[cr])))]
        L = int(rng.integers(4, 401))
        snr = {"clean": None, "snr": EDGE_11N[mcs] + float(rng.uniform(8, 18)), "edge": EDGE_11N[mcs] + float(rng.uniform(-1.5, 2.5))}.get(kind, EDGE_11N[mcs] + 12)
        cfo = float(rng.uniform(-CFO_11N, CFO_11N)) if rng.random() < 0.6 else 0.0
        a, b, _ = synth.make_frames_11n(1, psdu_len=L, mcs=mcs, seed0=0x5CB10000 + i, snr_db=snr, lead=lead, trail=64, cfo_hz=cfo, gain=0.5)
        nsym_data = -(-(8 * L + 22) // synth.HT_MCS[mcs][2])
        if kind in ("payload", "trunc") and nsym_data < 2: kind = "snr"
        # the HT data field starts after L-STF, L-LTF, L-SIG, two HT-SIG, HT-STF and two HT-LTF: 640 + 3 x 160 + 3 x 160 samples
        hit_rng = np.random.default_rng(0x5CB20000 + i)
        sig_at = 640 if kind == "signal" else 1600 - 160
        a = _damage(a[0], kind, lead, hit_rng, nsym_data, sig_at); hit_rng = np.random.default_rng(0x5CB20000 + i)
        b = _damage(b[0], kind, lead, hit_rng, nsym_data, sig_at)
        p0.append(a); p1.append(b); rate.append(mcs); plen.append(L); kinds.append(kind)
    iq0, off, ln = _pack(p0); iq1, _, _ = _pack(p1)
    return Uniques((iq0, iq1), off, ln, rate, plen, kinds)


@functools.lru_cache(maxsize=None)
def uniques_streams(n=256, seed=0x5CA1E5A5):
    """Continuous captures of 3 .. 5 frames.  The first three frames of a capture are at rate 3/4 but in one capture in 16, every later one
    in two of three: at least 85 % of the frames overall."""
    rng = np.random.default_rng(seed)
    parts, rate, plen, kinds = [], [], [], []
    others = (6000, 12000, 24000, 48000)
    for c in range(n):
        nf = int(rng.integers(3, 6)); rs, ls, segs = [], [], []
        for j in range(nf):
            r34 = rng.random() >= 1 / 16 if j < 3 else rng.random() < 2 / 3
            r = RATES_11A[2][int(rng.integers(0, 4))] if r34 else others[int(rng.integers(0, 4))]
            L = int(rng.integers(4, {6000: 250, 9000: 300, 12000: 400}.get(r, 700)))
            segs.append(_frame_11a(r, L, 0x5CA50000 + 8 * c + j, float(rng.uniform(22, 40)) if rng.random() < 0.8 else None,
                                   float(rng.uniform(-100e3, 100e3)), int(rng.integers(40, 400)), int(rng.integers(60, 500))))
            rs.append(r); ls.append(L)
        parts.append(np.concatenate(segs)); rate.append(rs); plen.append(ls); kinds.append("stream")
    iq, off, ln = _pack(parts)
    return Uniques(iq, off, ln, rate, plen, kinds)


def tile(u, n, seed):
    """A slot table of n rows over the uniques of `u`: (offsets uint64 [n], lengths uint32 [n], perm int64 [n]), slot i = unique perm[i].
    Every unique appears n // U or n // U + 1 times, in a seeded random order (not periodic: neighbouring slots, and so the code blocks of
    one group, come from unrelated uniques)."""
    U = len(u.off)
    perm = np.random.default_rng(seed).permutation(np.resize(np.arange(U), n))
    return u.off[perm], u.length[perm], perm
