"""Receive-chain captures at the int16 rails (test input only).

Every other test capture comes from synth.to_iq16: the signal is rounded to int8 and shifted left by 8, so a clean frame has a zero low
byte and never reaches +32767.  Real captures clip when the AGC overshoots, and radios have DC offsets.  The cases here start from synth
frames and work in the int16 domain (scale, offset, round, clip to [-32768, 32767]); they reach the saturating FFT adds, the pmaddwd
wrap, neg16(-32768), the int16 wrap of the 802.11b DC subtract, the 802.11n carrier-sense metric and the pilot atan.

cases_*() return a list of (name, capture) for one chain; a capture is int16 [n, 2] (802.11n: a pair, one per antenna).

Run as a script (python rail_inputs.py) it passes every case through the CPU oracle's entry points, naming each case on stdout before it
runs: test_cpu_oracle_rails.py runs it against an oracle built with a trapping signed-overflow check.
"""
import os, sys
if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from sora_b200 import synth

GAINS = (1 / 64, 1 / 8, 2, 4, 16)
DC_OFFSETS = ((20000, -20000), (-20000, 20000), (-7000, 13000))
PATTERNS = ("min", "rails", "nyquist", "tone", "square")


def clip16(x):
    return np.clip(np.round(x), -32768, 32767).astype(np.int16)

def scaled(iq, gain=1.0, dc=(0, 0)):
    """iq * gain + dc, rounded and clipped to int16."""
    return clip16(iq.astype(np.float64) * gain + np.asarray(dc, np.float64))

def pattern(kind, n, seed=0):
    """Full-scale input with no frame in it: [n, 2] int16."""
    t = np.arange(n)
    if kind == "min":                                   # constant -32768: neg16 / abs of the one value without a positive twin
        return np.full((n, 2), -32768, np.int16)
    if kind == "rails":                                 # every component on a random rail
        return np.where(np.random.default_rng(seed).random((n, 2)) < 0.5, -32768, 32767).astype(np.int16)
    if kind == "nyquist":                               # +-rails alternating every sample, both components
        return np.where((t % 2 == 0)[:, None], -32768, 32767).repeat(2, 1).astype(np.int16)
    if kind == "tone":                                  # full-scale complex tone, 1/13 of the sample rate
        z = 32768.0 * np.exp(2j * np.pi * t / 13.0)
        return clip16(np.stack([z.real, z.imag], 1))
    if kind == "square":                                # full-scale square wave, period 16 samples, im a quarter period behind re
        return np.stack([np.where((t // 8) % 2 == 0, 32767, -32768), np.where(((t + 4) // 8) % 2 == 0, 32767, -32768)], 1).astype(np.int16)
    raise ValueError(kind)

def burst_then(frame, burst):
    """`burst` x16, clipped on both rails, followed by the clean frame in the same slot; the slot stays a multiple of 28 samples long."""
    out = np.concatenate([scaled(burst, 16.0), frame])
    return out[: len(out) // 28 * 28]

def clipped_tail(frame, start):
    """The frame with everything from sample `start` on (its data symbols) x16, clipped on both rails: the header still decodes, so the
    data path (FFT, equaliser, demap / CCK correlator) runs on full-scale samples."""
    out = frame.copy(); out[start:] = scaled(frame[start:], 16.0)
    return out

def _common(frame, n, seed, tail_from):
    """The gains, DC offsets and full-scale patterns around one frame of n samples."""
    cs = [(f"gain{g:g}", scaled(frame, g)) for g in GAINS] + [("tail", clipped_tail(frame, tail_from))]
    cs += [(f"dc{d[0]:+d}{d[1]:+d}", scaled(frame, 1.0, d)) for d in DC_OFFSETS]
    cs += [(f"dc{DC_OFFSETS[0][0]:+d}{DC_OFFSETS[0][1]:+d}x4", scaled(frame, 4.0, DC_OFFSETS[0]))]
    cs += [(p, pattern(p, n, seed)) for p in PATTERNS]
    return cs

def cases_11a(rate_kbps, seed=0):
    """802.11a at 40 Msps: one 200-byte frame at rate_kbps, moved to the rails."""
    iq, _ = synth.make_frames(1, psdu_len=200, rate_kbps=rate_kbps, snr_db=30, lead=400, trail=228, seed0=0xA11A0000 + rate_kbps + seed)
    f = iq[0][: len(iq[0]) // 28 * 28]
    cs = _common(f, len(f), seed, 400 + 640 + 160)                # lead, preamble, SIGNAL: the first data symbol starts here
    cs.append(("burst", burst_then(f, f[:1400])))
    return cs

def cases_11b(rate_kbps, seed=0):
    """802.11b at 44 Msps: one 60-byte frame at rate_kbps, moved to the rails."""
    iq, _ = synth.make_frames_11b(1, psdu_len=60, rate_kbps=rate_kbps, snr_db=35, gain=0.3, seed0=0xB11B0000 + rate_kbps + seed)
    f = iq[0]
    cs = _common(f, len(f), seed, 400 + 192 * 44)                 # lead, long preamble and PLCP header (192 us): the PSDU starts here
    cs.append(("burst", burst_then(f, f[400:400 + 2800])))
    return cs

def htltf_tone(frame, start, flip):
    """The frame with its two HT-LTF symbols (160 samples each from `start`, 40 Msps) replaced by a full-scale tone on subcarrier -8, which
    is 16 samples periodic and so has the same phase in both symbols.  The HT-LTF bins p, q of the two symbols then reach about 32765: the
    channel estimate's (p + q) / 2 saturates when the second symbol is the same tone, (p - q) / 2 when it is negated (flip)."""
    t = np.arange(320)
    z = 32768.0 * np.exp(-2j * np.pi * 8 * t / 128.0)
    if flip: z[160:] = -z[160:]
    out = frame.copy(); out[start:start + 320] = clip16(np.stack([z.real, z.imag], 1))
    return out

def cases_11n(mcs, seed=0, chans=True):
    """802.11n 2x2 at 40 Msps: one 150-byte frame at mcs, moved to the rails; both antennas get the same treatment.  Also the HT-LTFs
    replaced by a full-scale tone, in phase on one antenna and sign-flipped on the other (both ways round), and with chans the frame
    through two rank-deficient channels (determinant 0)."""
    a, b, _ = synth.make_frames_11n(1, psdu_len=150, mcs=mcs, snr_db=30, lead=400, trail=228, seed0=0x11A00000 + mcs + seed)
    f0, f1 = a[0], b[0]
    n = len(f0) // 28 * 28; f0, f1 = f0[:n], f1[:n]
    ltf = 400 + 640 + 480 + 160                                    # lead, legacy preamble, L-SIG + HT-SIG, HT-STF: the HT-LTFs start here
    tail = ltf + 320                                               # and the first data symbol here
    cs = [(name, (x, _same(name, x, f1, seed, tail))) for name, x in _common(f0, n, seed, tail)]
    cs.append(("burst", (burst_then(f0, f0[:1400]), burst_then(f1, f1[:1400]))))
    cs.append(("htltf_tone", (htltf_tone(f0, ltf, False), htltf_tone(f1, ltf, True))))
    cs.append(("htltf_tone_swap", (htltf_tone(f0, ltf, True), htltf_tone(f1, ltf, False))))
    if chans:
        for cname, ch in (("rank1", ((1, 1), (1, 1))), ("single", ((1, 0), (0, 0)))):
            c0, c1, _ = synth.make_frames_11n(1, psdu_len=150, mcs=mcs, snr_db=None, lead=400, trail=228, chan=ch, seed0=0x11A00000 + mcs + seed)
            cs.append((cname, (c0[0][:n], c1[0][:n])))
    return cs

def _same(name, x0, f1, seed, tail):
    """The second antenna's capture for a case made from the first antenna's frame: same gain / offset applied to antenna 1's frame,
    a full-scale pattern with its own seed."""
    if name.startswith("gain"): return scaled(f1, float(name[4:]))
    if name == "tail": return clipped_tail(f1, tail)
    if name.startswith("dc"):
        for d in DC_OFFSETS:
            if name.startswith(f"dc{d[0]:+d}{d[1]:+d}"): return scaled(f1, 4.0 if name.endswith("x4") else 1.0, d)
    return pattern(name, len(x0), seed + 1)

def slots(caps):
    """Concatenate captures into one buffer: (flat, off, len) with every slot starting on a 4-sample boundary."""
    ln = np.array([len(c) for c in caps], np.uint32)
    off = np.concatenate([[0], np.cumsum((ln.astype(np.uint64) + 3) // 4 * 4)[:-1]]).astype(np.uint64)
    flat = np.zeros((int(off[-1]) + int(ln[-1]), 2), np.int16)
    for o, c in zip(off, caps): flat[int(o):int(o) + len(c)] = c
    return flat, off, ln


def _run_oracle():
    """Every case through the oracle entry points the device tests compare with."""
    import oracle_py
    say = lambda s: (print(s), sys.stdout.flush())
    for rate in (6000, 24000, 54000):
        for name, x in cases_11a(rate):
            say(f"11a {rate} {name}")
            oracle_py.rx11a_batch(x, [0], [len(x)])
            oracle_py.rx11a_batch(np.repeat(x, 2, axis=0), [0], [2 * len(x)])
            oracle_py.rx11a_run(oracle_py.resample_44_40(x), max_frames=1)
            oracle_py.rx11a_taps(x, max_sym=60)
    for rate in (1000, 2000, 5500, 11000):
        for name, x in cases_11b(rate):
            say(f"11b {rate} {name}")
            oracle_py.rx11b_batch(x, [0], [len(x)])
            oracle_py.rx11b_run(x, max_frames=4)
    for mcs, limit in ((8, 11), (10, 11), (14, 15)):
        oracle_py.set_ht_mcs_limit(limit)
        for name, (x, y) in cases_11n(mcs):
            say(f"11n {mcs} {name}")
            oracle_py.rx11n_batch(x, y, [0], [len(x)])
            oracle_py.rx11n_run(x, y, max_frames=4)
            oracle_py.rx11n_taps(x, y)
    oracle_py.set_ht_mcs_limit(11)
    say("done")

if __name__ == "__main__":
    if len(sys.argv) > 1:
        import oracle_py
        oracle_py.use_library(sys.argv[1])
    _run_oracle()

def cck_rail_frames_11b(rate_kbps, n=4, seed=0):
    """802.11b frames at 5.5 or 11 Mbps whose 64-byte PSDU is replaced by random rectangular chips on the int16 rails (32767 / -32768,
    four samples per chip).  The lead is 200 samples, so the energy detector fires on the first preamble vector and the DC estimate stays
    exactly 0: the CCK decoders see the rails themselves.  There the phase decision on the last chip (soradsp.h:190-199) halves re and im
    before re + im; without the halving re + im wraps and the delivered bytes change.  Returns int16 [n, slot, 2]."""
    iq, _ = synth.make_frames_11b(n, psdu_len=64, rate_kbps=rate_kbps, snr_db=None, gain=1.0, seed0=0x2A11 + rate_kbps + seed, lead=200)
    p0 = 200 + 192 * 44; nchip = 64 * (8 if rate_kbps == 11000 else 16)
    chips = np.where(np.random.default_rng(seed + rate_kbps).random((n, nchip, 2)) < 0.5, -32768, 32767).astype(np.int16)
    iq[:, p0:p0 + 4 * nchip] = np.repeat(chips, 4, axis=1)
    return iq
