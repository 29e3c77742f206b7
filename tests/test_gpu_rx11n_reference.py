"""The device's PLCP header parsers and its descrambler / frame sink against the reference's own compiled bricks (pytest -m gpu):
T11aPLCPParser, T11nSigParser and T11aDesc into TBB11aFrameSink from oracle/_ref/librx11n_ref.so (oracle/build_ref_rx11n.sh).

  - The header cases of tests/plcp_inputs.py through rx11a_batch and rx11n_batch: the device refuses exactly the headers the compiled
    parser refuses, fed the bits the SIGNAL decoder hands over, and reports its rate / MCS, length and symbol count.
  - Frames at every scrambler seed 1-127 and frames with a corrupted FCS, through both receivers: the device's status, CRC-32 and bytes
    equal the compiled descrambler and sink fed the scrambled SERVICE and PSDU bytes the Viterbi decoder delivers from a clean capture.
Reads only the compiled library and skips when it is not built."""
import numpy as np
import pytest

import oracle_py as O
import plcp_inputs as P
from sora_b200 import api, synth

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not O.ref_rx11n_available(), reason="oracle/_ref/librx11n_ref.so not built (needs the reference tree)")]


@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)


def _sig9(lsig, ht48):
    return np.frombuffer((lsig & 0xFFFFFF).to_bytes(3, "little") + ht48.to_bytes(6, "little"), np.uint8)


def test_headers_11a(eng):
    cases = P.cases_11a(); iq, off, ln = P.slots_of(cases)
    res, _ = eng.rx11a_batch(iq, off, ln, out_stride=2560)
    ref = O.ref_plcp11a_parse([c["word"] & 0x3FFFF for c in cases])     # the decoder hands over bits 0..17
    for c, r, f in zip(cases, res, ref):
        assert (r["status"] == P.E_PLCP) == (f[0] == 0), c["name"]
        if r["status"] == P.E_NONE: continue            # accepted, but the frame runs past the slot: no event, no fields
        if f[0]:
            assert (r["rate_kbps"], r["length"], r["nsym"]) == (f[2], f[3], f[4]), c["name"]


def test_headers_11n(eng):
    cases = P.cases_11n(); iq0, off, ln = P.slots_of(cases, "iq0"); iq1, _, _ = P.slots_of(cases, "iq1")
    res, _ = eng.rx11n_batch(iq0, iq1, off, ln)
    for c, r in zip(cases, res):
        lw, h34, cx = c["word"]
        f = O.ref_sig11n_parse(_sig9(lw & 0x3FFFF, h34 | (P.crc8_htsig(h34) ^ cx) << 34))[0]   # a fresh context per slot
        assert (r["status"] == P.E_PLCP) == (f[0] == 0), c["name"]
        if r["status"] == P.E_NONE: continue
        assert r["mcs"] == f[6], c["name"]
        if f[0]:
            assert (r["length"], r["nsym"]) == (f[3], f[4]), c["name"]


def _decoded(psdu, seed):
    bits = np.zeros(16 + 8 * len(psdu), np.uint8)
    bits[16:] = np.unpackbits(psdu, bitorder="little")
    bits ^= synth.scrambler_seq(seed, len(bits))
    return np.packbits(bits, bitorder="little")


def _bodies():
    """Frames at seeds 1..127, every fifth with one bit of its PSDU flipped after the FCS was computed."""
    bodies = []
    for s in range(1, 128):
        b = P.psdu(60 + s, 500 + s)
        if s % 5 == 0: b = b.copy(); b[s % len(b)] ^= 0x10
        bodies.append(b)
    return bodies


def _check_sink(res, out, bodies, seeds):
    n_ok = n_fail = 0
    for i, (b, s) in enumerate(zip(bodies, seeds)):
        e, crc, want = O.ref_desc_sink(_decoded(b, s), len(b))
        assert (res["status"][i], res["crc32"][i]) == (e, crc), (s, hex(int(res["status"][i])), hex(e))
        assert (out[i, :len(b)] == want).all(), s
        n_ok += e == O.E_FRAME_OK; n_fail += e == O.E_CRC32_FAIL
    assert n_ok > 90 and n_fail > 20


def test_sink_every_seed_11a(eng):
    bodies = _bodies(); seeds = list(range(1, 128))
    slots = [synth.to_iq16(synth.modulate(b, 36000, scramble_seeds=[s]), lead=200, trail=400)[0] for b, s in zip(bodies, seeds)]
    iq, off, ln = P.pack(slots)
    res, out = eng.rx11a_batch(iq, off, ln, out_stride=256)
    _check_sink(res, out, bodies, seeds)


def test_sink_every_seed_11n(eng):
    bodies = _bodies(); seeds = list(range(1, 128))
    s0, s1 = [], []
    for b, s in zip(bodies, seeds):
        tx = synth.modulate_11n(b, 9, scramble_seeds=[s])
        rx = np.einsum("ab,fbn->fan", np.asarray(P.CHAN, np.complex128), tx)
        s0.append(synth.to_iq16(rx[:, 0], lead=400, trail=200)[0]); s1.append(synth.to_iq16(rx[:, 1], lead=400, trail=200)[0])
    iq0, off, ln = P.pack(s0); iq1, _, _ = P.pack(s1)
    res, out = eng.rx11n_batch(iq0, iq1, off, ln)
    _check_sink(res, out, bodies, seeds)
