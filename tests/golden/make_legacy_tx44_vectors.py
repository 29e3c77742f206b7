#!/usr/bin/env python3
"""Known-answer vectors of the reference's LEGACY 802.11a transmitter at 44 Msps, one frame per rate, made by its own compiled code.

Run by hand after build() where oracle/_ref/libtx11a_legacy_ref.so exists (oracle/build_ref_tx11a_legacy.sh compiles BB11ATxFrameMod from
atx_*.c).  Each frame is BB11ATxFrameMod at SampleRate 44 of a fixed pseudo-random MPDU and its CRC-32 (Reserved1), with zeros read
behind the preamble table.  Outputs, under tests/golden/legacy_tx44/:
  legacy_tx44_<kbps>.i8   the complex int8 samples BB11ATxFrameMod writes, RCB zero padding included (SignalLength / 2 samples)
  legacy_tx44_<kbps>.bin  the MPDU + FCS that was modulated
The CPU suite requires the oracle (oracle/tx11a_legacy44.cpp) to reproduce every file, with or without the compiled library, so that the
44 Msps waveform stays pinned by the reference's own output where oracle/_ref cannot be built."""
import os, sys, zlib, numpy as np
HERE = os.path.dirname(os.path.abspath(__file__)); ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_tx11a_legacy as O

OUT = os.path.join(HERE, "legacy_tx44")
LEN = 150                                                               # MPDU bytes: an odd 9 Mbps symbol count, more than one window per rate


def main():
    assert O.ref_tx_available(), "oracle/_ref/libtx11a_legacy_ref.so not built"
    assert O.nsym(LEN + 4, 9000) % 2 == 1
    os.makedirs(OUT, exist_ok=True)
    for kbps in O.RATES:
        body = np.random.default_rng(kbps).integers(0, 256, LEN).astype(np.uint8)
        psdu = np.concatenate([body, np.frombuffer(zlib.crc32(bytes(body)).to_bytes(4, "little"), np.uint8)])
        w = O.ref_modulate(psdu, kbps, 44)
        psdu.tofile(os.path.join(OUT, f"legacy_tx44_{kbps}.bin")); w.tofile(os.path.join(OUT, f"legacy_tx44_{kbps}.i8"))
        print(kbps, len(w), "samples")


if __name__ == "__main__":
    main()
