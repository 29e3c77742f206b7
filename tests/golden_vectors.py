"""Loaders for the reference-held 802.11a waveforms under tests/golden (shared by the CPU and the GPU suites).

Every vector is a TRANSMIT waveform of the reference (what its modulator handed to the DAC); the receive chain sees it through a
noiseless unit channel: 20 Msps vectors are sample-repeated to the 40 Msps capture rate (TDownSample2 keeps samples 0 and 2 of
every 4, samples.hpp:27-49, so the decimated stream is the vector itself), 8-bit vectors are shifted like
ConvertModFile2DumpFile_8b does (demod11/modulate11a.cpp:178-179), and a power-of-two gain lifts the 16-bit ones over
cca_pwr_threshold."""
import os, numpy as np
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

ACK_PSDU = bytes.fromhex("d40000000250f2000004b033a9eb")      # ACK to 02:50:F2:00:00:04 incl. FCS (what BB11AModulateACK encodes, atx_fe.c:168-195)

def _pad(iq, lead=400, trail=428):
    return np.concatenate([np.zeros((lead, 2), np.int16), iq, np.zeros((trail, 2), np.int16)])

def dummy_vectors():
    """name -> (iq int16 [n,2] at 40 Msps, expected rate_kbps, expected PSDU bytes or None for 'equals fsample-6.psdu.bin')"""
    out = {}
    v = np.fromfile(os.path.join(GOLD, "dot11a_dummy_20m.i16"), np.int16).reshape(-1, 2)
    out["dummy_20m"] = (_pad(np.repeat((v.astype(np.int32) << 1).astype(np.int16), 2, axis=0)), 6000, None)
    v = np.fromfile(os.path.join(GOLD, "dot11a_dummy_16_40m.i16"), np.int16).reshape(-1, 2)
    out["dummy_16_40m"] = (_pad((v.astype(np.int32) << 2).astype(np.int16)), 6000, None)
    v = np.fromfile(os.path.join(GOLD, "dot11a_dummy_8_20m.i8"), np.int8).reshape(-1, 2)
    out["dummy_8_20m"] = (_pad(np.repeat(v.astype(np.int16) << 8, 2, axis=0)), 6000, ACK_PSDU)
    v = np.fromfile(os.path.join(GOLD, "dot11a_dummy_8_ack_40m.i8"), np.int8).reshape(-1, 2)
    out["dummy_8_ack_40m"] = (_pad(v.astype(np.int16) << 8), 6000, ACK_PSDU)
    return out

def fsample6_psdu():
    return np.fromfile(os.path.join(GOLD, "fsample-6.psdu.bin"), np.uint8)

def reference_tables():
    """The reference's lookup tables and constants as parsed out of its headers, and SHA-256 digests of what its compiled 802.11b
    transmit filter returns for the suites' inputs (make_reference_tables.py)."""
    return dict(np.load(os.path.join(GOLD, "reference_tables.npz")))

def digest(a):
    """SHA-256 of an integer table as little-endian int64, the form the large tables of reference_tables.npz are kept in."""
    import hashlib
    return np.frombuffer(hashlib.sha256(np.asarray(a, "<i8").tobytes()).digest(), np.uint8)
