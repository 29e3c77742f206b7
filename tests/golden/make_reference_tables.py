#!/usr/bin/env python3
"""Snapshot of every reference table and constant the CPU and GPU suites compare the restatements with, so that those comparisons run
without the reference tree.  Parses the LUT data out of the reference headers (tools/refcheck.py) and, for the legacy 802.11b transmit
filter, runs the reference's own compiled filter body (oracle/_ref, oracle/build_ref.sh) on the test inputs and keeps the SHA-256 of
each output.  Writes tests/golden/reference_tables.npz.

  python tests/golden/make_reference_tables.py <reference root>"""
import hashlib, os, re, sys, numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
sys.path.insert(0, os.path.dirname(TESTS)); sys.path.insert(0, TESTS); sys.path.insert(0, os.path.join(os.path.dirname(TESTS), "tools"))
import refcheck as rc
import oracle_py
from golden_vectors import digest

def pairs(path, name):
    s = rc._read(path); i = s.index(name + "[] ="); j = s.index("};", i)
    return np.array(re.findall(r"\{\s*(-?\d+)\s*,\s*(-?\d+)\s*\}", s[i:j]), dtype=np.int16)

def define(path, name):
    return int(re.search(r"#define\s+" + name + r"\s+(0x[0-9A-Fa-f]+|\d+)", rc._read(path)).group(1), 0)

def tables():
    t = {}
    for N in (16, 32, 64, 128):
        for M in (1, 2, 3): t[f"twiddle{N}_{M}"] = rc.ref_twiddle(N, M)[: N // 4]
    t["twiddle8"] = np.array(rc.parse_array(rc._read("kernel/core/inc/fft_lut_twiddle.h"), "wFFTLUT8")).reshape(-1, 2)
    for N in (64, 128): t[f"bitrev{N}"] = rc.ref_bitrev(N)
    for n, a in zip(("usin", "ucos", "uatan2"), rc.ref_trig()): t[n + "_sha256"] = digest(a)     # 65536 entries each: kept as digests
    t["vit_ma"], t["vit_mb"] = rc.ref_vit()
    for cls in ("BPSK", "QPSK", "QAM16", "QAM64"):
        t[f"deint11a_{cls}"] = rc.ref_deinterleave(cls)
        for s in range(2): t[f"deint11n_{cls}_S{s}"] = rc.ref_deinterleave_11n(f"{cls}_S{s}")
    t["lts_11a"] = np.array(rc.parse_array(rc._read("kernel/bb/Brick11/src/channel_11a.hpp"), "LTS_Sequence_11a"))
    t["pilot_sgn_11a"] = np.array(rc.parse_array(rc._read("kernel/bb/Brick11/src/pilot.hpp"), "PilotSgn"))
    for n, a in rc.ref_demap_luts().items(): t["demap_" + n] = a
    d = rc._read("kernel/bb/Brick11/src/dsp_demap.h"); d = d[d.index("This LUT is constructed"):]
    for n in ("bpsk", "qpsk", "16qam1", "16qam2", "64qam1", "64qam2", "64qam3"):
        t["demap11n_" + n] = np.array(rc.parse_array(d, "dsp_demapper::lookup_table_" + n))
    t["crc8"] = rc.ref_crc8()
    t["lltf_plus"], t["htltf_plus"] = rc.ref_ltf_masks()
    nd = rc.ref_ht_ndbps(); t["ht_ndbps"] = np.array([nd[m] for m in range(16)])
    t["l_stf"] = pairs("kernel/bb/Brick11/src/_b_lstf.h", "L_STF::_stf"); t["l_ltf"] = pairs("kernel/bb/Brick11/src/_b_lltf.h", "L_LTF::_ltf")
    t["ht_stf"] = pairs("kernel/bb/Brick11/src/_b_htstf.h", "HT_STF::_stf"); t["ht_ltf"] = pairs("kernel/bb/Brick11/src/_b_htltf.h", "HT_LTF::_ltf")
    s = rc._read("kernel/bb/Brick11/src/_b_dot11_pilot.h"); i = s.index("dot11_ofdm_pilot::_pilot_sign[pilot_size] ="); j = s.index("};", i)
    t["pilot_sign_11n"] = np.array([int(v) for v in re.findall(r"-?\d+", s[s.index("{", i):j])])
    t["barker11"] = np.array(rc.parse_array(rc._read("kernel/bb/Brick11/src/barkerspread.hpp"), "Barker11"))
    t["dqpsk_encode"] = pairs("kernel/bb/Brick11/src/cck.hpp", "DQPSKEncode"); t["cck11_d3d2"] = pairs("kernel/bb/Brick11/src/cck.hpp", "CCK11D3D2")
    t["long_tx_scrambler_register"] = np.array(define("kernel/inc/dot11_plcp.h", "DOT11B_PLCP_LONG_TX_SCRAMBLER_REGISTER"))
    t["long_preamble_sfd"] = np.array(define("kernel/inc/dot11_plcp.h", "DOT11B_PLCP_LONG_PREAMBLE_SFD"))
    with open(os.path.join(rc.REF, "kernel/test-data/fsample-6.dmp"), "rb") as f: t["fsample6_sha256"] = np.frombuffer(hashlib.sha256(f.read()).digest(), np.uint8)
    return t

def fir37_digests():
    """SHA-256 of the reference filter body's output on every input the suites feed it."""
    import test_cpu_oracle_tx11b_legacy as tc, test_gpu_tx11b_legacy as tg
    assert oracle_py.ref_fir37_available(), "build oracle/_ref first (oracle/build_ref.sh)"
    return {key: np.frombuffer(hashlib.sha256(oracle_py.ref_fir37(x).tobytes()).digest(), np.uint8)
            for key, x in list(tc.ref_body_cases()) + list(tg.ref_body_cases())}

if __name__ == "__main__":
    rc.REF = sys.argv[1]
    t = tables(); t.update(fir37_digests())
    def narrow(a):                                          # the smallest integer type that holds the table
        a = np.asarray(a)
        if a.dtype.kind != "i" or a.size == 0: return a
        return a.astype(next(d for d in (np.int8, np.int16, np.int32, np.int64) if np.iinfo(d).min <= a.min() and a.max() <= np.iinfo(d).max))
    np.savez_compressed(os.path.join(HERE, "reference_tables.npz"), **{k: narrow(v) for k, v in t.items()})
    print(len(t), "arrays")
