#!/usr/bin/env python3
"""Writes tests/golden/tx11b_legacy/ack_fir_tail.bin: the 512 bytes `temp[]` of kernel/bb/demod11/modulate11b.cpp:15-80, the tail of the
filtered short-preamble 2 Mbps ACK that TestModAck (modulate11b.cpp:100-165) compares its filter output with.  Run by hand where the reference
tree exists:  python3 tests/golden/make_tx11b_legacy_ack.py [reference root]"""
import os, re, sys
ref = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
src = open(os.path.join(ref, "kernel", "bb", "demod11", "modulate11b.cpp"), encoding="latin-1").read()
body = re.search(r"UCHAR\s+temp\[\]\s*=\s*\{(.*?)\};", src, re.S).group(1)
data = bytes(int(x, 16) for x in re.findall(r"0x[0-9A-Fa-f]+", body))
assert len(data) == 512, len(data)
out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "tx11b_legacy", "ack_fir_tail.bin")
open(out, "wb").write(data)
print(out, len(data))
