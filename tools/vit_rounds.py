#!/usr/bin/env python3
"""How many k_viterbi_re CTAs does an SM hold, and how fast is one round of them?  Standalone decoder, rate 3/4, 1500-byte blocks (config
#2's code blocks), the four-lane kernel forced (option viterbi_lane_min), launches of 8 x C code blocks for the CTA counts C given (default:
1 .. 12 per SM of 132 SMs, 22 per SM and config #2's 8 192).  The time stays nearly flat while the CTAs fit at once and jumps by a second
round when they do not, so the jump shows the resident count without a profiler.  Output: one line per launch."""
import os, sys, json
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import torch
from sora_b200 import api, synth
def main():
    dev = torch.device("cuda", 0); eng = api.Engine(0); st = torch.cuda.current_stream()
    eng.set_option("viterbi_lane_min", 0xFFFFFFFF)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas = [int(x) for x in sys.argv[1:]] or [sms * k for k in (1, 5, 9, 10, 11)] + [sms * 23 // 2, sms * 12, sms * 22, 8192]
    L = 1500; cr = api.CR_34
    nbits = 8 * L + 16 + 6; nbits += (-nbits) % 48
    rng = np.random.default_rng(1); U = 64
    bits = rng.integers(0, 2, (U, nbits)).astype(np.uint8); bits[:, 8 * L + 16:] = 0
    A, B = synth.conv_encode(bits); coded = synth.puncture(A, B, (3, 4))
    soft = np.where(coded > 0, rng.integers(5, 8, coded.shape), rng.integers(0, 3, coded.shape)).astype(np.uint8)
    nsoft = soft.shape[1]; stride = (nsoft + 15) // 16 * 16
    sp = np.zeros((U, stride), np.uint8); sp[:, :nsoft] = soft
    NBmax = max(ctas) * 8
    d_soft = torch.from_numpy(sp).to(dev).repeat((NBmax + U - 1) // U, 1)[:NBmax].contiguous()
    d_out = torch.zeros((NBmax, L + 2 + 14), dtype=torch.uint8, device=dev)
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    for c in ctas:
        NB = c * 8
        def step(): eng.viterbi_raw(d_soft.data_ptr(), stride, nsoft, NB, cr, L, d_out.data_ptr(), d_out.shape[1], stream=st.cuda_stream)
        for _ in range(2): step()
        torch.cuda.synchronize(); e0.record(st)
        for _ in range(5): step()
        e1.record(st); torch.cuda.synchronize()
        assert eng.last_viterbi_kernel() == "k_viterbi_re", eng.last_viterbi_kernel()
        print(json.dumps({"ctas": c, "ctas_per_sm": round(c / sms, 3), "ms": round(e0.elapsed_time(e1) / 5, 4)}), flush=True)
if __name__ == "__main__":
    main()
