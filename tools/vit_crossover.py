#!/usr/bin/env python3
"""Where does the one-lane-per-code-block Viterbi (k_viterbi_lane, 32 code blocks per warp) overtake the four-lanes kernel (k_viterbi_re,
8 per warp)?  Standalone decoder, rate 3/4, 1500-byte blocks (config #2's code blocks), batch sizes 1 024 .. 65 536, both kernels selected
through option viterbi_lane_min in one process.  Output: one line per batch size."""
import os, sys, json
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import torch
from sora_b200 import api, synth
def main():
    dev = torch.device("cuda", 0); eng = api.Engine(0); st = torch.cuda.current_stream()
    eng.set_option("viterbi_lane_max", 0xFFFFFFFF)       # no upper bound: 65 536 code blocks take the lane kernel too when lane_min allows
    L = 1500; cr = api.CR_34
    nbits = 8 * L + 16 + 6; nbits += (-nbits) % 48
    rng = np.random.default_rng(1); U = 64
    bits = rng.integers(0, 2, (U, nbits)).astype(np.uint8); bits[:, 8 * L + 16:] = 0
    A, B = synth.conv_encode(bits); coded = synth.puncture(A, B, (3, 4))
    soft = np.where(coded > 0, rng.integers(5, 8, coded.shape), rng.integers(0, 3, coded.shape)).astype(np.uint8)
    nsoft = soft.shape[1]; stride = (nsoft + 15) // 16 * 16
    sp = np.zeros((U, stride), np.uint8); sp[:, :nsoft] = soft
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    for NB in (1024, 2048, 4096, 8192, 16384, 24576, 32768, 49152, 65536):
        d_soft = torch.from_numpy(sp).to(dev).repeat((NB + U - 1) // U, 1)[:NB].contiguous()
        outs = {}; ms = {}
        for name, lane_min in (("k_viterbi_re", 0xFFFFFFFF), ("k_viterbi_lane", 0)):
            eng.set_option("viterbi_lane_min", lane_min)
            d_out = torch.zeros((NB, L + 2 + 14), dtype=torch.uint8, device=dev)
            def step(): eng.viterbi_raw(d_soft.data_ptr(), stride, nsoft, NB, cr, L, d_out.data_ptr(), d_out.shape[1], stream=st.cuda_stream)
            for _ in range(3): step()
            torch.cuda.synchronize(); e0.record(st)
            for _ in range(5): step()
            e1.record(st); torch.cuda.synchronize()
            ms[name] = e0.elapsed_time(e1) / 5; outs[name] = d_out[:, :L + 2].cpu().numpy()
            assert eng.last_viterbi_kernel() == name, eng.last_viterbi_kernel()
        assert (outs["k_viterbi_re"] == outs["k_viterbi_lane"]).all()
        print(json.dumps({"code_blocks": NB, "ms_k_viterbi_re": round(ms["k_viterbi_re"], 4), "ms_k_viterbi_lane": round(ms["k_viterbi_lane"], 4),
                          "lane_over_re": round(ms["k_viterbi_lane"] / ms["k_viterbi_re"], 3)}), flush=True)
        del d_soft
if __name__ == "__main__":
    main()
