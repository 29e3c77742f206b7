// Host emulation of the one-lane-per-code-block Viterbi kernel (sora_b200/csrc/viterbi_k7_lane.cuh): the DEVICE SOURCE ITSELF, compiled by g++
// with the CUDA intrinsics it uses written out in C++ (warp_emu.h).  Test infrastructure (tests/test_cpu_lane_emu.py compares it with the CPU
// oracle); it lets the -m "not gpu" suite check the kernel's trellis, history blocks, trigger schedule, traceback and bit packing where no GPU
// exists.  A lane never reads another lane's data, but the warp votes of the step loop decide together when the loop ends and which lanes
// step on without input while others still have some: so the 32 lanes of a CTA run as 32 threads, and every vote is a real vote of all 32.
//
//   g++ -O1 -std=c++20 -pthread -shared -fPIC -DSB_HOST_EMU -I sora_b200/csrc -o lane_emu.so tests/cpp/lane_emu.cpp
#include "warp_emu.h"
#include "viterbi_k7_lane.cuh"

// Decode nblocks code blocks the way sb200_viterbi_k7 launches the kernel (uniform parameters, no work list): every CTA of 32 lanes, every lane.
// lens / nsofts: per code block (the receive chains' FrameInfo path) or null.  hb: columns per history block, 6 or 8; 9 = 8 with the deferred walk.
extern "C" int lane_emu_viterbi(const uint8_t* soft, uint64_t soft_stride, uint32_t nsoft, uint32_t nblocks, int code_rate, uint32_t frame_len,
                                uint32_t depth, uint32_t lookahead, uint8_t* out, uint64_t out_stride, uint32_t* nraw,
                                const uint32_t* lens, const uint32_t* nsofts, int hb) {
    if (code_rate < 0 || code_rate > 2 || (hb != 6 && hb != 8 && hb != 9)) return -1;
    std::vector<sb::FrameInfo> fi;
    if (lens && nsofts) { fi.resize(nblocks); for (uint32_t i = 0; i < nblocks; i++) { fi[i] = sb::FrameInfo{}; fi[i].length = lens[i]; fi[i].soft_bytes = nsofts[i]; fi[i].code_rate = (uint32_t)code_rate; } }
    const sb::FrameInfo* info = fi.empty() ? nullptr : fi.data();
    sb::VitJob job{}; job.code_rate = (uint32_t)code_rate; job.frame_len = frame_len; job.nsoft = nsoft; job.depth = depth; job.lookahead = lookahead; job.raw = 1;
    const uint32_t ctas = (nblocks + SB_VL_FR - 1) / SB_VL_FR;
    std::vector<uint4> ring((size_t)ctas * SB_VL_NB8D * SB_VL_ENTRY);
    for (uint32_t c = 0; c < ctas; c++) warp_emu::run_cta(c, [&] {
#define SB_EMU_RUND(CR) sb::k_viterbi_lane<CR, 8, true>(soft, soft_stride, nblocks, nullptr, nullptr, info, job, out, out_stride, 0u, nraw, ring.data(), 0u)
#define SB_EMU_RUN(CR, HB) sb::k_viterbi_lane<CR, HB>(soft, soft_stride, nblocks, nullptr, nullptr, info, job, out, out_stride, 0u, nraw, ring.data(), 0u)
        if (hb == 6) { if (code_rate == sb::CR_12) SB_EMU_RUN(sb::CR_12, 6); else if (code_rate == sb::CR_23) SB_EMU_RUN(sb::CR_23, 6); else SB_EMU_RUN(sb::CR_34, 6); }
        else if (hb == 9) { if (code_rate == sb::CR_12) SB_EMU_RUND(sb::CR_12); else if (code_rate == sb::CR_23) SB_EMU_RUND(sb::CR_23); else SB_EMU_RUND(sb::CR_34); }
        else         { if (code_rate == sb::CR_12) SB_EMU_RUN(sb::CR_12, 8); else if (code_rate == sb::CR_23) SB_EMU_RUN(sb::CR_23, 8); else SB_EMU_RUN(sb::CR_34, 8); }
    });
    return 0;
}
