// Host emulation of the four-lanes-per-code-block Viterbi kernel (k_viterbi_re, sora_b200/csrc/viterbi_k7_re.cuh): the DEVICE SOURCE
// ITSELF, compiled by g++ with the CUDA intrinsics it uses written out in C++ (warp_emu.h).  Test infrastructure (tests/test_cpu_re_emu.py
// compares it with the CPU oracle).  The lanes of a code block exchange path metrics with quad shuffles, one lane of the block walks the
// shared-memory ring behind __syncwarp, and the warp votes decide together when the lockstep loop ends: the 32 lanes of a CTA run as 32
// threads, and every shuffle, __syncwarp and vote is a real exchange among the lanes it names.
//
//   g++ -O1 -std=c++20 -pthread -shared -fPIC -DSB_HOST_EMU -I sora_b200/csrc -o re_emu.so tests/cpp/re_emu.cpp
#include "warp_emu.h"
#include "viterbi_k7_re.cuh"

// Decode nblocks code blocks the way sb200_viterbi_k7 launches the kernel (uniform parameters, no work list), or with per-block lengths and
// soft-byte counts (lens / nsofts, the receive chains' FrameInfo path).
extern "C" int re_emu_viterbi(const uint8_t* soft, uint64_t soft_stride, uint32_t nsoft, uint32_t nblocks, int code_rate, uint32_t frame_len,
                              uint32_t depth, uint32_t lookahead, uint8_t* out, uint64_t out_stride, uint32_t* nraw,
                              const uint32_t* lens, const uint32_t* nsofts) {
    if (code_rate < 0 || code_rate > 2) return -1;
    std::vector<sb::FrameInfo> fi;
    if (lens && nsofts) { fi.resize(nblocks); for (uint32_t i = 0; i < nblocks; i++) { fi[i] = sb::FrameInfo{}; fi[i].length = lens[i]; fi[i].soft_bytes = nsofts[i]; fi[i].code_rate = (uint32_t)code_rate; } }
    const sb::FrameInfo* info = fi.empty() ? nullptr : fi.data();
    sb::VitJob job{}; job.code_rate = (uint32_t)code_rate; job.frame_len = frame_len; job.nsoft = nsoft; job.depth = depth; job.lookahead = lookahead; job.raw = 1;
    const uint32_t ctas = (nblocks + SB_VR_FR - 1) / SB_VR_FR;
    for (uint32_t c = 0; c < ctas; c++) warp_emu::run_cta(c, [&] {
#define SB_EMU_RUN(CR) sb::k_viterbi_re<CR>(soft, soft_stride, nblocks, nullptr, nullptr, info, job, out, out_stride, 0u, nraw)
        if (code_rate == sb::CR_12) SB_EMU_RUN(sb::CR_12); else if (code_rate == sb::CR_23) SB_EMU_RUN(sb::CR_23); else SB_EMU_RUN(sb::CR_34);
    });
    return 0;
}
