// Host emulation of k_viterbi_re (sora_b200/csrc/viterbi_k7_re.cuh) as persistent CTAs: the device source with its group loop as the
// device runs it (SB_EMU_PERSISTENT), on a grid smaller than the number of groups of code blocks.  The CUDA intrinsics of warp_emu.h (tests/cpp/
// re_emu.cpp) plus the three the loop needs: gridDim, atomicAdd on the per-launch group counter, and the broadcast of lane 0's ticket.
// Test infrastructure (tests/test_cpu_re_emu_persistent.py compares it with the CPU oracle).
//
//   g++ -O1 -std=c++20 -pthread -shared -fPIC -DSB_HOST_EMU -I sora_b200/csrc -o re_emu_grid.so tests/cpp/re_emu_grid.cpp
#define SB_EMU_PERSISTENT
#include "warp_emu.h"
static Dim gridDim;                                                             // set before the CTAs of a launch run
static inline uint32_t atomicAdd(uint32_t* p, uint32_t v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline uint32_t __shfl_sync(unsigned mask, uint32_t v, int src) { return warp_emu::exchange(mask, v)[src & 31]; }
#include "viterbi_k7_re.cuh"

// Decode nblocks code blocks (uniform parameters, or per-block lengths and soft-byte counts as in tests/cpp/re_emu.cpp) with a grid of
// `ctas` CTAs.  The CTAs run one after the other, so CTA 0 takes its own group and then every group no other CTA started with: it decodes
// several groups in a row, the ragged last one included.
extern "C" int re_emu_viterbi_grid(const uint8_t* soft, uint64_t soft_stride, uint32_t nsoft, uint32_t nblocks, int code_rate, uint32_t frame_len,
                                   uint32_t depth, uint32_t lookahead, uint8_t* out, uint64_t out_stride, uint32_t* nraw,
                                   const uint32_t* lens, const uint32_t* nsofts, uint32_t ctas) {
    if (code_rate < 0 || code_rate > 2 || ctas == 0) return -1;
    std::vector<sb::FrameInfo> fi;
    if (lens && nsofts) { fi.resize(nblocks); for (uint32_t i = 0; i < nblocks; i++) { fi[i] = sb::FrameInfo{}; fi[i].length = lens[i]; fi[i].soft_bytes = nsofts[i]; fi[i].code_rate = (uint32_t)code_rate; } }
    const sb::FrameInfo* info = fi.empty() ? nullptr : fi.data();
    sb::VitJob job{}; job.code_rate = (uint32_t)code_rate; job.frame_len = frame_len; job.nsoft = nsoft; job.depth = depth; job.lookahead = lookahead; job.raw = 1;
    const uint32_t groups = (nblocks + SB_VR_FR - 1) / SB_VR_FR, grid = std::min(ctas, groups);
    uint32_t next = 0;
    gridDim.x = grid;
    for (uint32_t c = 0; c < grid; c++) warp_emu::run_cta(c, [&] {
#define SB_EMU_RUN(CR) sb::k_viterbi_re<CR>(soft, soft_stride, nblocks, nullptr, nullptr, info, job, out, out_stride, 0u, nraw, &next)
        if (code_rate == sb::CR_12) SB_EMU_RUN(sb::CR_12); else if (code_rate == sb::CR_23) SB_EMU_RUN(sb::CR_23); else SB_EMU_RUN(sb::CR_34);
    });
    return 0;
}
