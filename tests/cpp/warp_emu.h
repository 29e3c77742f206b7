// Host emulation of one warp for the Viterbi kernels' device source (tests/cpp/lane_emu.cpp, tests/cpp/re_emu.cpp): the CUDA intrinsics
// they use written out in C++, and a CTA of 32 lanes run as 32 std::threads.  Warp votes, shuffles and __syncwarp are real exchanges
// between those threads through a std::barrier per lane group (the full warp, a lane quad), so a lane that leaves the
// lockstep loop on a vote, or a code block whose lanes run a divergent tail while other blocks wait at the next vote, behaves as on the GPU.
// __shared__ arrays are function statics: one CTA runs at a time, and its 32 threads share them.
#pragma once
#include <algorithm>
#include <barrier>
#include <cstdint>
#include <cstring>
#include <memory>
#include <thread>
#include <vector>

#define __device__
#define __host__
#define __global__
#define __forceinline__ inline
#define __noinline__ __attribute__((noinline))
#define __launch_bounds__(...)
#define __restrict__
#define __shared__ static

struct uint2 { uint32_t x, y; };
struct uint4 { uint32_t x, y, z, w; };
struct Dim { unsigned x = 0, y = 0, z = 0; };
static thread_local Dim threadIdx, blockIdx;

using std::min; using std::max;
static inline uint32_t __byte_perm(uint32_t a, uint32_t b, uint32_t s) {        // PRMT, default mode: selector nibble n picks byte n of {b, a}
    const uint64_t v = ((uint64_t)b << 32) | a; uint32_t r = 0;
    for (int i = 0; i < 4; i++) r |= (uint32_t)((v >> (8 * ((s >> (4 * i)) & 7u))) & 0xFFu) << (8 * i);
    return r;
}
static inline uint32_t __brev(uint32_t v) { uint32_t r = 0; for (int i = 0; i < 32; i++) r |= ((v >> i) & 1u) << (31 - i); return r; }
static inline uint32_t __vminu2(uint32_t a, uint32_t b) { return min(a & 0xFFFFu, b & 0xFFFFu) | (min(a >> 16, b >> 16) << 16); }
static inline uint32_t __vadd2(uint32_t a, uint32_t b) { return ((a + b) & 0xFFFFu) | (((a >> 16) + (b >> 16)) << 16); }     // per-half wrap-around add
static inline uint32_t __viaddmin_u16x2(uint32_t a, uint32_t b, uint32_t c) { return __vminu2(__vadd2(a, b), c); }           // min(a + b, c) per half, unsigned
template <class T> static inline T __ldg(const T* p) { return *p; }
template <class T> static inline T __ldcg(const T* p) { return *p; }
template <class T> static inline void __stcg(T* p, const T& v) { *p = v; }

namespace warp_emu {
// One lane group: every lane of `mask` calls the same intrinsic, writes its value, waits for the others and reads.  Two slot rows used in
// turn (each lane counts its own calls; the lanes of a group make the same calls) so one barrier per call suffices: a lane can only write a
// row again after the next call's barrier, which every reader of this call reaches after its read.
struct Group {
    std::barrier<> bar;
    uint32_t slot[2][32];
    unsigned parity[32] = {};
    explicit Group(int n) : bar(n) {}
};
struct Cta {
    std::unique_ptr<Group> full, quad[8];
    Cta() {
        full = std::make_unique<Group>(32);
        for (auto& g : quad) g = std::make_unique<Group>(4);
    }
};
inline Cta*& cta() { static thread_local Cta* c = nullptr; return c; }
inline Group* group(unsigned mask, unsigned lane) {
    if (mask == 0xFFFFFFFFu) return cta()->full.get();
    if (mask == 0xFu << (lane & ~3u)) return cta()->quad[lane >> 2].get();
    if (mask == 1u << lane) return nullptr;                                     // a lane alone
    std::abort();                                                               // the kernels use no other mask
}
// the values of all lanes of `mask` at this call (v[i] for the lanes i of the mask)
inline const uint32_t* exchange(unsigned mask, uint32_t v) {
    const unsigned lane = threadIdx.x & 31;
    Group* g = group(mask, lane);
    static thread_local uint32_t own[32];
    if (!g) { own[lane] = v; return own; }
    const unsigned p = g->parity[lane]; g->parity[lane] ^= 1u;
    g->slot[p][lane] = v;
    g->bar.arrive_and_wait();
    return g->slot[p];
}
// run fn() as the 32 lanes of CTA `block`, each on its own thread
template <class F> void run_cta(unsigned block, F fn) {
    Cta c;
    std::vector<std::thread> th;
    for (unsigned lane = 0; lane < 32; lane++)
        th.emplace_back([&, lane] { cta() = &c; blockIdx.x = block; threadIdx.x = lane; fn(); cta() = nullptr; });
    for (auto& t : th) t.join();
}
} // namespace warp_emu

static inline uint32_t __shfl_xor_sync(unsigned mask, uint32_t v, int d) { return warp_emu::exchange(mask, v)[(threadIdx.x & 31) ^ (unsigned)d]; }
static inline bool __any_sync(unsigned mask, bool p) {
    const uint32_t* s = warp_emu::exchange(mask, p);
    for (int i = 0; i < 32; i++) if ((mask >> i & 1u) && s[i]) return true;
    return false;
}
static inline bool __all_sync(unsigned mask, bool p) {
    const uint32_t* s = warp_emu::exchange(mask, p);
    for (int i = 0; i < 32; i++) if ((mask >> i & 1u) && !s[i]) return false;
    return true;
}
static inline unsigned __reduce_or_sync(unsigned mask, unsigned v) {
    const uint32_t* s = warp_emu::exchange(mask, v); unsigned r = 0;
    for (int i = 0; i < 32; i++) if (mask >> i & 1u) r |= s[i];
    return r;
}
static inline void __syncwarp(unsigned mask = 0xFFFFFFFFu) { warp_emu::exchange(mask, 0u); }
