// Host-side TDownSample2 gather (sora_b200/csrc/host_gather.cpp) timed alone: T threads over 16 384 slots of 9 824 samples (643 MB read,
// 322 MB written into a three-chunk staging ring, like the library's pinned buffers).
//   g++ -O2 -std=c++17 -pthread -o host_gather_bench host_gather_bench.cpp ../../sora_b200/csrc/host_gather.cpp && ./host_gather_bench 14
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>
#include <immintrin.h>
#include <sys/mman.h>
namespace sb { void gather_even(const uint32_t* src, uint32_t n2, uint32_t* dst); }
int main(int argc, char** argv) {
    const int T = argc > 1 ? atoi(argv[1]) : 1;
    const size_t slot = 9824, nslots = 16384, nsrc = slot * nslots, ring = slot / 2 * 4096 * 3;
    uint32_t* src = (uint32_t*)mmap(0, nsrc * 4, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    uint32_t* dst = (uint32_t*)mmap(0, ring * 4, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (src == MAP_FAILED || dst == MAP_FAILED) return 1;
    memset(src, 1, nsrc * 4); memset(dst, 1, ring * 4);
    double best = 1e30;
    for (int rep = 0; rep < 4; rep++) {
        const auto t0 = std::chrono::steady_clock::now();
        std::vector<std::thread> th;
        for (int w = 0; w < T; w++) th.emplace_back([&, w]() {
            for (size_t f = nslots * w / T; f < nslots * (w + 1) / T; f++) sb::gather_even(src + f * slot, slot / 2, dst + (f % (3 * 4096)) * (slot / 2));
            _mm_sfence();
        });
        for (auto& t : th) t.join();
        const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        if (rep && ms < best) best = ms;
    }
    printf("host gather, %2d threads: %.1f ms per 16384 slots, %.1f GB/s read + %.1f GB/s written (a 65536-slot step: %.1f ms)\n", T,
           best, nsrc * 4 / best / 1e6, nsrc * 2 / best / 1e6, best * 4);
    return 0;
}
