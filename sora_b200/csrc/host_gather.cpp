// sora_b200 — host side of option "host_decimate": TDownSample2 (kernel/bb/Brick11/src/samples.hpp:27-49 keeps samples 0 and 2 of every 4)
// performed by the host threads while they fill the pinned staging buffers, so that only the 20 Msps stream crosses PCIe.
// dst[j] = src[2 j], j < n2.  The packed copy is written once and read by the DMA engine only: streaming stores keep it from costing a
// read-for-ownership and from pushing the capture out of the cache; with AVX-512 a whole 64-byte line leaves per store (one write-combining
// buffer, one bus transaction) and the even samples of two vectors are picked by a single two-source permute.  Chosen once at run time.
// Software prefetch: measured on a Sapphire Rapids class host (tools/microbench/host_gather_bench.cpp), the hardware prefetcher alone streams
// 11 GB/s per thread through this loop, with prefetchnta 2 KB ahead 7.6 GB/s — the hints evict what the prefetcher had fetched.
#include <immintrin.h>
#include <cstdint>

namespace sb {

static void gather_even_sse2(const uint32_t* __restrict__ src, uint32_t n2, uint32_t* __restrict__ dst) {
    uint32_t j = 0;
    for (; j < n2 && ((uintptr_t)(dst + j) & 15u); j++) dst[j] = src[2 * j];
    for (; j + 8 <= n2; j += 8) {
        const __m128 a = _mm_loadu_ps((const float*)(src + 2 * j)), b = _mm_loadu_ps((const float*)(src + 2 * j + 4));
        const __m128 c = _mm_loadu_ps((const float*)(src + 2 * j + 8)), d = _mm_loadu_ps((const float*)(src + 2 * j + 12));
        _mm_stream_ps((float*)(dst + j), _mm_shuffle_ps(a, b, 0x88));
        _mm_stream_ps((float*)(dst + j + 4), _mm_shuffle_ps(c, d, 0x88));
    }
    for (; j < n2; j++) dst[j] = src[2 * j];
}

__attribute__((target("avx512f"))) static void gather_even_avx512(const uint32_t* __restrict__ src, uint32_t n2, uint32_t* __restrict__ dst) {
    uint32_t j = 0;
    for (; j < n2 && ((uintptr_t)(dst + j) & 63u); j++) dst[j] = src[2 * j];
    const __m512i even = _mm512_setr_epi32(0, 2, 4, 6, 8, 10, 12, 14, 16, 18, 20, 22, 24, 26, 28, 30);
    for (; j + 32 <= n2; j += 32) {
        const __m512i a = _mm512_loadu_si512(src + 2 * j), b = _mm512_loadu_si512(src + 2 * j + 16);
        const __m512i c = _mm512_loadu_si512(src + 2 * j + 32), d = _mm512_loadu_si512(src + 2 * j + 48);
        _mm512_stream_si512((__m512i*)(dst + j), _mm512_permutex2var_epi32(a, even, b));
        _mm512_stream_si512((__m512i*)(dst + j + 16), _mm512_permutex2var_epi32(c, even, d));
    }
    for (; j < n2; j++) dst[j] = src[2 * j];
}

void gather_even(const uint32_t* src, uint32_t n2, uint32_t* dst) {
    static const bool wide = __builtin_cpu_supports("avx512f");
    if (wide) gather_even_avx512(src, n2, dst);
    else gather_even_sse2(src, n2, dst);
}

}  // namespace sb
