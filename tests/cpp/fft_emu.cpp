// Host build of the device's 64-point transforms, for tests/test_cpu_fft_reference.py to compare with the reference's compiled FFT<64> /
// IFFT<64>: sora_b200/csrc/fixed.cuh and tables.cuh compiled by g++, with the four 16x2 SIMD intrinsics fixed.cuh uses written out per their
// documented semantics (as in packed_emu.cpp).
//   fft64 scalar   r4_butterfly / dft4 in the order of k_front11n's fft_from_regs: FFTSSE<64> on (e, e+16, e+32, e+48) with tw64[.][e],
//                  4 x FFTSSE<16> on (b, b+4, b+8, b+12) with tw16[.][e & 3], 16 x dft4 on (4e .. 4e+3); bin i read from slot bitrev6(i)
//   fft64 packed   the same order on packed words, pk_r4_butterfly / pk_dft4 with fac_tw twiddles: k_front11a's fft_from_regs
//   ifft64         host_ifft64 of tables.cuh as shipped (it builds the STS patterns the device correlates against)
//   sts            HostTables::sts from build_host_tables
//
//   g++ -O2 -std=c++17 -shared -fPIC -DSB_HOST_EMU -I sora_b200/csrc -o fft_emu.so tests/cpp/fft_emu.cpp
#include <cstdint>
#include <cstring>

#define __device__
#define __host__
#define __forceinline__ inline

static inline uint32_t __byte_perm(uint32_t a, uint32_t b, uint32_t s) {        // PRMT, default mode: selector nibble n picks byte n of {b, a}
    const uint64_t v = ((uint64_t)b << 32) | a; uint32_t r = 0;
    for (int i = 0; i < 4; i++) r |= (uint32_t)((v >> (8 * ((s >> (4 * i)) & 7u))) & 0xFFu) << (8 * i);
    return r;
}
static inline uint32_t per_half(uint32_t a, uint32_t b, int (*f)(int, int)) {  // f on the signed halves, each result truncated to 16 bits
    return ((uint32_t)f((int16_t)a, (int16_t)b) & 0xFFFFu) | ((uint32_t)f((int16_t)(a >> 16), (int16_t)(b >> 16)) << 16);
}
static inline uint32_t __vadd2(uint32_t a, uint32_t b) { return per_half(a, b, [](int x, int y) { return x + y; }); }
static inline uint32_t __vmaxs2(uint32_t a, uint32_t b) { return per_half(a, b, [](int x, int y) { return x > y ? x : y; }); }
static inline uint32_t __vmins2(uint32_t a, uint32_t b) { return per_half(a, b, [](int x, int y) { return x < y ? x : y; }); }
static inline uint32_t __vsub2(uint32_t a, uint32_t b) { return per_half(a, b, [](int x, int y) { return x - y; }); }

#include "tables.cuh"

using namespace sb;

static const HostTables& host_tables() { static HostTables* T = [] { HostTables* t = new HostTables(); build_host_tables(*t); return t; }(); return *T; }
static inline int rev6(int i) { int r = 0; for (int b = 0; b < 6; b++) r |= ((i >> b) & 1) << (5 - b); return r; }

// n vectors of 64 packed words each; packed = 0: scalar r4_butterfly / dft4, 1: pk_r4_butterfly / pk_dft4
extern "C" void emu_fft64(int packed, uint64_t n, const uint32_t* in, uint32_t* out) {
    const HostTables& T = host_tables();
    for (uint64_t v = 0; v < n; v++) {
        uint32_t x[64]; memcpy(x, in + 64 * v, sizeof x);
        for (int e = 0; e < 16; e++) {
            const cs16 w1 = unpack(T.tw64[0][e]), w2 = unpack(T.tw64[1][e]), w3 = unpack(T.tw64[2][e]);
            if (packed) pk_r4_butterfly(x[e], x[e + 16], x[e + 32], x[e + 48], fac_tw(w1), fac_tw(w2), fac_tw(w3));
            else { cs16 a = unpack(x[e]), b = unpack(x[e + 16]), c = unpack(x[e + 32]), d = unpack(x[e + 48]);
                   r4_butterfly(a, b, c, d, w1, w2, w3); x[e] = pack(a); x[e + 16] = pack(b); x[e + 32] = pack(c); x[e + 48] = pack(d); }
        }
        for (int e = 0; e < 16; e++) {
            const int base = (e >> 2) * 16 + (e & 3);
            const cs16 w1 = unpack(T.tw16[0][e & 3]), w2 = unpack(T.tw16[1][e & 3]), w3 = unpack(T.tw16[2][e & 3]);
            if (packed) pk_r4_butterfly(x[base], x[base + 4], x[base + 8], x[base + 12], fac_tw(w1), fac_tw(w2), fac_tw(w3));
            else { cs16 a = unpack(x[base]), b = unpack(x[base + 4]), c = unpack(x[base + 8]), d = unpack(x[base + 12]);
                   r4_butterfly(a, b, c, d, w1, w2, w3); x[base] = pack(a); x[base + 4] = pack(b); x[base + 8] = pack(c); x[base + 12] = pack(d); }
        }
        for (int e = 0; e < 16; e++) {
            if (packed) pk_dft4(x[4 * e], x[4 * e + 1], x[4 * e + 2], x[4 * e + 3]);
            else { cs16 a = unpack(x[4 * e]), b = unpack(x[4 * e + 1]), c = unpack(x[4 * e + 2]), d = unpack(x[4 * e + 3]);
                   dft4(a, b, c, d); x[4 * e] = pack(a); x[4 * e + 1] = pack(b); x[4 * e + 2] = pack(c); x[4 * e + 3] = pack(d); }
        }
        for (int i = 0; i < 64; i++) out[64 * v + i] = x[rev6(i)];
    }
}
// n vectors of 64 packed words through host_ifft64 (natural-order output)
extern "C" void emu_ifft64(uint64_t n, const uint32_t* in, uint32_t* out) {
    const HostTables& T = host_tables();
    for (uint64_t v = 0; v < n; v++) {
        cs16 x[64]; for (int i = 0; i < 64; i++) x[i] = unpack(in[64 * v + i]);
        host_ifft64(x, T);
        for (int i = 0; i < 64; i++) out[64 * v + i] = pack(x[i]);
    }
}
// the device's STS correlation patterns, [16][16] packed words
extern "C" void emu_sts(uint32_t* out) { memcpy(out, host_tables().sts, sizeof host_tables().sts); }
