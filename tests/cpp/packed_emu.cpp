// Host build of the packed complex-int16 helpers of sora_b200/csrc/fixed.cuh next to the scalar primitives they replace in k_front11a: the
// header itself compiled by g++, with the four 16x2 SIMD intrinsics it uses written out per their documented semantics.  Each entry point
// runs one helper over n input words and returns what the scalar path returns, both packed, so tests/test_cpu_packed.py compares them.
//
//   g++ -O2 -std=c++17 -shared -fPIC -DSB_HOST_EMU -I sora_b200/csrc -o packed_emu.so tests/cpp/packed_emu.cpp
#include <algorithm>
#include <cstdint>

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

#include "fixed.cuh"

using namespace sb;

// op: 0 pk_sra<1>, 1 pk_sra<2>, 2 pk_sra<4>, 3 pk_mulj, 4 pk_mulmj (against dft4's t3), 5 demap index bytes (re | im << 8)
extern "C" void packed_unary(int op, const uint32_t* a, uint32_t n, uint32_t* got, uint32_t* want) {
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t w = a[i]; const cs16 c = unpack(w);
        switch (op) {
            case 0: got[i] = pk_sra<1>(w); want[i] = pack(sra(c, 1)); break;
            case 1: got[i] = pk_sra<2>(w); want[i] = pack(sra(c, 2)); break;
            case 2: got[i] = pk_sra<4>(w); want[i] = pack(sra(c, 4)); break;
            case 3: got[i] = pk_mulj(w); want[i] = pack(mulj(c)); break;
            case 4: got[i] = pk_mulmj(w); want[i] = pack(mk(c.im, ~c.re)); break;
            default: {
                const uint32_t k = pk_demap_clamp(w);
                got[i] = ((k >> 4) & 0xFFu) | (((k >> 20) & 0xFFu) << 8);
                want[i] = ((unsigned)std::min(std::max(c.re >> 4, -128), 127) & 0xFFu) | (((unsigned)std::min(std::max(c.im >> 4, -128), 127) & 0xFFu) << 8);
            }
        }
    }
}
// op: 0 pk_cmul(fac_q15) vs cmul_q15, 1 pk_cmul(fac_tw) vs cmul_tw, 2 pk_cmul(fac_mul8) vs cmul32 >> 8,
//     3 fcomp of k_front11a (pk_cmul of the halves >> 1) vs cmul_q15(sra(a, 1), b)
extern "C" void packed_cmul(int op, const uint32_t* a, const uint32_t* b, uint32_t n, uint32_t* got, uint32_t* want) {
    for (uint32_t i = 0; i < n; i++) {
        const cs16 x = unpack(a[i]), y = unpack(b[i]);
        switch (op) {
            case 0: got[i] = pk_cmul(a[i], fac_q15(y)); want[i] = pack(cmul_q15(x, y)); break;
            case 1: got[i] = pk_cmul(a[i], fac_tw(y)); want[i] = pack(cmul_tw(x, y)); break;
            case 2: { got[i] = pk_cmul(a[i], fac_mul8(y)); int re, im; cmul32(re, im, x, y); want[i] = pack(mk(sx16(re >> 8), sx16(im >> 8))); break; }
            default: got[i] = pk_cmul((int)(short)a[i] >> 1, (int)a[i] >> 17, fac_q15(y)); want[i] = pack(cmul_q15(sra(x, 1), y));
        }
    }
}
// The radix-4 butterfly (op 0, twiddles w[3 i .. 3 i + 2]) and dft4 (op 1) on four words per case, packed against scalar.
extern "C" void packed_butterfly(int op, const uint32_t* in, const uint32_t* w, uint32_t n, uint32_t* got, uint32_t* want) {
    for (uint32_t i = 0; i < n; i++) {
        uint32_t p[4]; cs16 s[4];
        for (int k = 0; k < 4; k++) { p[k] = in[4 * i + k]; s[k] = unpack(p[k]); }
        if (op == 0) {
            const cs16 w1 = unpack(w[3 * i]), w2 = unpack(w[3 * i + 1]), w3 = unpack(w[3 * i + 2]);
            pk_r4_butterfly(p[0], p[1], p[2], p[3], fac_tw(w1), fac_tw(w2), fac_tw(w3));
            r4_butterfly(s[0], s[1], s[2], s[3], w1, w2, w3);
        } else {
            pk_dft4(p[0], p[1], p[2], p[3]);
            dft4(s[0], s[1], s[2], s[3]);
        }
        for (int k = 0; k < 4; k++) { got[4 * i + k] = p[k]; want[4 * i + k] = pack(s[k]); }
    }
}
