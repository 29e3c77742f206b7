// Host build of the per-bin helpers of k_front11a's phase tracker (sora_b200/csrc/fixed.cuh: fac_rotw, pk_cmul_xy, turn_pi) next to the
// scalar primitives they replace, the same way tests/cpp/packed_emu.cpp builds the FFT helpers.  tests/test_cpu_packed_rot.py compares them.
//
//   g++ -O2 -std=c++17 -shared -fPIC -DSB_HOST_EMU -I sora_b200/csrc -o packed_rot_emu.so tests/cpp/packed_rot_emu.cpp
#include <cstdint>

#define __device__
#define __host__
#define __forceinline__ inline

static inline uint32_t __byte_perm(uint32_t a, uint32_t b, uint32_t s) {        // PRMT, default mode: selector nibble n picks byte n of {b, a}
    const uint64_t v = ((uint64_t)b << 32) | a; uint32_t r = 0;
    for (int i = 0; i < 4; i++) r |= (uint32_t)((v >> (8 * ((s >> (4 * i)) & 7u))) & 0xFFu) << (8 * i);
    return r;
}
static inline uint32_t per_half(uint32_t a, uint32_t b, int (*f)(int, int)) {
    return ((uint32_t)f((int16_t)a, (int16_t)b) & 0xFFFFu) | ((uint32_t)f((int16_t)(a >> 16), (int16_t)(b >> 16)) << 16);
}
static inline uint32_t __vadd2(uint32_t a, uint32_t b) { return per_half(a, b, [](int x, int y) { return x + y; }); }
static inline uint32_t __vmaxs2(uint32_t a, uint32_t b) { return per_half(a, b, [](int x, int y) { return x > y ? x : y; }); }
static inline uint32_t __vmins2(uint32_t a, uint32_t b) { return per_half(a, b, [](int x, int y) { return x < y ? x : y; }); }
static inline uint32_t __vsub2(uint32_t a, uint32_t b) { return per_half(a, b, [](int x, int y) { return x - y; }); }

#include "fixed.cuh"

using namespace sb;

// op 0: pk_cmul(a, fac_rotw(w)) vs cmul_q15(a, unpack(w)) (w a rotation-table word: both halves in [-32767, 32767]);
// op 1: k_front11a's equalise + phase compensation, C = (F * eq) * comp with E handed over as the halves of pk_cmul_xy's sums, vs the
//       scalar chain cmul_q15(sx16(cmul32(F, ch) >> 8), unpack(w)); b = ch, c = w
extern "C" void packed_rot(int op, const uint32_t* a, const uint32_t* b, const uint32_t* c, uint32_t n, uint32_t* got, uint32_t* want) {
    for (uint32_t i = 0; i < n; i++) {
        const cs16 x = unpack(a[i]);
        if (op == 0) { got[i] = pk_cmul((int)(short)a[i], (int)a[i] >> 16, fac_rotw(b[i])); want[i] = pack(cmul_q15(x, unpack(b[i]))); continue; }
        int ex, ey, cx, cy;
        pk_cmul_xy(x.re, x.im, fac_mul8(unpack(b[i])), ex, ey);
        pk_cmul_xy(ex >> 16, ey >> 16, fac_rotw(c[i]), cx, cy);
        got[i] = ((uint32_t)(cx >> 16) & 0xFFFFu) | ((uint32_t)(cy >> 16) << 16);
        int re, im; cmul32(re, im, x, unpack(b[i]));
        want[i] = pack(cmul_q15(mk(sx16(re >> 8), sx16(im >> 8)), unpack(c[i])));
    }
}
// turn_pi(th, flip) vs sx16(th + 0x8000) / th, for every int16 angle
extern "C" void turn(const int32_t* th, uint32_t n, int32_t* got, int32_t* want) {
    for (uint32_t i = 0; i < n; i++) {
        got[2 * i] = turn_pi(th[i], false); want[2 * i] = th[i];
        got[2 * i + 1] = turn_pi(th[i], true); want[2 * i + 1] = sx16(th[i] + 0x8000);
    }
}
