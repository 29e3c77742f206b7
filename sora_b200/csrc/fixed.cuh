// sora_b200 — lane-exact fixed-point primitives for sm_90a device code.
//
// Scalar (one complex int16 sample per call) definitions of the arithmetic the reference performs with
// SSE vectors.  Each function cites the reference primitive whose per-lane result it reproduces
// (kernel/core/inc/vector128.h).  These are written against the *documented instruction semantics*
// (pmaddwd wraps at 2^31, psraw/psrad are arithmetic, paddsw saturates, "conj"/"mul_j" are one's
// complement) and are checked bit-for-bit against the SSE oracle by tests/test_gpu_stages.py.
#pragma once
#include <stdint.h>
#ifndef SB_HOST_EMU                  // tests/cpp/packed_emu.cpp compiles this header for the host with the intrinsics written out
#include <cuda_runtime.h>
#endif

namespace sb {

struct cs16 { int re, im; };     // values always kept in int16 range (sign-extended)

__host__ __device__ __forceinline__ int sx16(int v) { return (int)(short)v; }                 // truncate to int16
__host__ __device__ __forceinline__ int sat16(int v) { return v > 32767 ? 32767 : (v < -32768 ? -32768 : v); }
__host__ __device__ __forceinline__ int wadd(int a, int b) { return (int)((unsigned)a + (unsigned)b); }   // pmaddwd / paddd wrap
__host__ __device__ __forceinline__ int wsub(int a, int b) { return (int)((unsigned)a - (unsigned)b); }   // psubd / int C wrap
__host__ __device__ __forceinline__ int wneg(int a) { return (int)(0u - (unsigned)a); }                  // int C negate (INT_MIN stays)

__host__ __device__ __forceinline__ cs16 unpack(uint32_t w) { cs16 c; c.re = (int)(short)(w & 0xFFFF); c.im = (int)w >> 16; return c; }
__host__ __device__ __forceinline__ uint32_t pack(cs16 c) { return ((uint32_t)c.re & 0xFFFFu) | ((uint32_t)c.im << 16); }
__host__ __device__ __forceinline__ cs16 mk(int re, int im) { cs16 c; c.re = re; c.im = im; return c; }

__host__ __device__ __forceinline__ cs16 sra(cs16 a, int n) { return mk(a.re >> n, a.im >> n); }          // psraw
__host__ __device__ __forceinline__ cs16 adds(cs16 a, cs16 b) { return mk(sat16(a.re + b.re), sat16(a.im + b.im)); }   // paddsw
__host__ __device__ __forceinline__ cs16 subs(cs16 a, cs16 b) { return mk(sat16(a.re - b.re), sat16(a.im - b.im)); }   // psubsw
__host__ __device__ __forceinline__ cs16 subw(cs16 a, cs16 b) { return mk(sx16(a.re - b.re), sx16(a.im - b.im)); }     // psubw
__host__ __device__ __forceinline__ cs16 cnot(cs16 a) { return mk(~a.re, ~a.im); }                          // pxor with all-ones
__host__ __device__ __forceinline__ int neg16(int v) { return sx16(-v); }                                   // psignw negate (-32768 stays)

// a * conj(b), full int32 re/im                       (vector128.h:1031-1037 conj_mul)
__host__ __device__ __forceinline__ void cmul_conj32(int& re, int& im, cs16 a, cs16 b) {
    re = wadd(a.re * b.re, a.im * b.im);
    im = wadd(neg16(b.im) * a.re, b.re * a.im);
}
// a * b, full int32 re/im                             (vector128.h:1072-1078 mul)
__host__ __device__ __forceinline__ void cmul32(int& re, int& im, cs16 a, cs16 b) {
    re = wadd(a.re * b.re, a.im * neg16(b.im));
    im = wadd(a.re * b.im, a.im * b.re);
}
// Q15 product with truncating repack                  (vector128.h:1199-1211 mul(vcs,vcs))
__host__ __device__ __forceinline__ cs16 cmul_q15(cs16 a, cs16 b) {
    int re, im; cmul32(re, im, a, b); return mk(sx16(re >> 15), sx16(im >> 15));
}
// FFT twiddle product (one's-complement conjugate)     (vector128.h:1235-1246 mul_shift)
__host__ __device__ __forceinline__ cs16 cmul_tw(cs16 a, cs16 w) {
    int re = wadd(a.re * w.re, a.im * (int)(short)~w.im);
    int im = wadd(a.re * w.im, a.im * w.re);
    return mk(sx16(re >> 15), sx16(im >> 15));
}
// approximate multiply by j                            (vector128.h:1258-1261 mul_j)
__host__ __device__ __forceinline__ cs16 mulj(cs16 a) { return mk(~a.im, a.re); }

// Radix-4 DIF butterfly of FFT<N> first stages         (core/inc/fft_r4dif.h:12-47 FFTSSE)
// in: a,b,c,d at strides N/4; out: y0 (no twiddle), y1 (x W^2e), y2 (x W^e), y3 (x W^3e) at the same four slots
__host__ __device__ __forceinline__ void r4_butterfly(cs16& a, cs16& b, cs16& c, cs16& d, cs16 w1, cs16 w2, cs16 w3) {
    a = sra(a, 2); b = sra(b, 2); c = sra(c, 2); d = sra(d, 2);
    cs16 ac = adds(a, c), bd = adds(b, d), a_c = subs(a, c), b_d = subs(b, d);
    cs16 jbd = mulj(b_d);
    a = adds(ac, bd);
    b = cmul_tw(subs(ac, bd), w2);
    c = cmul_tw(subs(a_c, jbd), w1);
    d = cmul_tw(adds(a_c, jbd), w3);
}
// 4-point DFT inside one SSE vector                    (core/inc/fft_r4dif.h:62-86 FFTSSEEx<4>)
// outputs stay in the vector's lane order [X0, X2, X1, X3]
__host__ __device__ __forceinline__ void dft4(cs16& v0, cs16& v1, cs16& v2, cs16& v3) {
    cs16 x0 = sra(v0, 2), x1 = sra(v1, 2), x2 = sra(v2, 2), x3 = sra(v3, 2);
    cs16 s0 = adds(x0, x2), s1 = adds(x1, x3), s2 = adds(cnot(x2), x0), s3 = adds(cnot(x3), x1);
    cs16 t3 = mk(s3.im, ~s3.re);                      // lane 3 times -j (swap, then complement the new im)
    v0 = adds(s0, s1); v1 = adds(cnot(s1), s0); v2 = adds(s2, t3); v3 = adds(cnot(t3), s2);
}

// ------------------------------------------------------------------------------------------------
// Packed forms: one complex int16 per 32-bit word, re in bits 0-15, im in bits 16-31 (the layout of pack()), on the 16x2 SIMD
// integer instructions.  Each one states when it equals its scalar counterpart above; tests/test_cpu_packed.py and
// tests/test_cpu_packed_rot.py check that on the host, exhaustively or on random and edge words.
// ------------------------------------------------------------------------------------------------
// paddw / psubw: per-half wrap-around.  Equal to adds / subs wherever the exact sum lies in [-32768, 32767].
__device__ __forceinline__ uint32_t pk_add(uint32_t a, uint32_t b) { return __vadd2(a, b); }
__device__ __forceinline__ uint32_t pk_sub(uint32_t a, uint32_t b) { return __vsub2(a, b); }
// sra(a, N), any input: logical shift, clear the bits the high half pushed into the low one, sign-extend each half from bit 15 - N
// as (t ^ s) - s, the subtraction written as the add of -s (16x2 adds take no negated operand)
template <int N> __device__ __forceinline__ uint32_t pk_sra(uint32_t a) {
    const uint32_t m = (0xFFFFu >> N) * 0x10001u, s = (0x8000u >> N) * 0x10001u, ns = (0x10000u - (0x8000u >> N)) * 0x10001u;
    return __vadd2(((a >> N) & m) ^ s, ns);
}
__device__ __forceinline__ uint32_t pk_mulj(uint32_t a) { return __byte_perm(a, 0, 0x1032) ^ 0x0000FFFFu; }    // mulj: (~im, re), any input
__device__ __forceinline__ uint32_t pk_mulmj(uint32_t a) { return __byte_perm(a, 0, 0x1032) ^ 0xFFFF0000u; }   // (im, ~re): dft4's t3, any input
// Factor of a complex product a * b whose components are then taken as sx16(x >> S): b's halves pre-multiplied by 2^(16 - S), `nim` being
// what a.im is multiplied by in the real part.  The 32-bit wrapped sum a.re * (re << (16 - S)) + a.im * (nim << (16 - S)) is
// x << (16 - S) mod 2^32, whose high half is bits S..S+15 of x, i.e. sx16(x >> S): one PRMT repacks both components.  Exact for any input.
struct cfac { int re, im, nim; };
template <int S> __device__ __forceinline__ cfac mkfac(int re, int im, int nim) { return cfac{re * (1 << (16 - S)), im * (1 << (16 - S)), nim * (1 << (16 - S))}; }
__device__ __forceinline__ cfac fac_q15(cs16 b) { return mkfac<15>(b.re, b.im, neg16(b.im)); }        // cmul_q15(a, b)
__device__ __forceinline__ cfac fac_tw(cs16 w) { return mkfac<15>(w.re, w.im, (int)(short)~w.im); }   // cmul_tw(a, w)
__device__ __forceinline__ cfac fac_mul8(cs16 b) { return mkfac<8>(b.re, b.im, neg16(b.im)); }        // cmul32(a, b) >> 8, sx16
__device__ __forceinline__ uint32_t pk_cmul(int re, int im, cfac f) {
    const uint32_t x = (uint32_t)re * (uint32_t)f.re + (uint32_t)im * (uint32_t)f.nim, y = (uint32_t)re * (uint32_t)f.im + (uint32_t)im * (uint32_t)f.re;
    return __byte_perm(x, y, 0x7632);
}
__device__ __forceinline__ uint32_t pk_cmul(uint32_t a, cfac f) { return pk_cmul((int)(short)a, (int)a >> 16, f); }
// The two 32-bit sums of pk_cmul without the repack: (int)x >> 16 and (int)y >> 16 are the product's re and im, ready for the next product.
__device__ __forceinline__ void pk_cmul_xy(int re, int im, const cfac& f, int& x, int& y) {
    x = (int)((uint32_t)re * (uint32_t)f.re + (uint32_t)im * (uint32_t)f.nim); y = (int)((uint32_t)re * (uint32_t)f.im + (uint32_t)im * (uint32_t)f.re);
}
// cmul_q15(a, unpack(w)) for a word w of the rotation table, (round(32767 cos), -round(32767 sin)): both halves lie in [-32767, 32767],
// where neg16 is plain negation, so the real part is a.re * re - a.im * im and the factor needs no third component.  Built straight from
// the word: each half sign-extended and doubled (S = 15 of mkfac).
struct rfac { int re, im; };
__device__ __forceinline__ rfac fac_rotw(uint32_t w) { return rfac{(int)(w << 16) >> 15, (int)(w & 0xFFFF0000u) >> 15}; }
__device__ __forceinline__ void pk_cmul_xy(int re, int im, rfac f, int& x, int& y) {
    x = (int)((uint32_t)re * (uint32_t)f.re - (uint32_t)im * (uint32_t)f.im); y = (int)((uint32_t)re * (uint32_t)f.im + (uint32_t)im * (uint32_t)f.re);
}
__device__ __forceinline__ uint32_t pk_cmul(int re, int im, rfac f) { int x, y; pk_cmul_xy(re, im, f, x, y); return __byte_perm((uint32_t)x, (uint32_t)y, 0x7632); }
// sx16(th + 0x8000) for th in [-32768, 32767] (a pilot angle turned by pi): flipping bit 15 and every bit above it.  flip = 0 leaves th.
__host__ __device__ __forceinline__ int turn_pi(int th, bool flip) { return th ^ (flip ? (int)0xFFFF8000u : 0); }
// The demapper's index byte per half, (uint8)min(max(v >> 4, -128), 127): >> 4 is monotone and maps -2048 / 2047 to -128 / 127, so
// clamping v to [-2048, 2047] first gives the same value, and its bits 4..11 are that byte.  Any input; re's byte in bits 4..11, im's in 20..27.
__device__ __forceinline__ uint32_t pk_demap_clamp(uint32_t a) { return __vmins2(__vmaxs2(a, 0xF800F800u), 0x07FF07FFu); }

// r4_butterfly on packed words.  After the >> 2 every component lies in [-8192, 8191]: ac, bd in [-16384, 16382], a_c, b_d in
// [-16383, 16383], jbd in [-16384, 16383]; so ac +- bd and a_c -+ jbd lie in [-32768, 32767] and every saturating add of the scalar
// butterfly is a wrap-around one here.
__device__ __forceinline__ void pk_r4_butterfly(uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d, const cfac& w1, const cfac& w2, const cfac& w3) {
    a = pk_sra<2>(a); b = pk_sra<2>(b); c = pk_sra<2>(c); d = pk_sra<2>(d);
    const uint32_t ac = pk_add(a, c), bd = pk_add(b, d), a_c = pk_sub(a, c), b_d = pk_sub(b, d), jbd = pk_mulj(b_d);
    a = pk_add(ac, bd);
    b = pk_cmul(pk_sub(ac, bd), w2);
    c = pk_cmul(pk_sub(a_c, jbd), w1);
    d = pk_cmul(pk_add(a_c, jbd), w3);
}
// dft4 on packed words.  x in [-8192, 8191] after the >> 2; s0, s1, s2 = x0 - x2 - 1, s3 in [-16384, 16382]; t3, ~s1, ~t3 in
// [-16384, 16383]; every output sum lies in [-32768, 32765], so again no saturating add can clip.
__device__ __forceinline__ void pk_dft4(uint32_t& v0, uint32_t& v1, uint32_t& v2, uint32_t& v3) {
    const uint32_t x0 = pk_sra<2>(v0), x1 = pk_sra<2>(v1), x2 = pk_sra<2>(v2), x3 = pk_sra<2>(v3);
    const uint32_t s0 = pk_add(x0, x2), s1 = pk_add(x1, x3), s2 = pk_add(~x2, x0), s3 = pk_add(~x3, x1);
    const uint32_t t3 = pk_mulmj(s3);
    v0 = pk_add(s0, s1); v1 = pk_add(~s1, s0); v2 = pk_add(s2, t3); v3 = pk_add(~t3, s2);
}

} // namespace sb
