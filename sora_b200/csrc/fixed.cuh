// sora_b200 — lane-exact fixed-point primitives for sm_90a device code.
//
// Scalar (one complex int16 sample per call) definitions of the arithmetic the reference performs with
// SSE vectors.  Each function cites the reference primitive whose per-lane result it reproduces
// (kernel/core/inc/vector128.h).  These are written against the *documented instruction semantics*
// (pmaddwd wraps at 2^31, psraw/psrad are arithmetic, paddsw saturates, "conj"/"mul_j" are one's
// complement) and are checked bit-for-bit against the SSE oracle by tests/test_gpu_stages.py.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

namespace sb {

struct cs16 { int re, im; };     // values always kept in int16 range (sign-extended)

__host__ __device__ __forceinline__ int sx16(int v) { return (int)(short)v; }                 // truncate to int16
__host__ __device__ __forceinline__ int sat16(int v) { return v > 32767 ? 32767 : (v < -32768 ? -32768 : v); }
__host__ __device__ __forceinline__ int wadd(int a, int b) { return (int)((unsigned)a + (unsigned)b); }   // pmaddwd / paddd wrap

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

} // namespace sb
