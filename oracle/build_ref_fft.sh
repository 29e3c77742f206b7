#!/bin/sh
# oracle/_ref/libfft_ref.so: the reference's fixed-point OFDM transforms, compiled from its own headers where they lie: FFT<64>
# (kernel/core/inc/fft_r4dif.h), IFFT<64> and IFFT<128> (ifft_r4dif.h), with the twiddle and bit-reversal tables of fft_lut_twiddle.h and
# fft_lut_bitreversal.h.  Nothing of the transforms is restated: the radix-4 stages, FFTSSEEx<4> / <8>, IFFTSSEEx<4> / <8>, the tables
# and the bit-reversed read-out all come from source.
#
# The four headers include <vector128.h> with angle brackets, so the shim directory, first on the include path, supplies it; their quoted
# includes of each other resolve beside them in the reference tree.  The real vector128.h is not used: it declares the SSSE3 / SSE4
# intrinsics itself as extern "C" functions (vector128.h:28-72), which g++ defines as inline functions of its own headers, and the debug tap
# below must sit inside the saturating adds, the pack and pmaddwd.  So the shim defines only what the four headers use, each operation as
# the intrinsic vector128.h maps it to (line cited):
#   types      vcs (COMPLEX16 x 4, :138), and the vs / vi views mul_shift and conj_mul_shift go through (:130, :132); COMPLEX16 (complex.h:5)
#   shifts     shift_right on vcs (_mm_srai_epi16, :832) and on vi (_mm_srai_epi32, :830)
#   arithmetic saturated_add / saturated_sub on vcs (_mm_adds_epi16 / _mm_subs_epi16, :645, :655), xor on vcs (_mm_xor_si128, :567),
#              sign on vcs (_mm_sign_epi16, :535)
#   shuffles   permutate<imm> (_mm_shuffle_epi32, :688), permutate_high<imm> / permutate_low<imm> (_mm_shufflehi/lo_epi16, :683, :677)
#   complex    conj (:966, an XOR of the imaginary halves), conjre (:952-961, psignw: a true negate of the real halves), flip (:992-996),
#              mul_j (:1258-1261, flip then XOR), pairwise_muladd (_mm_madd_epi16, :920), pack(vi, vi) (:876-883: each 32-bit lane masked
#              to its low 16 bits and interleaved, so it wraps; not packssdw), mul_shift (:1235-1246), conj_mul_shift (:1215-1231)
#   constants  the vector128_consts masks (:179-284) the transforms and helpers name
#   macros     DSP_INLINE / DSP_INLINE1 (:22-24); __declspec(selectany / align(16) / deprecated) of the table headers
# A debug tap counts, per call of the entry points, the lanes where saturated_add / saturated_sub clipped, where pack dropped significant
# bits (the shifted 32-bit value does not fit in int16) and where pmaddwd wrapped (both products 2^30): ref_fft_debug below.
# Nothing of the reference is copied into the repository.  TEST INFRASTRUCTURE ONLY.
#   usage: oracle/build_ref_fft.sh [reference root, default /root/reference]
set -e
REF="${1:-/root/reference}"
SRC="$REF/kernel/core/inc"
HERE="$(cd "$(dirname "$0")" && pwd)"
[ -f "$SRC/fft_r4dif.h" ] || { echo "build_ref_fft: $SRC/fft_r4dif.h not found (fine outside the build container: the prebuilt oracle/_ref is used)"; exit 0; }
INC="$HERE/_ref/fft_inc"
rm -rf "$INC"; mkdir -p "$INC"
cat > "$INC/vector128.h" <<'SHIM'
#pragma once
#include <smmintrin.h>
#include <stddef.h>
#include <string.h>
#define DSP_INLINE inline __attribute__((always_inline))
#define DSP_INLINE1 inline
#define __declspec(x) SB_DECLSPEC_##x
#define SB_DECLSPEC_selectany
#define SB_DECLSPEC_deprecated
#define SB_DECLSPEC_align(n) __attribute__((aligned(n)))
typedef struct _COMPLEX16 { short re, im; } COMPLEX16;
#define SB_VEC(NAME, TDATA)                                                                                     \
struct NAME {                                                                                                   \
    static const size_t size = 16 / sizeof(TDATA);                                                              \
    NAME() {}                                                                                                   \
    explicit NAME(__m128i r) : _raw(r) {}                                                                       \
    template<typename TA> explicit NAME(const TA& a) : _raw((__m128i)a) {}                                      \
    operator __m128i() const { return _raw; }                                                                   \
    __m128i _raw;                                                                                               \
};
SB_VEC(vs, short)
SB_VEC(vi, int)
SB_VEC(vcs, COMPLEX16)
namespace sbref { void tap_sat(__m128i sat, __m128i wrap, int op); void tap_pack(__m128i v); void tap_madd(__m128i v); }
class vector128_consts {
public:
    template<typename T> static T __0x0000FFFF0000FFFF0000FFFF0000FFFF() { return (T)_mm_set1_epi32(0x0000FFFF); }
    template<typename T> static T __0xFFFF0000FFFF0000FFFF0000FFFF0000() { return (T)_mm_set1_epi32((int)0xFFFF0000); }
    template<typename T> static T __0xFFFFFFFF00000000FFFFFFFF00000000() { return (T)_mm_set_epi32(-1, 0, -1, 0); }
    template<typename T> static T __0xFFFFFFFFFFFFFFFF0000000000000000() { return (T)_mm_set_epi32(-1, -1, 0, 0); }
    template<typename T> static T __0xFFFF0000FFFF00000000000000000000() { return (T)_mm_set_epi32((int)0xFFFF0000, (int)0xFFFF0000, 0, 0); }
    template<typename T> static T __0xFFFF0000000000000000000000000000() { return (T)_mm_set_epi32((int)0xFFFF0000, 0, 0, 0); }
};
inline vcs shift_right(const vcs& a, int n) { return vcs(_mm_srai_epi16(a, n)); }
inline vi shift_right(const vi& a, int n) { return vi(_mm_srai_epi32(a, n)); }
inline vcs saturated_add(const vcs& a, const vcs& b) { __m128i r = _mm_adds_epi16(a, b); sbref::tap_sat(r, _mm_add_epi16(a, b), 0); return vcs(r); }
inline vcs saturated_sub(const vcs& a, const vcs& b) { __m128i r = _mm_subs_epi16(a, b); sbref::tap_sat(r, _mm_sub_epi16(a, b), 1); return vcs(r); }
inline vcs xor(const vcs& a, const vcs& b) { return vcs(_mm_xor_si128(a, b)); }
inline vcs sign(const vcs& a, const vcs& b) { return vcs(_mm_sign_epi16(a, b)); }
template<int imm> inline vcs permutate(const vcs& a) { return vcs(_mm_shuffle_epi32(a, imm)); }
template<int imm> inline vcs permutate_high(const vcs& a) { return vcs(_mm_shufflehi_epi16(a, imm)); }
template<int imm> inline vcs permutate_low(const vcs& a) { return vcs(_mm_shufflelo_epi16(a, imm)); }
inline vcs conj(const vcs& a) { return xor(a, vector128_consts::__0xFFFF0000FFFF0000FFFF0000FFFF0000<vcs>()); }
inline vcs conjre(const vcs& a) { return sign(a, vcs(_mm_set1_epi32(0x00018000))); }
inline vcs flip(const vcs& a) { vcs b = permutate_low<0xb1>(a); return permutate_high<0xb1>(b); }
inline vcs mul_j(const vcs& a) { return xor(flip(a), vector128_consts::__0x0000FFFF0000FFFF0000FFFF0000FFFF<vcs>()); }
inline vi pairwise_muladd(const vs& a, const vs& b) { __m128i r = _mm_madd_epi16(a, b); sbref::tap_madd(r); return vi(r); }
inline vs pack(const vi& a, const vi& b) {
    sbref::tap_pack(a); sbref::tap_pack(b);
    const __m128i m = vector128_consts::__0x0000FFFF0000FFFF0000FFFF0000FFFF<vi>();
    return vs(_mm_or_si128(_mm_and_si128(a, m), _mm_slli_epi32(_mm_and_si128(b, m), 16)));
}
inline vcs conj_mul_shift(const vcs& a, const vcs& b, int nbits_right) {
    vcs vcs1 = conjre(a);
    vcs1 = flip(vcs1);
    vi vi0 = pairwise_muladd((vs&)a, (vs&)b);
    vi vi1 = pairwise_muladd((vs&)vcs1, (vs&)b);
    vi0 = shift_right(vi0, nbits_right);
    vi1 = shift_right(vi1, nbits_right);
    return (vcs)pack(vi0, vi1);
}
inline vcs mul_shift(const vcs& a, const vcs& b, int nbits_right) {
    vi vi0 = pairwise_muladd((vs&)a, (vs)conj(b));
    vi vi1 = pairwise_muladd((vs&)a, (vs)flip(b));
    vi0 = shift_right(vi0, nbits_right);
    vi1 = shift_right(vi1, nbits_right);
    return (vcs)pack(vi0, vi1);
}
SHIM
cat > "$INC/entry.cpp" <<'ENTRY'
#include <stdint.h>
#include "fft_r4dif.h"
#include "ifft_r4dif.h"

namespace sbref {
// [0] saturated_add lanes that clipped, [1] saturated_sub lanes that clipped, [2] pack lanes whose 32-bit value lies outside int16
// (the high bits pack drops were significant), [3] pmaddwd lanes that wrapped (a0 b0 + a1 b1 = 2^31: both products are 2^30)
static thread_local uint64_t counts[4];
static inline unsigned lanes16(__m128i ne) { return (unsigned)__builtin_popcount((unsigned)_mm_movemask_epi8(ne)) / 2; }
static inline unsigned lanes32(__m128i ne) { return (unsigned)__builtin_popcount((unsigned)_mm_movemask_epi8(ne)) / 4; }
void tap_sat(__m128i sat, __m128i wrap, int op) { counts[op] += 8 - lanes16(_mm_cmpeq_epi16(sat, wrap)); }
void tap_pack(__m128i v) { counts[2] += 4 - lanes32(_mm_cmpeq_epi32(v, _mm_srai_epi32(_mm_slli_epi32(v, 16), 16))); }
void tap_madd(__m128i v) { counts[3] += lanes32(_mm_cmpeq_epi32(v, _mm_set1_epi32(INT32_MIN))); }
}

// n vectors of N interleaved int16 complex values, each through the reference's no-side-effect wrapper (FFTSafe / IFFTSafe)
template<int N, bool INV> static void run(size_t n, const int16_t* in, int16_t* out) {
    for (int k = 0; k < 4; k++) sbref::counts[k] = 0;
    vcs x[N / 4], y[N / 4];
    for (size_t i = 0; i < n; i++) {
        memcpy(x, in + 2 * N * i, sizeof x);
        if (INV) IFFTSafe<N>(x, y); else FFTSafe<N>(x, y);
        memcpy(out + 2 * N * i, y, sizeof y);
    }
}

extern "C" {
void ref_fft64(size_t n, const int16_t* in, int16_t* out) { run<64, false>(n, in, out); }
void ref_ifft64(size_t n, const int16_t* in, int16_t* out) { run<64, true>(n, in, out); }
void ref_ifft128(size_t n, const int16_t* in, int16_t* out) { run<128, true>(n, in, out); }
// what the tap counted during the last ref_fft64 / ref_ifft64 / ref_ifft128 call of this thread (see sbref::counts)
void ref_fft_debug(uint64_t out[4]) { for (int k = 0; k < 4; k++) out[k] = sbref::counts[k]; }
}
ENTRY
mkdir -p "$HERE/_ref"
rc=0
${CXX:-g++} -O2 -std=c++17 -mssse3 -msse4.1 -fno-strict-aliasing -fno-operator-names -fpermissive -fPIC -w -shared \
  -I"$INC" -I"$SRC" "$INC/entry.cpp" -o "$HERE/_ref/libfft_ref.so.tmp.$$" || rc=$?
[ $rc -eq 0 ] || { rm -f "$HERE/_ref/libfft_ref.so.tmp.$$"; echo "build_ref_fft: compile failed" >&2; exit 1; }
mv -f "$HERE/_ref/libfft_ref.so.tmp.$$" "$HERE/_ref/libfft_ref.so"
echo "build_ref_fft: oracle/_ref/libfft_ref.so"
