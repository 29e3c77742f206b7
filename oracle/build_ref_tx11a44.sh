#!/bin/sh
# oracle/_ref/libupsample44_ref.so: the reference's 40 -> 44 Msps upsampler (Upsample40MTo44M_160 / _3, kernel/bb/dot11a/inc/bb/mod/upsample.h),
# compiled from its own header where it lies.  upsample.h includes "complex.h" and "vector128.h"; neither lies next to it, so both resolve
# to a shim written here that defines only what the header uses: COMPLEX16, vs / vcs with their data_type, mul_shift<15> (pmulhrsw),
# concat_extract (palignr), permutate<a0,a1,a2,a3> on vcs (pshufd), add (paddw), and / or, set_zero and store (movdqu), as
# kernel/core/inc/vector128.h defines them (lines 552, 603, 688, 1252, 1362).  `and` / `or` are function names there, so the header is compiled
# with -fno-operator-names.  The entry drives Upsample40MTo44M_160 on a cSymbol[160] immediately followed by cSymbol44M[177], as
# BB11A_TX_VECTOR lays them out (kernel/inc/bb/bba.h:161-165), so the one-vector over-read at the end of the input is exercised for real.
# Nothing of the reference is copied into the repository.  TEST INFRASTRUCTURE ONLY.
#   usage: oracle/build_ref_tx11a44.sh [reference root, default /root/reference]
set -e
REF="${1:-/root/reference}"
HDR="$REF/kernel/bb/dot11a/inc/bb/mod/upsample.h"
HERE="$(cd "$(dirname "$0")" && pwd)"
[ -f "$HDR" ] || { echo "build_ref_tx11a44: $HDR not found (fine outside the build container: the prebuilt oracle/_ref is used)"; exit 0; }
INC="$HERE/_ref/tx11a44_inc"
rm -rf "$INC"; mkdir -p "$INC"
: > "$INC/complex.h"
cat > "$INC/vector128.h" <<'SHIM'
#pragma once
#include <immintrin.h>
#define __declspec(x)
#define __int16 short
#define DSP_INLINE inline
struct COMPLEX16 { short re, im; };
struct vs {
    typedef short data_type[8] __attribute__((aligned(16)));
    __m128i v;
    vs() {}
    vs(__m128i x) : v(x) {}
    explicit vs(const short* p) : v(_mm_loadu_si128((const __m128i*)p)) {}
};
struct vcs {
    typedef short data_type[8] __attribute__((aligned(16)));
    __m128i v;
    vcs() {}
    vcs(__m128i x) : v(x) {}
    vcs(const vs& x) : v(x.v) {}
    explicit vcs(const short* p) : v(_mm_loadu_si128((const __m128i*)p)) {}
    COMPLEX16& operator[](int i) { return ((COMPLEX16*)&v)[i]; }
    const COMPLEX16& operator[](int i) const { return ((const COMPLEX16*)&v)[i]; }
};
template<int n> inline vs mul_shift(const vs& a, const vs& b);
template<> inline vs mul_shift<15>(const vs& a, const vs& b) { return vs(_mm_mulhrs_epi16(a.v, b.v)); }
template<int nbytes, typename T> inline T concat_extract(const T& a, const T& b) { return T(_mm_alignr_epi8(a.v, b.v, nbytes)); }
template<int a0, int a1, int a2, int a3> inline vcs permutate(const vcs& a) { return vcs(_mm_shuffle_epi32(a.v, _MM_SHUFFLE(a3, a2, a1, a0))); }
inline vcs add(const vcs& a, const vcs& b) { return vcs(_mm_add_epi16(a.v, b.v)); }
inline vcs and(const vcs& a, const vcs& b) { return vcs(_mm_and_si128(a.v, b.v)); }
inline vcs or(const vcs& a, const vcs& b) { return vcs(_mm_or_si128(a.v, b.v)); }
inline void set_zero(vcs& a) { a.v = _mm_setzero_si128(); }
inline void store(void* p, const vcs& a) { _mm_storeu_si128((__m128i*)p, a.v); }
SHIM
cat > "$INC/entry.cpp" <<'ENTRY'
#include "vector128.h"
#include UPSAMPLE_H
#include <stddef.h>
#include <string.h>
struct TxBuffers { alignas(16) COMPLEX16 cSymbol[160]; alignas(16) COMPLEX16 cSymbol44M[176 + 1]; };
static_assert(offsetof(TxBuffers, cSymbol44M) == 160 * sizeof(COMPLEX16), "cSymbol44M must follow cSymbol");
/* in_place != 0: the input lies in cSymbol, the output goes to cSymbol44M right behind it (what UpsampleAndCopyNT does for SIGNAL and data);
   otherwise the input is followed by the four samples `behind` (the preamble chunks) */
extern "C" void ref_upsample44_160(const short* in160, const short* behind4, int in_place, short* out176) {
    TxBuffers t; memset(&t, 0, sizeof t);
    alignas(16) COMPLEX16 buf[164], o[176];
    if (in_place) { memcpy(t.cSymbol, in160, sizeof t.cSymbol); Upsample40MTo44M_160(t.cSymbol, t.cSymbol44M); memcpy(out176, t.cSymbol44M, 176 * sizeof(COMPLEX16)); }
    else { memcpy(buf, in160, 160 * sizeof(COMPLEX16)); memcpy(buf + 160, behind4, 4 * sizeof(COMPLEX16)); Upsample40MTo44M_160(buf, o); memcpy(out176, o, sizeof o); }
}
extern "C" void ref_upsample44_3(const short* in4, short* out4) {
    alignas(16) COMPLEX16 i[4], o[4]; memcpy(i, in4, sizeof i); Upsample40MTo44M_3(i, o); memcpy(out4, o, sizeof o);
}
ENTRY
mkdir -p "$HERE/_ref"
${CXX:-g++} -O1 -fno-strict-aliasing -mssse3 -fno-operator-names -fPIC -w -shared -I"$INC" -DUPSAMPLE_H="\"$HDR\"" "$INC/entry.cpp" \
  -o "$HERE/_ref/libupsample44_ref.so.tmp.$$" && mv -f "$HERE/_ref/libupsample44_ref.so.tmp.$$" "$HERE/_ref/libupsample44_ref.so"
echo "build_ref_tx11a44: oracle/_ref/libupsample44_ref.so"
