#!/bin/sh
# The reference spectrum analyser's meters and the transform under them, compiled from the reference's own headers where they lie:
#   oracle/_ref/libmeter_ref.so  TSpecMeter<N> for every N = 4 .. 32768 and TPowerMeter<N> for N = 1, 3, 4, 5, 128, 840, 4096, 65536
#                                (kernel/sdl/inc/sdlmeasure.hpp), each driven through Process on N-sample bursts into a sink that keeps
#                                what it is handed.  The framework headers are oracle/ref_shim.sh's; sdlplot.hpp is an empty shim with
#                                the named_plotter base and MAX_NAME_LEN that the uninstantiated TInspectTube names.
#   oracle/_ref/libfftn_ref.so   FFT<N> (kernel/core/inc/fft_r4dif.h, through FFTSafe) for every N = 4 .. 32768, with the twiddle tables
#                                FFT_GetTwiddleConst<N, M> and the read-out FFTLUTMapTable<N>.  It is compiled against the vector128.h shim
#                                that oracle/build_ref_fft.sh writes (run first), whose debug tap counts, per call, the lanes where
#                                saturated_add / saturated_sub clipped, where pack dropped significant bits and where pmaddwd wrapped.
# Two libraries, because the two shims define the same vector operations differently (the tap).  Nothing of the reference is copied into
# the repository.  TEST INFRASTRUCTURE ONLY.
#   usage: oracle/build_ref_meter.sh [reference root, default /root/reference]
set -e
REF="${1:-/root/reference}"
SDL="$REF/kernel/sdl/inc"
CORE="$REF/kernel/core/inc"
HERE="$(cd "$(dirname "$0")" && pwd)"
[ -f "$SDL/sdlmeasure.hpp" ] || { echo "build_ref_meter: $SDL/sdlmeasure.hpp not found (fine outside the build container: the prebuilt oracle/_ref is used)"; exit 0; }
"$HERE/build_ref_fft.sh" "$REF" >/dev/null
INC="$HERE/_ref/meter_inc"
rm -rf "$INC"
. "$HERE/ref_shim.sh"
ref_shim "$INC"
cat > "$INC/sdlplot.hpp" <<'SHIM'
#pragma once
#define MAX_NAME_LEN 64
struct named_plotter { const char* GetName() const { return ""; } };
SHIM
cat > "$INC/entry.cpp" <<'ENTRY'
#include <stdint.h>
#include <string.h>
#include <vector>
#include "const.h"
#include "vector128.h"
namespace sbref { int phase; void tap_pack(__m128i, int) {} void tap_zero(__m128i) {} void tap_clamp(__m128i, __m128i) {} void tap_madd(__m128i) {}
                  void tap_spack(__m128i, __m128i) {} }
#include "sdlmeasure.hpp"

struct Ctx : CF_VOID {};
// a sink that keeps every burst of B ints it is handed
template<size_t B> class KeepInts : public TSink<Ctx> {
public:
    DEFINE_IPORT(int, B);
    std::vector<int> got;
    explicit KeepInts(Ctx& ctx) : TSink<Ctx>(ctx) {}
    BOOL_FUNC_PROCESS(ipin) { while (ipin.check_read()) { got.insert(got.end(), ipin.peek(), ipin.peek() + B); ipin.pop(); } return true; }
};

// `Meter` fed n bursts of N samples (in + 2 N i int16), one Process per burst; the sink's ints into out (B per burst)
template<template<class, class> class Meter, size_t N, size_t B> static void run(size_t n, const int16_t* in, int32_t* out) {
    Ctx* ctx = new Ctx;
    KeepInts<B>* s = new KeepInts<B>(*ctx);
    Meter<Ctx, KeepInts<B> >* m = new Meter<Ctx, KeepInts<B> >(*ctx, s);
    TPinQueue<COMPLEX16, N, N>* q = new TPinQueue<COMPLEX16, N, N>();
    for (size_t i = 0; i < n; i++) { memcpy(q->append(), in + 2 * N * i, N * sizeof(COMPLEX16)); m->Process(*q); }
    memcpy(out, s->got.data(), s->got.size() * sizeof(int));
    delete q; delete m; delete ctx;
}
template<size_t N> struct Spec { template<class C, class X> using F = typename TSpecMeter<N>::template Filter<C, X>; };
template<size_t N> struct Pwr { template<class C, class X> using F = typename TPowerMeter<N>::template Filter<C, X>; };

extern "C" {
// TSpecMeter<N> on n frames of N samples: N ints per frame.  Returns 0, or -1 for an N not built.
int ref_spec_meter(uint32_t N, size_t n, const int16_t* in, int32_t* out) {
    switch (N) {
#define SB_SPEC(K) case K: run<Spec<K>::template F, K, K>(n, in, out); return 0;
        SB_SPEC(4) SB_SPEC(8) SB_SPEC(16) SB_SPEC(32) SB_SPEC(64) SB_SPEC(128) SB_SPEC(256) SB_SPEC(512) SB_SPEC(1024) SB_SPEC(2048) SB_SPEC(4096)
        SB_SPEC(8192) SB_SPEC(16384) SB_SPEC(32768)
    }
    return -1;
}
// TPowerMeter<N> on n blocks of N samples: one int per block.  Returns 0, or -1 for an N not built.
int ref_power_meter(uint32_t N, size_t n, const int16_t* in, int32_t* out) {
    switch (N) {
#define SB_PWR(K) case K: run<Pwr<K>::template F, K, 1>(n, in, out); return 0;
        SB_PWR(1) SB_PWR(3) SB_PWR(4) SB_PWR(5) SB_PWR(128) SB_PWR(840) SB_PWR(4096) SB_PWR(65536)
    }
    return -1;
}
}
ENTRY
cat > "$INC/fftn.cpp" <<'ENTRY'
#include <stdint.h>
#include <vector>
#include "fft_r4dif.h"

namespace sbref {
// [0] saturated_add lanes that clipped, [1] saturated_sub lanes that clipped, [2] pack lanes whose 32-bit value lies outside int16,
// [3] pmaddwd lanes that wrapped: the same tap as oracle/build_ref_fft.sh's libfft_ref.so
static thread_local uint64_t counts[4];
static inline unsigned lanes16(__m128i ne) { return (unsigned)__builtin_popcount((unsigned)_mm_movemask_epi8(ne)) / 2; }
static inline unsigned lanes32(__m128i ne) { return (unsigned)__builtin_popcount((unsigned)_mm_movemask_epi8(ne)) / 4; }
void tap_sat(__m128i sat, __m128i wrap, int op) { counts[op] += 8 - lanes16(_mm_cmpeq_epi16(sat, wrap)); }
void tap_pack(__m128i v) { counts[2] += 4 - lanes32(_mm_cmpeq_epi32(v, _mm_srai_epi32(_mm_slli_epi32(v, 16), 16))); }
void tap_madd(__m128i v) { counts[3] += lanes32(_mm_cmpeq_epi32(v, _mm_set1_epi32(INT32_MIN))); }
}

// n vectors of N interleaved int16 complex values through FFTSafe<N>
template<int N> static void run(size_t n, const int16_t* in, int16_t* out) {
    for (int k = 0; k < 4; k++) sbref::counts[k] = 0;
    std::vector<vcs> x(N / 4), y(N / 4);
    for (size_t i = 0; i < n; i++) {
        memcpy(x.data(), in + 2 * (size_t)N * i, N * 4);
        FFTSafe<N>(x.data(), y.data());
        memcpy(out + 2 * (size_t)N * i, y.data(), N * 4);
    }
}
template<int N> static void tables(int16_t* tw, int16_t* map) {
    if (N >= 8) {
        const int rows = N == 8 ? 1 : 3;             // FFT_GetTwiddleConst<8, 1> is the only table of N = 8 (FFTSSEEx<8>'s wFFTLUT8)
        for (int m = 0; m < rows; m++) {
            const vcs* t = m == 0 ? FFT_GetTwiddleConst<N, 1>() : m == 1 ? FFT_GetTwiddleConst<N == 8 ? 16 : N, 2>() : FFT_GetTwiddleConst<N == 8 ? 16 : N, 3>();
            memcpy(tw + 2 * (N / 4) * m, t, N == 8 ? 16 : N);   // N / 4 entries of 4 bytes (wFFTLUT8: 4)
        }
    }
    for (int i = 0; i < N; i++) map[i] = FFTLUTMapTable<N>(i);
}

extern "C" {
// FFT<N> on n vectors of N samples.  Returns 0, or -1 for an N not built.
int ref_fftn(uint32_t N, size_t n, const int16_t* in, int16_t* out) {
    switch (N) {
#define SB_FFT(K) case K: run<K>(n, in, out); return 0;
        SB_FFT(4) SB_FFT(8) SB_FFT(16) SB_FFT(32) SB_FFT(64) SB_FFT(128) SB_FFT(256) SB_FFT(512) SB_FFT(1024) SB_FFT(2048) SB_FFT(4096)
        SB_FFT(8192) SB_FFT(16384) SB_FFT(32768)
    }
    return -1;
}
// what the tap counted during the last ref_fftn call of this thread (see sbref::counts)
void ref_fftn_debug(uint64_t out[4]) { for (int k = 0; k < 4; k++) out[k] = sbref::counts[k]; }
// the tables of FFT<N>: tw = FFT_GetTwiddleConst<N, M>() for M = 1, 2, 3 (N / 4 complex each; N = 8: M = 1 only), map = FFTLUTMapTable<N>
int ref_fftn_tables(uint32_t N, int16_t* tw, int16_t* map) {
    switch (N) {
#define SB_TAB(K) case K: tables<K>(tw, map); return 0;
        SB_TAB(4) SB_TAB(8) SB_TAB(16) SB_TAB(32) SB_TAB(64) SB_TAB(128) SB_TAB(256) SB_TAB(512) SB_TAB(1024) SB_TAB(2048) SB_TAB(4096)
        SB_TAB(8192) SB_TAB(16384) SB_TAB(32768)
    }
    return -1;
}
}
ENTRY
mkdir -p "$HERE/_ref"
rc=0
${CXX:-g++} -O1 -std=c++17 -fwrapv -mssse3 -msse4.1 -fno-strict-aliasing -fno-operator-names -fpermissive -fPIC -shared -w \
  -include functional -include memory -I"$INC" -I"$SDL" -I"$REF/kernel/brick/inc" -I"$CORE" -I"$HERE/../sora_b200/brick" "$INC/entry.cpp" -o "$HERE/_ref/libmeter_ref.so.tmp.$$" || rc=$?
[ $rc -eq 0 ] || { rm -f "$HERE/_ref/libmeter_ref.so.tmp.$$"; echo "build_ref_meter: libmeter_ref.so compile failed" >&2; exit 1; }
${CXX:-g++} -O1 -std=c++17 -mssse3 -msse4.1 -fno-strict-aliasing -fno-operator-names -fpermissive -fPIC -shared -w \
  -I"$HERE/_ref/fft_inc" -I"$CORE" "$INC/fftn.cpp" -o "$HERE/_ref/libfftn_ref.so.tmp.$$" || rc=$?
[ $rc -eq 0 ] || { rm -f "$HERE/_ref/libmeter_ref.so.tmp.$$" "$HERE/_ref/libfftn_ref.so.tmp.$$"; echo "build_ref_meter: libfftn_ref.so compile failed" >&2; exit 1; }
mv -f "$HERE/_ref/libmeter_ref.so.tmp.$$" "$HERE/_ref/libmeter_ref.so"
mv -f "$HERE/_ref/libfftn_ref.so.tmp.$$" "$HERE/_ref/libfftn_ref.so"
echo "build_ref_meter: oracle/_ref/libmeter_ref.so, oracle/_ref/libfftn_ref.so"
