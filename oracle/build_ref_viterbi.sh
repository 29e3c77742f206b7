#!/bin/sh
# oracle/_ref/libviterbi_ref.so: the reference's K=7 Viterbi, compiled from its own headers where they lie: T11aViterbi<...>::Filter
# (kernel/bb/Brick11/src/viterbi.hpp), TViterbiCore and Viterbi_sig11 (viterbicore.h) and the branch-metric / index tables (viterbilut.h).
# Nothing of the Viterbi is restated: the brick's Process loop, the core, the LUTs and the traceback all come from source.
#
# viterbi.hpp and viterbicore.h include headers that pull in the whole Windows kernel build, so they resolve to shims written here instead.
# A quoted #include looks beside the including file first, so the four Brick11/src headers the build needs (viterbi.hpp, viterbicore.h,
# viterbilut.h, ieee80211const.h) are reached through symbolic links in the shim directory, and the shims sit beside them there: they win
# over ieee80211a_cmn.h and ieee80211facade.hpp of Brick11/src.  The links are removed once the library is built.  The shims:
#   vector128.h  vub / vus (kernel/core/inc/vector128.h:96-131, PVECTOR_STRUCT) and the dozen operations viterbicore.h uses, each the
#                intrinsic vector128.h maps it to: add / sub on vub (_mm_add_epi8 / _mm_sub_epi8, :593, :616), and / or, interleave_low /
#                interleave_high on vub (_mm_unpacklo/hi_epi8, :485), smin on vub (_mm_min_epu8, :1297) and on vus (unsigned 16-bit min:
#                _mm_min_epu16 with __SSE4__, else the 0x8000-biased signed min of :421-428, the same function), hmin on vub / vus in the
#                shuffle order of DEFINE_OP_DUPLICATION16 / 8_OPERATION (:387-418), extract<0> on vus (_mm_extract_epi16, :542);
#   const.h      the repo's own sora_b200/brick/brick.hpp (the BRICK macros, TFilter / TSink, pin queues), SELECTANY, A16, FINL;
#   tpltrick.h   empty (viterbi.hpp uses none of it);
#   ieee80211a_cmn.h     ieee80211const.h from Brick11/src (CR_12 / CR_23 / CR_34);
#   ieee80211facade.hpp  CF_11aRxVector with frame_length / code_rate (ieee80211facade.hpp:223-230) and CF_Error with error_code
#                        (kernel/brick/inc/stdfacade.h:9-18), field types as declared there, so CTX_VAR_RO binds the field itself.
# A debug tap counts what Normalize sees: viterbicore.h applies `sub` to a vub only to normalise (TViterbiCore::Normalize :461-464 and the
# two normalisations of Viterbi_sig11), four calls in a row over the 64 states, so the shim's sub records each column it is given.  The
# entry reports the largest unwrapped value of the minimum Normalize subtracts (see ref_viterbi_debug below).
# Nothing of the reference is copied into the repository.  TEST INFRASTRUCTURE ONLY.
#   usage: oracle/build_ref_viterbi.sh [reference root, default /root/reference]
set -e
REF="${1:-/root/reference}"
SRC="$REF/kernel/bb/Brick11/src"
HERE="$(cd "$(dirname "$0")" && pwd)"
[ -f "$SRC/viterbi.hpp" ] || { echo "build_ref_viterbi: $SRC/viterbi.hpp not found (fine outside the build container: the prebuilt oracle/_ref is used)"; exit 0; }
INC="$HERE/_ref/viterbi_inc"
rm -rf "$INC"; mkdir -p "$INC"
: > "$INC/tpltrick.h"
cat > "$INC/const.h" <<'SHIM'
#pragma once
#include "brick.hpp"
#define __int8 char
#define __int16 short
#define __int64 long long
#define __forceinline inline __attribute__((always_inline))
#define __declspec(x)
#define SELECTANY
#define A16 __attribute__((aligned(16)))
#define E_ERROR_SUCCESS 0x00000000
SHIM
cat > "$INC/vector128.h" <<'SHIM'
#pragma once
#include <smmintrin.h>
#include "const.h"
#define SB_VEC(NAME, TDATA)                                                                                     \
struct NAME {                                                                                                   \
    static const size_t size = 16 / sizeof(TDATA);                                                              \
    typedef TDATA data_type[size] __attribute__((aligned(16)));                                                 \
    typedef TDATA elem_type;                                                                                    \
    NAME() {}                                                                                                   \
    explicit NAME(__m128i r) : _raw(r) {}                                                                       \
    template<typename TA> explicit NAME(const TA& a) : _raw((__m128i)a) {}                                      \
    NAME(const data_type& pa) : _raw(_mm_loadu_si128((const __m128i*)pa)) {}                                    \
    NAME& operator=(const data_type& pa) { _raw = _mm_loadu_si128((const __m128i*)pa); return *this; }          \
    operator __m128i() const { return _raw; }                                                                   \
    __m128i _raw;                                                                                               \
};
SB_VEC(vub, unsigned char)
SB_VEC(vus, unsigned short)
namespace sbref { void tap_normalize(const vub& column); }
inline vub add(const vub& a, const vub& b) { return vub(_mm_add_epi8(a, b)); }
inline vub sub(const vub& a, const vub& b) { sbref::tap_normalize(a); return vub(_mm_sub_epi8(a, b)); }
inline vub and(const vub& a, const vub& b) { return vub(_mm_and_si128(a, b)); }
inline vub or(const vub& a, const vub& b) { return vub(_mm_or_si128(a, b)); }
inline vub interleave_low(const vub& a, const vub& b) { return vub(_mm_unpacklo_epi8(a, b)); }
inline vub interleave_high(const vub& a, const vub& b) { return vub(_mm_unpackhi_epi8(a, b)); }
inline vub smin(const vub& a, const vub& b) { return vub(_mm_min_epu8(a, b)); }
inline vus smin(const vus& a, const vus& b) { return vus(_mm_min_epu16(a, b)); }
inline vub hmin(const vub& a) {
    __m128i x1 = a, x0 = _mm_shuffle_epi32(x1, 0x4E);
    x0 = _mm_min_epu8(x0, x1); x1 = _mm_shuffle_epi32(x0, 0xB1); x0 = _mm_min_epu8(x0, x1);
    x0 = _mm_unpacklo_epi8(x0, x0); x0 = _mm_unpacklo_epi8(x0, x0);
    x1 = _mm_shuffle_epi32(x0, 0x4E); x0 = _mm_min_epu8(x0, x1); x1 = _mm_shuffle_epi32(x0, 0xB1); x0 = _mm_min_epu8(x0, x1);
    return vub(x0);
}
inline vus hmin(const vus& a) {
    __m128i r0 = a, r1 = _mm_shuffle_epi32(r0, 0x4E), r2 = _mm_min_epu16(r0, r1);
    r1 = _mm_shuffle_epi32(r2, 0xB1); r2 = _mm_min_epu16(r2, r1);
    r1 = _mm_shufflelo_epi16(r2, 0xB1); r1 = _mm_shuffle_epi32(r1, _MM_SHUFFLE(0, 1, 0, 1)); r2 = _mm_min_epu16(r2, r1);
    return vus(r2);
}
template<int index> inline unsigned short extract(const vus& a) { return (unsigned short)_mm_extract_epi16(a, index); }
SHIM
cat > "$INC/ieee80211a_cmn.h" <<'SHIM'
#pragma once
#include "const.h"
#include "ieee80211const.h"
SHIM
cat > "$INC/ieee80211facade.hpp" <<'SHIM'
#pragma once
#include "const.h"
class CF_11aRxVector { FACADE_FIELD(ushort, frame_length); FACADE_FIELD(ushort, code_rate); };
class CF_Error { FACADE_FIELD(ulong, error_code); public: CF_Error() { error_code() = E_ERROR_SUCCESS; } };
SHIM
cat > "$INC/entry.cpp" <<'ENTRY'
#include <vector>
#include "viterbi.hpp"

namespace sbref {
// Debug tap on Normalize.  The 64 path metrics it normalises are uint8 and wrap; a column is unwrapped by placing the start of the
// window after the largest circular gap between its values (the survivors span far less than 128: every state is six steps from the
// best one), and by the window starting below 256 (the best path metric grows by at most 29 per rate-3/4 puncture group, 8 groups
// between two normalisations: < 256).  max_min: the largest unwrapped value of the minimum Normalize subtracts (> 255: the minimum it
// took was a wrapped metric); max_any: the largest unwrapped metric of any state at a normalisation (> 255: metrics wrapped).
static thread_local unsigned ncol, max_min, max_any;
static thread_local unsigned char col[64];
void tap_normalize(const vub& column) {
    _mm_storeu_si128((__m128i*)(col + 16 * ncol), column);
    if (++ncol < 4) return;
    ncol = 0;
    bool seen[256] = {};
    for (int s = 0; s < 64; s++) seen[col[s]] = true;
    unsigned v[64], k = 0;
    for (unsigned x = 0; x < 256; x++) if (seen[x]) v[k++] = x;
    unsigned mn = v[0], start = v[0], best_gap = v[0] + 256 - v[k - 1];
    for (unsigned i = 1; i < k; i++) if (v[i] - v[i - 1] > best_gap) { best_gap = v[i] - v[i - 1]; start = v[i]; }
    unsigned span = 0;
    for (int s = 0; s < 64; s++) { unsigned d = (col[s] - start) & 255; if (d > span) span = d; }
    unsigned true_min = start + ((mn - start) & 255);
    if (true_min > max_min) max_min = true_min;
    if (start + span > max_any) max_any = start + span;
}
}

template<class T_CTX> class ByteSink : public TSink<T_CTX> {
public:
    DEFINE_IPORT(uchar, 1);
    std::vector<unsigned char> bytes;
    explicit ByteSink(T_CTX& ctx) : TSink<T_CTX>(ctx) {}
    BOOL_FUNC_PROCESS(ipin) { while (ipin.check_read()) { bytes.push_back(*ipin.peek()); ipin.pop(); } return true; }
};

typedef LOCAL_CONTEXT(T11aViterbi) Ctx;

// The brick from a fresh context, driven with nsoft / N_INPUT bursts; returns the bytes it emitted, or (size_t)-1 when the input would
// run the trellis past TRELLIS_MAX columns (the reference's trellis array does not wrap).
template<size_t TM, size_t NI, size_t D, size_t LA>
static size_t run(const unsigned char* soft, size_t nsoft, int code_rate, unsigned frame_len, unsigned char* out) {
    typedef typename T11aViterbi<TM, NI, D, LA>::template Filter<Ctx, ByteSink<Ctx>> F;
    const size_t per = code_rate == CR_12 ? 2 : code_rate == CR_34 ? 4 : 3, steps = code_rate == CR_12 ? 1 : code_rate == CR_34 ? 3 : 2;
    if (nsoft % NI || nsoft / per * steps >= TM) return (size_t)-1;
    Ctx ctx; ctx.frame_length() = (ushort)frame_len; ctx.code_rate() = (ushort)code_rate; ctx.error_code() = E_ERROR_SUCCESS;
    ByteSink<Ctx>* sink = new ByteSink<Ctx>(ctx);
    // the flush can trace back more bits than m_outbuf[TRELLIS_DEPTH / 8 + 1] holds (up to TRELLIS_DEPTH + TRELLIS_LOOKAHEAD + 24):
    // the brick is placed in a buffer with room behind it, so that the bytes it writes there stay its own
    std::vector<unsigned char> mem(sizeof(F) + 4096 + alignof(F));
    F* f = new ((void*)(((uintptr_t)mem.data() + alignof(F) - 1) / alignof(F) * alignof(F))) F(ctx, sink);
    TPinQueue<uchar, NI, NI>* q = new TPinQueue<uchar, NI, NI>();
    for (size_t i = 0; i < nsoft; i += NI) { memcpy(q->append(), soft + i, NI); f->Process(*q); }
    size_t n = sink->bytes.size();
    memcpy(out, sink->bytes.data(), n);
    delete q; f->~F();
    return n;
}

extern "C" {
// Viterbi_sig11 (viterbicore.h:36) with the >> 6 of T11aViterbiSig (viterbi.hpp:38-39).
unsigned ref_viterbi_sig11(const unsigned char soft[48]) {
    vub trellis[64 / 16 * 48];
    unsigned output = 0;
    Viterbi_sig11(trellis, (const char*)soft, (char*)&output);
    return output >> 6;
}
// inst 0: <5000*8, 48, 256, 24> (802.11a); 1: <5000*8, 312, 192, 36> (802.11n); 2: <5000*8, 48, 24> (the short window).
size_t ref_viterbi_block(int inst, const unsigned char* soft, size_t nsoft, int code_rate, unsigned frame_len, unsigned char* out) {
    sbref::ncol = sbref::max_min = sbref::max_any = 0;
    switch (inst) {
    case 0: return run<5000 * 8, 48, 256, 24>(soft, nsoft, code_rate, frame_len, out);
    case 1: return run<5000 * 8, 312, 192, 36>(soft, nsoft, code_rate, frame_len, out);
    case 2: return run<5000 * 8, 48, 24, 24>(soft, nsoft, code_rate, frame_len, out);
    }
    return (size_t)-1;
}
// what the tap saw during the last ref_viterbi_block call of this thread: [0] max_min, [1] max_any
void ref_viterbi_debug(unsigned out[2]) { out[0] = sbref::max_min; out[1] = sbref::max_any; }
}
ENTRY
for h in viterbi.hpp viterbicore.h viterbilut.h ieee80211const.h; do ln -s "$SRC/$h" "$INC/$h"; done
mkdir -p "$HERE/_ref"
rc=0
${CXX:-g++} -O2 -std=c++17 -msse4.1 -fno-strict-aliasing -fno-operator-names -fpermissive -fPIC -w -shared \
  -I"$HERE/../sora_b200/brick" "$INC/entry.cpp" -o "$HERE/_ref/libviterbi_ref.so.tmp.$$" || rc=$?
for h in viterbi.hpp viterbicore.h viterbilut.h ieee80211const.h; do rm -f "$INC/$h"; done
[ $rc -eq 0 ] || { rm -f "$HERE/_ref/libviterbi_ref.so.tmp.$$"; echo "build_ref_viterbi: compile failed" >&2; exit 1; }
mv -f "$HERE/_ref/libviterbi_ref.so.tmp.$$" "$HERE/_ref/libviterbi_ref.so"
echo "build_ref_viterbi: oracle/_ref/libviterbi_ref.so"
