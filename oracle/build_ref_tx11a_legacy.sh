#!/bin/sh
# oracle/_ref/libtx11a_legacy_ref.so: the reference's legacy 802.11a transmitter, BB11ATxFrameMod and BB11AModulateACK (kernel/bb/dot11a/dot11/
# atx_fe.c, atx_6.c .. atx_54.c with atx_9.c's own symbol-pair encoder, through atx_tpl_imp.h, atx_tpl.h and atx.h), compiled from its own
# source where it lies, with the inc/bb/mod/ headers those files use (ofdmsymbol.h, convenc.h, ainterleave.h, amap.h, addpilot.h, copynt.h,
# ifft64x.h, upsample.h), IFFTSSEEx<128> of kernel/core/inc/ifft_r4dif.h, and the lutst/ tables as data (scramble_11a.c, conv_encoder_*.c,
# interleave_*.c, mapa_*.c, pilotsgn.c, preamble40_11a.c).  Nothing of the transmitter is restated.
#
# A shim directory, first on the include path, stands for the framework headers, which only MSVC / the WDK compile.  It defines only what
# these files use:
#   vector128.h   vs / vi / vcs / vb with their data_type (vector128.h:96-138) and each operation as the intrinsic vector128.h maps it to:
#                 shift_right on vs / vcs (_mm_srai_epi16, :832) and vi (_mm_srai_epi32, :830), shift_left on vcs (_mm_slli_epi16, :818),
#                 saturated_add / saturated_sub on vcs (_mm_adds_epi16 / _mm_subs_epi16, :645, :655), add on vcs (_mm_add_epi16, :603),
#                 and / or / xor (_mm_and_si128 / _mm_or_si128 / _mm_xor_si128, :567), sign (_mm_sign_epi16, :535), permutate<imm> and
#                 permutate<a0, a1, a2, a3> (_mm_shuffle_epi32, :338-341, :688), permutate_high / permutate_low (_mm_shufflehi/lo_epi16, :683,
#                 :677), concat_extract<n> (_mm_alignr_epi8, :552), mul_shift<15> on vs (_mm_mulhrs_epi16, :1250-1255), saturated_pack(vs, vs)
#                 (_mm_packs_epi16, :870), store (_mm_storeu_si128, :1362), store_nt (_mm_stream_si128, :1355), set_zero (:439), and the
#                 complex helpers and vector128_consts masks the IFFT names, as oracle/build_ref_fft.sh gives them;
#   soratypes.h   the Windows integer names, COMPLEX8 / COMPLEX16, __forceinline, A16, ASSERT, KdPrint, and the spin locks as no-ops;
#   bb/bba.h      the constants and BB11A_TX_VECTOR cut from kernel/inc/bb/bba.h with sed (the reference's member order and alignment, so that
#                 cSymbol[160] is immediately followed by cSymbol44M[177] and Upsample40MTo44M_160's over-read is real), the DOT11A_RATE_*
#                 codes, dot11_pkt.h (MAC_ADDRESS, DOT11_MAC_ACK_FRAME, INPUT_MAX) from where it lies, RCB_BUFFER_ALIGN* and
#                 ALIGN_WITH_RCB_BUFFER_PADDING_ZERO cut from kernel/core/inc/_tx_manager2.h, and MDL / PACKET_BASE / the TX descriptor with
#                 SoraPacketGetTxSampleBuffer / SoraPacketSetSignalLength over them;
#   bb/mod.h      ofdmsymbol.h only (the receive headers mod.h also lists are not used) and BITS_PER_BYTE_SHIFT (mod/viterbi.h:3);
#   CRC32.h       gc_CRC32LUT and CalcCRC32 cut from kernel/core/inc/CRC32.h with sed (ULONG 32 bits, as under MSVC);
#   complex.h     empty (COMPLEX16 comes with soratypes.h).
# BBRAND is RtlRandomEx (atx.h:5-9), a deterministic LCG here; the scrambler ignores it anyway (atx_tpl.h:19, bReg = 0xFF).
#
# The preamble over-read: at 44 Msps, CopyPreamble16_NT's fourth chunk makes Upsample40MTo44M_160 load one vector past PREAMBLE40_11A_LUT.
# The transmitter files are compiled with PREAMBLE40_11A_LUT renamed to a buffer that holds the compiled table followed by 8 samples the
# caller sets (ref_tx11a_legacy_set_pad; zeros by default, which is what the device library reads there, DESIGN.md §1).
#
# A debug tap counts lanes (ref_tx11a_legacy_debug, cumulative until ref_tx11a_legacy_debug_reset):
#   [0] Window's saturated_add clipped (the saturated_add that follows IFFT64x's shift_left: IFFTSSEEx's own run before that shift)
#   [1] Window's plain += of last[0] wrapped (ofdmsymbol.h:37-38; judged at that saturated_add from the same operands)
#   [2] saturated_pack in Copy_NT clipped (the shifted 16-bit value lies outside int8)
#   [3] shift_left(.., 2) in IFFT64x lost significant bits
#   [4] IFFTSSEEx<128>'s own saturated_add / saturated_sub clipped
# Entry points are the ref_* functions; everything else is hidden, so that nothing here interposes on the device library's BB11A* symbols
# when both are loaded in one process.  Nothing of the reference is copied into the repository.  TEST INFRASTRUCTURE ONLY.
#   usage: oracle/build_ref_tx11a_legacy.sh [reference root, default /root/reference]
set -e
REF="${1:-/root/reference}"
SRC="$REF/kernel/bb/dot11a/dot11"
HERE="$(cd "$(dirname "$0")" && pwd)"
[ -f "$SRC/atx_fe.c" ] || { echo "build_ref_tx11a_legacy: $SRC/atx_fe.c not found (fine outside the build container: the prebuilt oracle/_ref is used)"; exit 0; }
INC="$HERE/_ref/tx11a_legacy_inc"
rm -rf "$INC"; mkdir -p "$INC/bb"
: > "$INC/complex.h"
cat > "$INC/soratypes.h" <<'SHIM'
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include <assert.h>
typedef int32_t HRESULT; typedef unsigned char UCHAR, *PUCHAR, BOOLEAN; typedef unsigned short USHORT; typedef unsigned int UINT;
typedef uint32_t ULONG, *PULONG; typedef void* PVOID; typedef int BOOL; typedef unsigned char KIRQL; typedef int KSPIN_LOCK;
#define IN
#define OUT
#define S_OK 0
#define E_FAIL ((HRESULT)0x80004005L)
#define __int8 char
#define __int16 short
#define __int64 long long
#define __forceinline inline __attribute__((always_inline))
#define A16 __attribute__((aligned(16)))
#define ASSERT(x) assert(x)
#define KdPrint(x)
#define KeAcquireSpinLock(l, irql) ((void)(l), (void)(irql))
#define KeReleaseSpinLock(l, irql) ((void)(l), (void)(irql))
#define RtlZeroMemory(p, n) memset((p), 0, (n))
#define STATIC_LUT
typedef struct _COMPLEX8 { signed char re, im; } COMPLEX8, *PCOMPLEX8, TXSAMPLE, *PTXSAMPLE;
typedef struct _COMPLEX16 { short re, im; } COMPLEX16;
static inline ULONG RtlRandomEx(ULONG* seed) { *seed = *seed * 1103515245u + 12345u; return *seed >> 1; }
SHIM
cat > "$INC/vector128.h" <<'SHIM'
#pragma once
#include <smmintrin.h>
#include "soratypes.h"
#define DSP_INLINE inline __attribute__((always_inline))
#define DSP_INLINE1 inline
#define __declspec(x) SB_DECLSPEC_##x
#define SB_DECLSPEC_selectany __attribute__((weak))
#define SB_DECLSPEC_deprecated
#define SB_DECLSPEC_align(n) __attribute__((aligned(n)))
#define SB_VEC(NAME, TDATA)                                                                                     \
struct NAME {                                                                                                   \
    static const size_t size = 16 / sizeof(TDATA);                                                              \
    typedef TDATA data_type[size] __attribute__((aligned(16)));                                                 \
    NAME() {}                                                                                                   \
    explicit NAME(__m128i r) : _raw(r) {}                                                                       \
    NAME(const data_type& pa) : _raw(*(const __m128i*)pa) {}                                                    \
    template<typename TA> explicit NAME(const TA& a) : _raw((__m128i)a) {}                                      \
    operator __m128i() const { return _raw; }                                                                   \
    TDATA& operator[](int i) { return ((TDATA*)&_raw)[i]; }                                                     \
    const TDATA& operator[](int i) const { return ((const TDATA*)&_raw)[i]; }                                   \
    __m128i _raw;                                                                                               \
};
SB_VEC(vs, short)
SB_VEC(vi, int)
SB_VEC(vcs, COMPLEX16)
SB_VEC(vb, signed char)
namespace sbref { void tap_sat(__m128i sat, __m128i a, __m128i b, __m128i wrap); void tap_spack(__m128i a, __m128i b); void tap_shl(__m128i a, int n); }
class vector128_consts {
public:
    template<typename T> static T __0x0000FFFF0000FFFF0000FFFF0000FFFF() { return (T)_mm_set1_epi32(0x0000FFFF); }
    template<typename T> static T __0xFFFF0000FFFF0000FFFF0000FFFF0000() { return (T)_mm_set1_epi32((int)0xFFFF0000); }
    template<typename T> static T __0xFFFFFFFF00000000FFFFFFFF00000000() { return (T)_mm_set_epi32(-1, 0, -1, 0); }
    template<typename T> static T __0xFFFFFFFFFFFFFFFF0000000000000000() { return (T)_mm_set_epi32(-1, -1, 0, 0); }
    template<typename T> static T __0xFFFF0000FFFF00000000000000000000() { return (T)_mm_set_epi32((int)0xFFFF0000, (int)0xFFFF0000, 0, 0); }
    template<typename T> static T __0xFFFF0000000000000000000000000000() { return (T)_mm_set_epi32((int)0xFFFF0000, 0, 0, 0); }
};
inline vs shift_right(const vs& a, int n) { return vs(_mm_srai_epi16(a, n)); }
inline vcs shift_right(const vcs& a, int n) { return vcs(_mm_srai_epi16(a, n)); }
inline vi shift_right(const vi& a, int n) { return vi(_mm_srai_epi32(a, n)); }
inline vcs shift_left(const vcs& a, int n) { sbref::tap_shl(a, n); return vcs(_mm_slli_epi16(a, n)); }
inline vcs saturated_add(const vcs& a, const vcs& b) { __m128i r = _mm_adds_epi16(a, b); sbref::tap_sat(r, a, b, _mm_add_epi16(a, b)); return vcs(r); }
inline vcs saturated_sub(const vcs& a, const vcs& b) { __m128i r = _mm_subs_epi16(a, b); sbref::tap_sat(r, a, b, _mm_sub_epi16(a, b)); return vcs(r); }
inline vcs add(const vcs& a, const vcs& b) { return vcs(_mm_add_epi16(a, b)); }
inline vcs and(const vcs& a, const vcs& b) { return vcs(_mm_and_si128(a, b)); }
inline vcs or(const vcs& a, const vcs& b) { return vcs(_mm_or_si128(a, b)); }
inline vcs xor(const vcs& a, const vcs& b) { return vcs(_mm_xor_si128(a, b)); }
inline vcs sign(const vcs& a, const vcs& b) { return vcs(_mm_sign_epi16(a, b)); }
template<int imm> inline vcs permutate(const vcs& a) { return vcs(_mm_shuffle_epi32(a, imm)); }
template<int a0, int a1, int a2, int a3> inline vcs permutate(const vcs& a) { return vcs(_mm_shuffle_epi32(a, _MM_SHUFFLE(a3, a2, a1, a0))); }
template<int imm> inline vcs permutate_high(const vcs& a) { return vcs(_mm_shufflehi_epi16(a, imm)); }
template<int imm> inline vcs permutate_low(const vcs& a) { return vcs(_mm_shufflelo_epi16(a, imm)); }
template<int nbytes, typename T> inline T concat_extract(const T& a, const T& b) { return T(_mm_alignr_epi8(a, b, nbytes)); }
template<int nbits_right> inline vs mul_shift(const vs& a, const vs& b);
template<> inline vs mul_shift<15>(const vs& a, const vs& b) { return vs(_mm_mulhrs_epi16(a, b)); }
inline vb saturated_pack(const vs& a, const vs& b) { sbref::tap_spack(a, b); return vb(_mm_packs_epi16(a, b)); }
template<typename T> inline void store(void* p, const T& a) { _mm_storeu_si128((__m128i*)p, a); }
template<typename T> inline void store_nt(T* p, const T& a) { _mm_stream_si128((__m128i*)p, a); }
template<typename T> inline void set_zero(T& a) { a = T(_mm_setzero_si128()); }
inline vcs conj(const vcs& a) { return xor(a, vector128_consts::__0xFFFF0000FFFF0000FFFF0000FFFF0000<vcs>()); }
inline vcs conjre(const vcs& a) { return sign(a, vcs(_mm_set1_epi32(0x00018000))); }
inline vcs flip(const vcs& a) { vcs b = permutate_low<0xb1>(a); return permutate_high<0xb1>(b); }
inline vcs mul_j(const vcs& a) { return xor(flip(a), vector128_consts::__0x0000FFFF0000FFFF0000FFFF0000FFFF<vcs>()); }
inline vi pairwise_muladd(const vs& a, const vs& b) { return vi(_mm_madd_epi16(a, b)); }
inline vs pack(const vi& a, const vi& b) {
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
{
  echo '#pragma once'
  echo '#include "soratypes.h"'
  echo '#include "dot11_pkt.h"'
  tr -d '\r' < "$REF/kernel/inc/bb/bba.h" | sed -n '/^#define CHANNEL_FACTOR_SIZE/,/^#define COMPLEX_PER_OFDM_SYMBOL/p'
  tr -d '\r' < "$REF/kernel/inc/bb/bba.h" | sed -n '/^typedef struct _BB11A_TX_VECTOR/,/^} BB11A_TX_VECTOR/p'
  tr -d '\r' < "$REF/kernel/inc/bb/bba.h" | sed -n '/^#define DOT11A_RATE_/p'
  tr -d '\r' < "$REF/kernel/core/inc/_tx_manager2.h" | sed -n '/^#define RCB_BUFFER_ALIGN_MASK/,/^}$/p'
  cat <<'HDR'
typedef struct _MDL { struct _MDL* Next; void* StartVa; ULONG ByteOffset; ULONG ByteCount; } MDL, *PMDL;
typedef struct { void* pSampleBuffer; ULONG SampleBufferSize; ULONG SignalLength; } SBREF_TX_DESC;
typedef struct { PMDL pMdl; SBREF_TX_DESC* pTxDesc; ULONG PacketSize; ULONG Reserved1; } PACKET_BASE, *PPACKET_BASE;
static inline void SoraPacketGetTxSampleBuffer(PPACKET_BASE p, PTXSAMPLE* b, ULONG* n) { *b = (PTXSAMPLE)p->pTxDesc->pSampleBuffer; *n = p->pTxDesc->SampleBufferSize; }
static inline void SoraPacketSetSignalLength(PPACKET_BASE p, ULONG n) { p->pTxDesc->SignalLength = n; }
HDR
} > "$INC/bb/bba.h"
printf '#pragma once\n#define BITS_PER_BYTE_SHIFT 3\n#include "bb/mod/ofdmsymbol.h"\n' > "$INC/bb/mod.h"
{
  echo '#pragma once'
  echo '#include "soratypes.h"'
  tr -d '\r' < "$REF/kernel/core/inc/CRC32.h" | sed -n '/gc_CRC32LUT\[256\] =/,/^};$/p' \
    | sed 's/^SORA_EXTERN_C SELECTANY extern const unsigned long/static const ULONG/'
  tr -d '\r' < "$REF/kernel/core/inc/CRC32.h" | sed -n '/^CalcCRC32(PUCHAR pByte, ULONG Length)/,/^}$/p' | sed '1s/^/static inline ULONG /'
} > "$INC/CRC32.h"
cat > "$INC/entry.cpp" <<'ENTRY'
#include "bb/bba.h"
#include <emmintrin.h>
#include <stdlib.h>

HRESULT BB11ATxFrameMod(PBB11A_TX_VECTOR info, PPACKET_BASE pPacket);
ULONG BB11AModulateACK(unsigned int SampleRate, const PMAC_ADDRESS RecvMacAddress, PVOID PhyACKBuffer);
// the compiled lutst/preamble40_11a.c table, and the buffer the transmitter files read as PREAMBLE40_11A_LUT: the table, then 8 samples
extern "C" const COMPLEX16 sbref_preamble40_lut[640];
extern "C" { A16 COMPLEX16 sbref_preamble40_read[640 + 8]; }

namespace sbref {
static uint64_t counts[5];
static int after_shl;                                   // IFFT64x's shift_left has run: the next saturated_add is Window's
static inline unsigned lanes16(__m128i ne) { return (unsigned)__builtin_popcount((unsigned)_mm_movemask_epi8(ne)) / 2; }
void tap_sat(__m128i sat, __m128i a, __m128i b, __m128i wrap) {
    const unsigned clipped = 8 - lanes16(_mm_cmpeq_epi16(sat, wrap));
    if (!after_shl) { counts[4] += clipped; return; }
    after_shl = 0; counts[0] += clipped;
    // ofdmsymbol.h:37-38: pcSymbol[0].re += pcLast->re (and .im), plain int16 adds of lanes 0 and 1 of this result and of b
    alignas(16) short r[8], l[8]; _mm_store_si128((__m128i*)r, sat); _mm_store_si128((__m128i*)l, b); (void)a;
    for (int k = 0; k < 2; k++) { const int s = r[k] + l[k]; counts[1] += s > 32767 || s < -32768; }
}
void tap_spack(__m128i a, __m128i b) {
    const __m128i lo = _mm_set1_epi16(-128), hi = _mm_set1_epi16(127);
    const __m128i ab[2] = {a, b};
    for (__m128i v : ab) counts[2] += 8 - lanes16(_mm_cmpeq_epi16(v, _mm_max_epi16(lo, _mm_min_epi16(hi, v))));
}
void tap_shl(__m128i a, int n) {
    counts[3] += 8 - lanes16(_mm_cmpeq_epi16(a, _mm_srai_epi16(_mm_slli_epi16(a, n), n)));
    after_shl = 1;
}
static struct Init { Init() { memcpy(sbref_preamble40_read, sbref_preamble40_lut, sizeof sbref_preamble40_lut); } } init;
}

#define SBREF_API extern "C" __attribute__((visibility("default")))
// a BB11A_TX_VECTOR as BB11ATxContextInit leaves it (a_init.c:62-77: zeros, ulRandSeed 1104), 16-byte aligned
SBREF_API void* ref_tx11a_legacy_ctx_new(void) {
    PBB11A_TX_VECTOR v = (PBB11A_TX_VECTOR)aligned_alloc(16, (sizeof(BB11A_TX_VECTOR) + 15) & ~(size_t)15);
    memset(v, 0, sizeof *v); v->ulRandSeed = 1104; return v;
}
SBREF_API void ref_tx11a_legacy_ctx_free(void* ctx) { free(ctx); }
// BB11ATxFrameMod on the MDL chain (PacketSize = the chain's byte count), FCS = Reserved1, at rate_code (DOT11A_RATE_*) and sample_rate.
// ctx: a context from ref_tx11a_legacy_ctx_new, kept across calls; NULL: a fresh one.  The sample buffer is a 16-byte aligned copy of
// out[0 .. out_bytes) (Copy_NT streams), copied back whole, so bytes the transmitter leaves alone stay as the caller had them.
SBREF_API int ref_tx11a_legacy_frame_mod(void* ctx, unsigned rate_code, unsigned sample_rate, MDL* chain, uint32_t fcs, void* out,
                                         uint32_t out_bytes, uint32_t* signal_length) {
    PBB11A_TX_VECTOR v = (PBB11A_TX_VECTOR)(ctx ? ctx : ref_tx11a_legacy_ctx_new());
    v->SampleRate = sample_rate; v->ti_uiDataRate = rate_code;
    ULONG size = 0; for (MDL* m = chain; m; m = m->Next) size += m->ByteCount;
    void* buf = aligned_alloc(16, (out_bytes + 15) & ~15u); memcpy(buf, out, out_bytes);
    SBREF_TX_DESC d = {buf, out_bytes, 0};
    PACKET_BASE p = {chain, &d, size, fcs};
    const HRESULT hr = BB11ATxFrameMod(v, &p);
    _mm_sfence();
    memcpy(out, buf, out_bytes); free(buf);
    *signal_length = d.SignalLength;
    if (!ctx) free(v);
    return (int)hr;
}
// BB11AModulateACK(sample_rate, ra, out): returns what it returns (the signal length in bytes); out needs 16-byte alignment
SBREF_API uint32_t ref_tx11a_legacy_ack(unsigned sample_rate, const uint8_t* ra, void* out) {
    MAC_ADDRESS a; memcpy(a.Address, ra, 6);
    const ULONG n = BB11AModulateACK(sample_rate, &a, out);
    _mm_sfence(); return n;
}
// the compiled PREAMBLE40_11A_LUT (640 COMPLEX16), and the 8 samples the transmitter reads behind it
SBREF_API void ref_tx11a_legacy_preamble(int16_t* out1280) { memcpy(out1280, sbref_preamble40_lut, sizeof sbref_preamble40_lut); }
SBREF_API void ref_tx11a_legacy_set_pad(const int16_t* pad16) { memcpy(sbref_preamble40_read + 640, pad16, 8 * sizeof(COMPLEX16)); }
// the tap's lane counts since the last reset (see the build script's header for [0] .. [4])
SBREF_API void ref_tx11a_legacy_debug(uint64_t* out5) { for (int k = 0; k < 5; k++) out5[k] = sbref::counts[k]; }
SBREF_API void ref_tx11a_legacy_debug_reset(void) { for (int k = 0; k < 5; k++) sbref::counts[k] = 0; sbref::after_shl = 0; }
ENTRY
mkdir -p "$HERE/_ref"
CXXF="-O2 -std=c++17 -mssse3 -msse4.1 -fno-strict-aliasing -fno-operator-names -fpermissive -fPIC -w -fvisibility=hidden -fvisibility-inlines-hidden"
IDIR="-I$INC -I$REF/kernel/bb/dot11a/inc -I$REF/kernel/core/inc -I$REF/kernel/inc"
OBJ="$INC/obj"; mkdir -p "$OBJ"
OBJS=""
for f in atx_fe atx_6 atx_9 atx_12 atx_18 atx_24 atx_36 atx_48 atx_54; do
  ${CXX:-g++} $CXXF $IDIR -DPREAMBLE40_11A_LUT=sbref_preamble40_read -x c++ -c "$SRC/$f.c" -o "$OBJ/$f.o"
  OBJS="$OBJS $OBJ/$f.o"
done
for f in scramble_11a conv_encoder_1_2 conv_encoder_2_3 conv_encoder_3_4 interleave_6m interleave_12m interleave_24m interleave_48m \
         mapa_bpsk mapa_qpsk mapa_16qam mapa_64qam pilotsgn preamble40_11a; do
  ${CXX:-g++} $CXXF $IDIR -DPREAMBLE40_11A_LUT=sbref_preamble40_lut -x c++ -c "$REF/kernel/bb/dot11a/lutst/$f.c" -o "$OBJ/$f.o"
  OBJS="$OBJS $OBJ/$f.o"
done
${CXX:-g++} $CXXF $IDIR -c "$INC/entry.cpp" -o "$OBJ/entry.o"
rc=0
${CXX:-g++} -shared -o "$HERE/_ref/libtx11a_legacy_ref.so.tmp.$$" $OBJS "$OBJ/entry.o" || rc=$?
[ $rc -eq 0 ] || { rm -f "$HERE/_ref/libtx11a_legacy_ref.so.tmp.$$"; echo "build_ref_tx11a_legacy: link failed" >&2; exit 1; }
mv -f "$HERE/_ref/libtx11a_legacy_ref.so.tmp.$$" "$HERE/_ref/libtx11a_legacy_ref.so"
echo "build_ref_tx11a_legacy: oracle/_ref/libtx11a_legacy_ref.so"
