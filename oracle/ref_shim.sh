#!/bin/sh
# Sourced by the build_ref_*.sh scripts that compile reference bricks from their own headers: `ref_shim DIR` writes the headers those
# bricks include in place of the reference's framework headers, which only MSVC / the WDK compile.  Each stands for what the reference
# header gives the bricks, with the line it comes from.  TEST INFRASTRUCTURE ONLY; nothing of the reference is copied here.
# The shims:
#   tpltrick.h    intpow, ceiling_div (tpltrick.h:23-31), Log2, IsPower2, DummyInitializer and static_wrapper (tpltrick.h:95-148; the header itself redeclares template
#                 parameters as member typedefs, :91-96, which GCC rejects); operator_repeater.h: rep_mul, rep_shift_right, rep_sub,
#                 rep_memzero, rep_memcpy, rep_or as the loops operator_repeater.h:42-173, 314 unroll (its rep_saturated_sub names a member
#                 that does not exist, :182, which GCC rejects even uninstantiated);
#   const.h       the repo's own sora_b200/brick/brick.hpp (BRICK macros, TFilter / TSink, pin queues) with CTX_VAR_RW / CTX_VAR_RO /
#                 FACADE_FIELD taking the array extent the reference writes (CTX_VAR_RW(vcs, ChannelCoeffs, [16]), brick.h:426-470), a
#                 DEFINE_LOCAL_CONTEXT of up to ten facades, FINL / SELECTANY / A16 / MEM_ALIGN (core/inc/const.h:81-86), and
#                 _dump_symbol / _dump_text as no-ops (brick/inc/bb_debug.h:11-45 only print; with SB_DUMP_TEXT_TAP defined, _dump_text is
#                 left to the library, whose debug tap counts the messages);
#   brick.h, sora.h, dspcomm.h, soratime.h, bb/bba.h
#                 what those headers give the bricks here: brick/inc/dspcomm.h:5-21's includes (vector128.h, fft.h, intalg.h, dspalg.hpp,
#                 plus operator_repeater.h), SoraStopwatch with a no-op Restart (soratime.h) for CF_TimeStamps, SORA_RADIO_RX_STREAM / FLAG for CF_RxStream,
#                 COMPLEX32 (complex.h:6), SORA_RX_SIGNAL_UNIT_SIZE 16 / _NUM_PER_DESC 7 (_rx_manager.h:79-81);
#   vector128.h   vs / vi / vcs / vub (vector128.h:96-138, element access :107-108), SignalBlock (:1643-1648), and each operation as the
#                 intrinsic or body vector128.h gives it:
#     shifts      shift_right and >> on vcs (_mm_srai_epi16, :832) and on vi (_mm_srai_epi32, :830)
#     arithmetic  saturated_add / saturated_sub on vcs (_mm_adds/subs_epi16, :645, :655), xor (:567), and / or, sign (_mm_sign_epi16,
#                 :535), smin / smax on vcs (_mm_min/max_epi16, :1295, :1318), set_zero (:439)
#     shuffles    permutate<imm>, permutate_high<imm>, permutate_low<imm> (:688, :683, :677)
#     complex     conj (:966, XOR), conj0 (:979-989, psignw with 0x8000 on the imaginary halves: -32768 stays -32768), conjre (:952-961,
#                 psignw), flip (:992-996), mul_j (:1258-1261), pairwise_muladd / muladd (_mm_madd_epi16, :920-921), SquaredNorm
#                 (:932, muladd(a, a)), hadd on vi (:758, the four lanes summed and duplicated), pack(vi, vi) (:876-883: masked and
#                 interleaved, it wraps) and pack(vcs&, vi, vi) (:887-890), conj_mul into vi re / im (:1038-1044), mul into vi re / im
#                 (:1075-1081, conj0 then flip), mul(vcs, vcs) (:1201-1211: >> 15 then the wrapping pack) and the * on vcs it stands
#                 behind (DEFINE_OPERATOR_OVERLOAD(*, vcs, mul), :1500), mul_shift / conj_mul_shift (:1215-1246)
#     constants   the vector128_consts masks (:179-284) the FFT names
#     macros      DSP_INLINE / DSP_INLINE1 (:22-24); __declspec(selectany / align / deprecated)
#     802.11b     vcb and vci (:136, :140; COMPLEX32 is complex.h:6), shift_right / >> on vci (_mm_srai_epi32, :833),
#                 shift_element_left / shift_element_right (_mm_slli_si128 / _mm_srli_si128, :855-864: template arguments in the
#                 order barkerspread.hpp:294, :376 write them), insert<ndx> on vcs (_mm_insert_epi32, :1466), load (:1352)
#   complex_ext.h the COMPLEX16 operators + and - (short results, complex_ext.h:94, :107), >> (:115) and norm2 (:134-138); += and -= of
#                 a COMPLEX16 into a COMPLEX32 (:89-103);
#   operator_repeater.h, further: rep_sqrnorm (:195-211, SquaredNorm per vector) and rep_sum (:214-230, += on vi);
#   windef.h, soratypes.h   the Windows integer names the 802.11b headers use (USHORT, PUSHORT, BOOLEAN, BYTE / WORD / DWORD, ...)
#                 and soratypes.h:22-33's typedefs (its `ulong` is the compiler's `unsigned long`: a build that wants MSVC's 32-bit
#                 width defines the name itself);
#   demux.h       TDemux with up to eight outputs (kernel/brick/inc/demux.h:13-152: AddRef of every output, Reset and Flush of every
#                 output, an empty Process), DEFINE_OPORTS (brick.h:204-240), FlushPort(N) (brick.h:461), DummyBrick (brick.h:477-490),
#                 and the TDEMUX2/4/5/8 macro sets (demux.h:154-266, :343-382);
#   vector128.h, further: vb and saturated_pack(vs, vs) (_mm_packs_epi16, vector128.h:870), whose lanes feed sbref::tap_spack.
ref_shim() {
mkdir -p "$1/bb"
cat > "$1/const.h" <<'SHIM'
#pragma once
#include "brick.hpp"
#include <vector>
#define __int8 char
#define __int16 short
#define __int32 int
#define __int64 long long
#define __forceinline inline __attribute__((always_inline))
#define SELECTANY
#define A16 __attribute__((aligned(16)))
#define MEM_ALIGN(n) __attribute__((aligned(n)))
#define UCHAR unsigned char
#define A32 __attribute__((aligned(32)))
#undef CTX_VAR_RW
#undef CTX_VAR_RO
#undef FACADE_FIELD
#undef DEFINE_LOCAL_CONTEXT
#define CTX_VAR_RW(TYPE, NAME, ...) TYPE (&NAME)__VA_ARGS__;
#define CTX_VAR_RO(TYPE, NAME, ...) TYPE const (&NAME)__VA_ARGS__;
#define FACADE_FIELD(TYPE, NAME, ...) private: TYPE __##NAME##__ __VA_ARGS__; public: auto NAME() -> TYPE (&)__VA_ARGS__ { return __##NAME##__; }
#define SB_VBASES_7(a, b, c, d, e, f, g) SB_VBASES_6(a, b, c, d, e, f), virtual public g
#define SB_VBASES_8(a, b, c, d, e, f, g, h) SB_VBASES_7(a, b, c, d, e, f, g), virtual public h
#define SB_VBASES_9(a, b, c, d, e, f, g, h, i) SB_VBASES_8(a, b, c, d, e, f, g, h), virtual public i
#define SB_VBASES_10(a, b, c, d, e, f, g, h, i, j) SB_VBASES_9(a, b, c, d, e, f, g, h, i), virtual public j
#define SB_VB_PICK10(_1, _2, _3, _4, _5, _6, _7, _8, _9, _10, NAME, ...) NAME
#define DEFINE_LOCAL_CONTEXT(TPL_BRICK, ...) struct __LocalContext_##TPL_BRICK : SB_VB_PICK10(__VA_ARGS__, SB_VBASES_10, SB_VBASES_9, \
    SB_VBASES_8, SB_VBASES_7, SB_VBASES_6, SB_VBASES_5, SB_VBASES_4, SB_VBASES_3, SB_VBASES_2, SB_VBASES_1)(__VA_ARGS__) {};
template<int N> inline void _dump_symbol(const char*, const COMPLEX16*) {}
#ifdef SB_DUMP_TEXT_TAP
void _dump_text(const char* fmt, ...);
#else
inline void _dump_text(const char*, ...) {}
#endif
SHIM
printf '#pragma once\n#include "const.h"\n' > "$1/brick.h"
cat > "$1/tpltrick.h" <<'SHIM'
#pragma once
#include "const.h"
template<int N> struct Log2 { enum { value = Log2<N / 2>::value + 1 }; };
template<> struct Log2<1> { enum { value = 0 }; };
template<int N> struct IsPower2 { enum { IsFalse = (N & 1) + IsPower2<N / 2>::IsFalse }; };
template<> struct IsPower2<1> { enum { IsFalse = 0 }; };
template<int x, unsigned int p> struct intpow { enum { value = x * intpow<x, p - 1>::value }; };
template<int x> struct intpow<x, 0> { enum { value = 1 }; };
template<int x, int y> struct ceiling_div { enum { value = (x + y - 1) / y }; };
struct DummyInitializer { void operator()(...) { } };
template<typename T, typename INITIALIZER = DummyInitializer> class static_wrapper {
    static T value __attribute__((aligned(16)));
public:
    static_wrapper(INITIALIZER init_func = INITIALIZER()) { init_func(value); }
    operator T&() const { return value; }
    T& get() const { return value; }
};
template<typename T, typename INITIALIZER> T static_wrapper<T, INITIALIZER>::value;
SHIM
cat > "$1/operator_repeater.h" <<'SHIM'
#pragma once
#include "vector128.h"
template<size_t N, typename T> inline void rep_mul(T* dst, const T* src0, const T* src1) { for (size_t i = 0; i < N; i++) *dst++ = (*src0++) * (*src1++); }
template<size_t N, typename T> inline void rep_shift_right(T* dst, const T* src, const int nbits) { for (size_t i = 0; i < N; i++) *dst++ = (*src++) >> nbits; }
template<size_t N, typename T> inline void rep_sub(T* dst, const T* src, const T& val) { for (size_t i = 0; i < N; i++) *dst++ = sub(*src++, val); }
template<size_t N, typename T> inline void rep_memzero(T* dst) { for (size_t i = 0; i < N; i++) set_zero(*dst++); }
template<size_t N, typename T> inline void rep_memcpy(T* dst, const T* src) { for (size_t i = 0; i < N; i++) *dst++ = *src++; }
template<size_t N, typename T> inline void rep_or(T* dst, const T* src0, const T* src1) { for (size_t i = 0; i < N; i++) *dst++ = (*src0++) | (*src1++); }
template<size_t N> inline void rep_sqrnorm(vi* dst, const vcs* src) { for (size_t i = 0; i < N; i++) *dst++ = SquaredNorm(*src++); }
template<size_t N, typename T> inline void rep_sum(T& result, const T* src) { for (size_t i = 0; i < N; i++) result += *src++; }
SHIM
cat > "$1/sora.h" <<'SHIM'
#pragma once
#include "const.h"
#include "vector128.h"
#include "complex_ext.h"
typedef struct SORA_RADIO_RX_STREAM SORA_RADIO_RX_STREAM;
typedef unsigned char FLAG;
#define NODEFAULT __builtin_unreachable()
inline int ceil_div(int x, int mod) { return (x + mod - 1) / mod; }
SHIM
cat > "$1/complex_ext.h" <<'SHIM'
#pragma once
#include "const.h"
inline COMPLEX16 operator+(const COMPLEX16& a, const COMPLEX16& b) { COMPLEX16 r; r.re = (short)(a.re + b.re); r.im = (short)(a.im + b.im); return r; }
inline COMPLEX16 operator-(const COMPLEX16& a, const COMPLEX16& b) { COMPLEX16 r; r.re = (short)(a.re - b.re); r.im = (short)(a.im - b.im); return r; }
inline COMPLEX16 operator>>(const COMPLEX16& a, int n) { COMPLEX16 r; r.re = (short)(a.re >> n); r.im = (short)(a.im >> n); return r; }
inline int norm2(const COMPLEX16& a) { return a.re * a.re + a.im * a.im; }
inline COMPLEX32& operator+=(COMPLEX32& a, const COMPLEX16& b) { a.re += b.re; a.im += b.im; return a; }
inline COMPLEX32& operator-=(COMPLEX32& a, const COMPLEX16& b) { a.re -= b.re; a.im -= b.im; return a; }
SHIM
cat > "$1/windef.h" <<'SHIM'
#pragma once
typedef unsigned char BYTE, BOOLEAN, *PUCHAR;
typedef unsigned short WORD, USHORT, *PUSHORT;
typedef unsigned int DWORD, UINT, *PUINT;
#ifndef TRUE
#define TRUE 1
#define FALSE 0
#endif
#define IN
#define OUT
SHIM
cat > "$1/soratypes.h" <<'SHIM'
#pragma once
#include <emmintrin.h>
#include "windef.h"
#include "const.h"
typedef int s_int32; typedef unsigned int s_uint32; typedef short s_int16; typedef unsigned short s_uint16;
typedef COMPLEX16 SAMPLE, *PSAMPLE;
SHIM
cat > "$1/demux.h" <<'SHIM'
#pragma once
#include "const.h"
#include <type_traits>
class DummyBrick : public IReferenceCounting, public IControlPoint {
public:
    typedef ::iport_traits<void, 1> iport_traits;
    void Reset() override {}
    void Flush() override {}
    template<class T_IPIN> bool Process(T_IPIN& pin) { pin.clear(); return true; }
};
inline DummyBrick DummyBrickInstance;
#define NON_DUMMYBRICK(INDEX) (!std::is_same<T_NEXT##INDEX, DummyBrick>::value)
template<class T_CTX, class T_NEXT0 = DummyBrick, class T_NEXT1 = DummyBrick, class T_NEXT2 = DummyBrick, class T_NEXT3 = DummyBrick,
         class T_NEXT4 = DummyBrick, class T_NEXT5 = DummyBrick, class T_NEXT6 = DummyBrick, class T_NEXT7 = DummyBrick>
class TDemux : public TBrick<T_CTX>, public IReferenceCounting, public IControlPoint {
protected:
    T_NEXT0* __next_0; T_NEXT1* __next_1; T_NEXT2* __next_2; T_NEXT3* __next_3; T_NEXT4* __next_4; T_NEXT5* __next_5; T_NEXT6* __next_6;
    T_NEXT7* __next_7;
    T_NEXT0* Next0() { return __next_0; } T_NEXT1* Next1() { return __next_1; } T_NEXT2* Next2() { return __next_2; }
    T_NEXT3* Next3() { return __next_3; } T_NEXT4* Next4() { return __next_4; } T_NEXT5* Next5() { return __next_5; }
    T_NEXT6* Next6() { return __next_6; } T_NEXT7* Next7() { return __next_7; }
public:
    typedef TDemux TDemuxBase;
    TDemux(T_CTX& ctx, T_NEXT0* n0 = NULL, T_NEXT1* n1 = NULL, T_NEXT2* n2 = &DummyBrickInstance, T_NEXT3* n3 = &DummyBrickInstance,
           T_NEXT4* n4 = &DummyBrickInstance, T_NEXT5* n5 = &DummyBrickInstance, T_NEXT6* n6 = &DummyBrickInstance,
           T_NEXT7* n7 = &DummyBrickInstance)
        : TBrick<T_CTX>(ctx), __next_0(n0), __next_1(n1), __next_2(n2), __next_3(n3), __next_4(n4), __next_5(n5), __next_6(n6), __next_7(n7) {
        if (NON_DUMMYBRICK(0)) AddRef(Next0()); if (NON_DUMMYBRICK(1)) AddRef(Next1()); if (NON_DUMMYBRICK(2)) AddRef(Next2());
        if (NON_DUMMYBRICK(3)) AddRef(Next3()); if (NON_DUMMYBRICK(4)) AddRef(Next4()); if (NON_DUMMYBRICK(5)) AddRef(Next5());
        if (NON_DUMMYBRICK(6)) AddRef(Next6()); if (NON_DUMMYBRICK(7)) AddRef(Next7());
    }
    ~TDemux() {
        if (NON_DUMMYBRICK(0)) IReferenceCounting::Release(Next0()); if (NON_DUMMYBRICK(1)) IReferenceCounting::Release(Next1());
        if (NON_DUMMYBRICK(2)) IReferenceCounting::Release(Next2()); if (NON_DUMMYBRICK(3)) IReferenceCounting::Release(Next3());
        if (NON_DUMMYBRICK(4)) IReferenceCounting::Release(Next4()); if (NON_DUMMYBRICK(5)) IReferenceCounting::Release(Next5());
        if (NON_DUMMYBRICK(6)) IReferenceCounting::Release(Next6()); if (NON_DUMMYBRICK(7)) IReferenceCounting::Release(Next7());
    }
    void Reset() {
        if (NON_DUMMYBRICK(0)) Next0()->Reset(); if (NON_DUMMYBRICK(1)) Next1()->Reset(); if (NON_DUMMYBRICK(2)) Next2()->Reset();
        if (NON_DUMMYBRICK(3)) Next3()->Reset(); if (NON_DUMMYBRICK(4)) Next4()->Reset(); if (NON_DUMMYBRICK(5)) Next5()->Reset();
        if (NON_DUMMYBRICK(6)) Next6()->Reset(); if (NON_DUMMYBRICK(7)) Next7()->Reset();
    }
    void Flush() {
        if (NON_DUMMYBRICK(0)) Next0()->Flush(); if (NON_DUMMYBRICK(1)) Next1()->Flush(); if (NON_DUMMYBRICK(2)) Next2()->Flush();
        if (NON_DUMMYBRICK(3)) Next3()->Flush(); if (NON_DUMMYBRICK(4)) Next4()->Flush(); if (NON_DUMMYBRICK(5)) Next5()->Flush();
        if (NON_DUMMYBRICK(6)) Next6()->Flush(); if (NON_DUMMYBRICK(7)) Next7()->Flush();
    }
    template<class T_IPIN> bool Process(T_IPIN&) { return true; }
};
#undef FlushPort
#define FlushPort(N) do { if (opin##N().pad()) this->Next##N()->Process(opin##N()); this->Next##N()->Flush(); } while (false)
#define DEFINE_OPORTS(INDEX, TYPE, BURST)                                                                                      \
    typedef ::oport_traits<TYPE, BURST, 1> oport_traits##INDEX;                                                                \
    typedef typename DeducedPinQueue<oport_traits##INDEX, typename T_NEXT##INDEX::iport_traits>::type opin_type##INDEX;          \
    opin_type##INDEX __opin##INDEX##_;                                                                                           \
    opin_type##INDEX& opin##INDEX() { return __opin##INDEX##_; }
#define TDEMUX2_ARGS class T_CTX, class T_NEXT0, class T_NEXT1
#define TDEMUX2_PARAMS T_CTX, T_NEXT0, T_NEXT1
#define STD_DEMUX2_CONSTRUCTOR(name) name(T_CTX& ctx, T_NEXT0* n0, T_NEXT1* n1) : TDemux<TDEMUX2_PARAMS>(ctx, n0, n1)
#define STD_TDEMUX2_RESET() FINL void Reset() { this->TDemuxBase::Reset(); opin0().clear(); opin1().clear(); __ResetSelf(); } FINL void __ResetSelf()
#define TDEMUX4_ARGS class T_CTX, class T_NEXT0, class T_NEXT1, class T_NEXT2, class T_NEXT3
#define TDEMUX4_PARAMS T_CTX, T_NEXT0, T_NEXT1, T_NEXT2, T_NEXT3
#define STD_DEMUX4_CONSTRUCTOR(name) name(T_CTX& ctx, T_NEXT0* n0, T_NEXT1* n1, T_NEXT2* n2, T_NEXT3* n3) : TDemux<TDEMUX4_PARAMS>(ctx, n0, n1, n2, n3)
#define STD_TDEMUX4_RESET() FINL void Reset() { this->TDemuxBase::Reset(); opin0().clear(); opin1().clear(); opin2().clear(); opin3().clear(); __ResetSelf(); } \
    FINL void __ResetSelf()
#define TDEMUX5_ARGS class T_CTX, class T_NEXT0, class T_NEXT1, class T_NEXT2, class T_NEXT3, class T_NEXT4
#define TDEMUX5_PARAMS T_CTX, T_NEXT0, T_NEXT1, T_NEXT2, T_NEXT3, T_NEXT4
#define STD_DEMUX5_CONSTRUCTOR(name) name(T_CTX& ctx, T_NEXT0* n0, T_NEXT1* n1, T_NEXT2* n2, T_NEXT3* n3, T_NEXT4* n4) \
    : TDemux<TDEMUX5_PARAMS>(ctx, n0, n1, n2, n3, n4)
#define STD_TDEMUX5_RESET() FINL void Reset() { this->TDemuxBase::Reset(); opin0().clear(); opin1().clear(); opin2().clear(); opin3().clear(); \
    opin4().clear(); __ResetSelf(); } FINL void __ResetSelf()
#define TDEMUX8_ARGS class T_CTX, class T_NEXT0, class T_NEXT1, class T_NEXT2, class T_NEXT3, class T_NEXT4, class T_NEXT5, class T_NEXT6, class T_NEXT7
#define TDEMUX8_PARAMS T_CTX, T_NEXT0, T_NEXT1, T_NEXT2, T_NEXT3, T_NEXT4, T_NEXT5, T_NEXT6, T_NEXT7
#define STD_DEMUX8_CONSTRUCTOR(name) name(T_CTX& ctx, T_NEXT0* n0, T_NEXT1* n1, T_NEXT2* n2, T_NEXT3* n3, T_NEXT4* n4, T_NEXT5* n5, T_NEXT6* n6, \
                                          T_NEXT7* n7) : TDemux<TDEMUX8_PARAMS>(ctx, n0, n1, n2, n3, n4, n5, n6, n7)
#define STD_TDEMUX8_RESET() FINL void Reset() { this->TDemuxBase::Reset(); opin0().clear(); opin1().clear(); opin2().clear(); opin3().clear(); \
    opin4().clear(); opin5().clear(); opin6().clear(); opin7().clear(); __ResetSelf(); } FINL void __ResetSelf()
#define CREATE_BRICK_DEMUX2(NAME, TPL, CTX, N0, N1) \
    typedef TPL<std::remove_reference<decltype(CTX)>::type, std::remove_reference<decltype(*N0)>::type, std::remove_reference<decltype(*N1)>::type> __C_##NAME; \
    __C_##NAME* NAME = new __C_##NAME(CTX, N0, N1);
#define CREATE_BRICK_DEMUX5(NAME, TPL, CTX, N0, N1, N2, N3, N4) \
    typedef TPL<std::remove_reference<decltype(CTX)>::type, std::remove_reference<decltype(*N0)>::type, std::remove_reference<decltype(*N1)>::type, \
                std::remove_reference<decltype(*N2)>::type, std::remove_reference<decltype(*N3)>::type, std::remove_reference<decltype(*N4)>::type> __C_##NAME; \
    __C_##NAME* NAME = new __C_##NAME(CTX, N0, N1, N2, N3, N4);
#define CREATE_BRICK_DEMUX8(NAME, TPL, CTX, N0, N1, N2, N3, N4, N5, N6, N7) \
    typedef TPL<std::remove_reference<decltype(CTX)>::type, std::remove_reference<decltype(*N0)>::type, std::remove_reference<decltype(*N1)>::type, \
                std::remove_reference<decltype(*N2)>::type, std::remove_reference<decltype(*N3)>::type, std::remove_reference<decltype(*N4)>::type, \
                std::remove_reference<decltype(*N5)>::type, std::remove_reference<decltype(*N6)>::type, std::remove_reference<decltype(*N7)>::type> __C_##NAME; \
    __C_##NAME* NAME = new __C_##NAME(CTX, N0, N1, N2, N3, N4, N5, N6, N7);
SHIM
cat > "$1/soratime.h" <<'SHIM'
#pragma once
struct SoraStopwatch { explicit SoraStopwatch(bool) {} void Restart() {} };
SHIM
cat > "$1/dspcomm.h" <<'SHIM'
#pragma once
#include "const.h"
#include "vector128.h"
#include <fft.h>
#include <intalg.h>
#include "operator_repeater.h"
#include <dspalg.hpp>
SHIM
cat > "$1/bb/bba.h" <<'SHIM'
#pragma once
#include "../const.h"
#include "../vector128.h"
#define SORA_RX_SIGNAL_UNIT_SIZE 16
#define SORA_RX_SIGNAL_UNIT_NUM_PER_DESC 7
#define SORA_RX_SIGNAL_UNIT_COMPLEX16_NUM (SORA_RX_SIGNAL_UNIT_SIZE / sizeof(COMPLEX16))
SHIM
cat > "$1/vector128.h" <<'SHIM'
#pragma once
#include <smmintrin.h>
#include <stddef.h>
#include <string.h>
#include "const.h"
#define DSP_INLINE inline __attribute__((always_inline))
#define DSP_INLINE1 inline
#define __declspec(x) SB_DECLSPEC_##x
#define SB_DECLSPEC_selectany
#define SB_DECLSPEC_deprecated
#define SB_DECLSPEC_align(n) __attribute__((aligned(n)))
#define SB_VEC(NAME, TDATA)                                                                                     \
struct NAME {                                                                                                   \
    static const size_t size = 16 / sizeof(TDATA);                                                              \
    typedef TDATA data_type[size] __attribute__((aligned(16)));                                                 \
    typedef TDATA elem_type;                                                                                    \
    typedef __m128i raw_type;                                                                                   \
    NAME() {}                                                                                                   \
    explicit NAME(__m128i r) : _raw(r) {}                                                                       \
    template<typename TA> explicit NAME(const TA& a) : _raw((__m128i)a) {}                                      \
    NAME(const data_type& pa) : _raw(_mm_loadu_si128((const __m128i*)pa)) {}                                    \
    operator __m128i() const { return _raw; }                                                                   \
    TDATA& operator[](size_t i) { return ((TDATA*)&_raw)[i]; }                                                  \
    const TDATA& operator[](size_t i) const { return ((const TDATA*)&_raw)[i]; }                                \
    __m128i _raw;                                                                                               \
};
SB_VEC(vs, short)
SB_VEC(vi, int)
SB_VEC(vub, unsigned char)
SB_VEC(vcs, COMPLEX16)
typedef struct _COMPLEX32 { int re, im; } COMPLEX32;
SB_VEC(vci, COMPLEX32)
SB_VEC(vcb, COMPLEX8)
SB_VEC(vb, signed char)
struct COMPLEXU32 { unsigned int re, im; };
SB_VEC(vcui, COMPLEXU32)
template<typename T> inline T& cast_ref(void* p) { return *reinterpret_cast<T*>(p); }
template<typename T> inline const T& cast_ref(const void* p) { return *reinterpret_cast<const T*>(p); }
struct SignalBlock {
    static const size_t size = 7;
    vcs _data[size];
    vcs& operator[](size_t index) { return _data[index]; }
    const vcs& operator[](size_t index) const { return _data[index]; }
};
namespace sbref { extern int phase; void tap_pack(__m128i v, int k); void tap_zero(__m128i v); void tap_clamp(__m128i r, __m128i a);
                  void tap_madd(__m128i v); void tap_spack(__m128i a, __m128i b); }
class vector128_consts {
public:
    template<typename T> static T __0x0000FFFF0000FFFF0000FFFF0000FFFF() { return (T)_mm_set1_epi32(0x0000FFFF); }
    template<typename T> static T __0xFFFF0000FFFF0000FFFF0000FFFF0000() { return (T)_mm_set1_epi32((int)0xFFFF0000); }
    template<typename T> static T __0xFFFFFFFF00000000FFFFFFFF00000000() { return (T)_mm_set_epi32(-1, 0, -1, 0); }
    template<typename T> static T __0xFFFFFFFFFFFFFFFF0000000000000000() { return (T)_mm_set_epi32(-1, -1, 0, 0); }
    template<typename T> static T __0xFFFF0000FFFF00000000000000000000() { return (T)_mm_set_epi32((int)0xFFFF0000, (int)0xFFFF0000, 0, 0); }
    template<typename T> static T __0xFFFF0000000000000000000000000000() { return (T)_mm_set_epi32((int)0xFFFF0000, 0, 0, 0); }
};
template<typename T> inline void set_zero(T& a) { a = T(_mm_setzero_si128()); }
inline vcs shift_right(const vcs& a, int n) { return vcs(_mm_srai_epi16(a, n)); }
inline vi shift_right(const vi& a, int n) { vi r(_mm_srai_epi32(a, n)); if (n == 8) sbref::tap_zero(r); return r; }
inline vcs operator>>(const vcs& a, int n) { return shift_right(a, n); }
inline vi operator>>(const vi& a, int n) { return shift_right(a, n); }
inline vi operator+(const vi& a, const vi& b) { return vi(_mm_add_epi32(a, b)); }
inline vi& operator+=(vi& a, const vi& b) { a = a + b; return a; }
inline vci shift_right(const vci& a, int n) { return vci(_mm_srai_epi32(a, n)); }
inline vci operator>>(const vci& a, int n) { return shift_right(a, n); }
template<typename T, int n> inline T shift_element_left(const T& a) { return T(_mm_slli_si128(a, n * sizeof(typename T::elem_type))); }
template<typename T, int n> inline T shift_element_right(const T& a) { return T(_mm_srli_si128(a, n * sizeof(typename T::elem_type))); }
template<int ndx> inline vcs insert(const vcs& a, COMPLEX16 b) { unsigned int w; memcpy(&w, &b, 4); return vcs(_mm_insert_epi32(a, (int)w, ndx)); }
template<typename T> inline void load(T& r, const void* p) { r = T(_mm_loadu_si128((const __m128i*)p)); }
inline vi& operator*=(vi& a, const vi& b) { a = vi(_mm_mullo_epi32(a, b)); return a; }
inline vcs saturated_add(const vcs& a, const vcs& b) { return vcs(_mm_adds_epi16(a, b)); }
inline vcs saturated_sub(const vcs& a, const vcs& b) { return vcs(_mm_subs_epi16(a, b)); }
inline vcs xor(const vcs& a, const vcs& b) { return vcs(_mm_xor_si128(a, b)); }
inline vcs sign(const vcs& a, const vcs& b) { return vcs(_mm_sign_epi16(a, b)); }
inline vcs smin(const vcs& a, const vcs& b) { vcs r(_mm_min_epi16(a, b)); sbref::tap_clamp(r, a); return r; }
inline vcs smax(const vcs& a, const vcs& b) { vcs r(_mm_max_epi16(a, b)); sbref::tap_clamp(r, a); return r; }
template<int imm> inline vcs permutate(const vcs& a) { return vcs(_mm_shuffle_epi32(a, imm)); }
template<int a0, int a1, int a2, int a3> inline vcs permutate(const vcs& a) { return vcs(_mm_shuffle_epi32(a, _MM_SHUFFLE(a3, a2, a1, a0))); }
inline vcui interleave_low(const vcui& a, const vcui& b) { return vcui(_mm_unpacklo_epi64(a, b)); }
inline vcs add(const vcs& a, const vcs& b) { return vcs(_mm_add_epi16(a, b)); }
inline vcs sub(const vcs& a, const vcs& b) { return vcs(_mm_sub_epi16(a, b)); }
inline vcs hadd(const vcs& a) {
    __m128i s = _mm_add_epi16(a, _mm_shuffle_epi32(a, 0x4E));
    return vcs(_mm_add_epi16(s, _mm_shuffle_epi32(s, 0xB1)));
}
inline int SquaredNorm(const COMPLEX16& c) { return c.re * c.re + c.im * c.im; }
template<int imm> inline vcs permutate_high(const vcs& a) { return vcs(_mm_shufflehi_epi16(a, imm)); }
template<int imm> inline vcs permutate_low(const vcs& a) { return vcs(_mm_shufflelo_epi16(a, imm)); }
inline vcs conj(const vcs& a) { return xor(a, vector128_consts::__0xFFFF0000FFFF0000FFFF0000FFFF0000<vcs>()); }
inline vcs conj0(const vcs& a) { return sign(a, vcs(_mm_set1_epi32((int)0x80000001))); }
inline vcs conjre(const vcs& a) { return sign(a, vcs(_mm_set1_epi32(0x00018000))); }
inline vcs flip(const vcs& a) { vcs b = permutate_low<0xb1>(a); return permutate_high<0xb1>(b); }
inline vcs mul_j(const vcs& a) { return xor(flip(a), vector128_consts::__0x0000FFFF0000FFFF0000FFFF0000FFFF<vcs>()); }
inline vi pairwise_muladd(const vs& a, const vs& b) { __m128i r = _mm_madd_epi16(a, b); sbref::tap_madd(r); return vi(r); }
inline vi muladd(const vcs& a, const vcs& b) { __m128i r = _mm_madd_epi16(a, b); sbref::tap_madd(r); return vi(r); }
inline vi SquaredNorm(const vcs& a) { return muladd(a, a); }
inline vi hadd(const vi& a) {
    __m128i s = _mm_add_epi32(a, _mm_shuffle_epi32(a, 0x4E));
    return vi(_mm_add_epi32(s, _mm_shuffle_epi32(s, 0xB1)));
}
inline vs pack(const vi& a, const vi& b) {
    const __m128i m = vector128_consts::__0x0000FFFF0000FFFF0000FFFF0000FFFF<vi>();
    return vs(_mm_or_si128(_mm_and_si128(a, m), _mm_slli_epi32(_mm_and_si128(b, m), 16)));
}
inline vb saturated_pack(const vs& a, const vs& b) { sbref::tap_spack(a, b); return vb(_mm_packs_epi16(a, b)); }
inline void pack(vcs& r, const vi& re, const vi& im) { sbref::tap_pack(re, 0); sbref::tap_pack(im, 0); r = (vcs)pack(re, im); }
inline void conj_mul(vi& re, vi& im, const vcs& a, const vcs& b) {
    vcs vs1 = flip(b);
    vs1 = conjre(vs1);
    re = pairwise_muladd((vs&)a, (vs&)b);
    im = pairwise_muladd((vs&)vs1, (vs&)a);
}
inline void mul(vi& re, vi& im, const vcs& a, const vcs& b) {
    vcs vs1 = conj0(b);
    vcs vs2 = flip(b);
    re = muladd(a, vs1);
    im = muladd(a, vs2);
}
inline vcs mul(const vcs& a, const vcs& b) {
    vi re, im;
    mul(re, im, a, b);
    re = shift_right(re, 15);
    im = shift_right(im, 15);
    sbref::tap_pack(re, 1); sbref::tap_pack(im, 1);
    return (vcs)pack(re, im);
}
inline vcs operator*(const vcs& a, const vcs& b) { return mul(a, b); }
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
}
