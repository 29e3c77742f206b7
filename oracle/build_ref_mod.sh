#!/bin/sh
# oracle/_ref/libmod_ref.so: the reference's 802.11a brick modulator, compiled from its own headers where they lie, brick by brick and as
# the two graphs kernel/bb/demod11/fb11amod_config.hpp builds:
#   CreatePreamble11a_40M (:150-158): TTS11aSrc (Brick11/src/preamble11a.hpp) -> TPackSample16to8 -> TModSink;
#   CreateModGraph11a_40M (:75-118): TBB11aSrc -> T11aSc -> TBB11aMRSelect (PHY_11a.hpp:11-304, scramble.hpp:170-262) -> TConvEncode_12 /
#     _23 / _34 (conv_enc.hpp) -> T11aInterleaveBPSK / QPSK / QAM16 / QAM64 (interleave.hpp) -> TMap11aBPSK / QPSK / QAM16 / QAM64<>
#     (mapper11a.hpp) -> TNoInline -> T11aAddPilot<> (pilot.hpp:10-119) -> TIFFTx (fft.hpp:9-60, IFFT<128> of the reference's fft.h)
#     -> TPackSample16to8 -> TModSink.
# TNoInline, TModSink, TPackSample16to8 and TDropAny are cut at build time out of kernel/brick/inc/stdbrick.hpp, whose other bricks
# need the radio stream headers.  The entry restates two things only, each citing the lines it restates: the graph wiring, and the
# driver of Test11A_FB_Mod (kernel/bb/demod11/fb11a_mod.cpp:27-74: set_mod_buffer, preamble Reset / Process, init, then Reset, Process,
# Flush of the data graph), with sc_seed set per frame after init() (init() writes 0xFF, :53) because the device takes one seed per
# frame.  The shims are oracle/ref_shim.sh's (TDemux with eight outputs among them).
#
# `ulong` is 32 bits, as under MSVC: T11Interleave packs its output in 32-bit entries ("ulong is 32 bits", interleave.hpp:24), TModSink
# keeps error_code in one and TBB11aSrc hands the FCS on through (uchar*)&crc32.  A static_assert checks it.  -fwrapv: MSVC wraps
# signed overflow; -ffp-contract=off and no -ffast-math: the mapper levels are (short)(10720 / 1.414) and the like, in double.
# A debug tap counts which edges the inputs reach (ref_mod_debug below): pack lanes that saturate and, read from
# what TModSink wrote, the 9 Mbps symbol-pair padding and frames where GetPadingByte's padding yields a symbol beyond the standard's N_SYM.
# Nothing of the reference is copied into the repository.  TEST INFRASTRUCTURE ONLY.
#   usage: oracle/build_ref_mod.sh [reference root, default /root/reference]
set -e
REF="${1:-/root/reference}"
B11="$REF/kernel/bb/Brick11/src"
BINC="$REF/kernel/brick/inc"
CORE="$REF/kernel/core/inc"
HERE="$(cd "$(dirname "$0")" && pwd)"
[ -f "$B11/PHY_11a.hpp" ] || { echo "build_ref_mod: $B11/PHY_11a.hpp not found (fine outside the build container: the prebuilt oracle/_ref is used)"; exit 0; }
INC="$HERE/_ref/mod_inc"
rm -rf "$INC"
. "$HERE/ref_shim.sh"
ref_shim "$INC"
# stdbrick.hpp: the four bricks the modulator graphs name, each cut whole from its DEFINE_LOCAL_CONTEXT to the closing `};`
{ printf '#pragma once\n#include "const.h"\n#include "vector128.h"\n#include "stdfacade.h"\n'
  for b in TNoInline TModSink TPackSample16to8 TDropAny; do sed -n "/^DEFINE_LOCAL_CONTEXT($b,/,/^};/p" "$BINC/stdbrick.hpp"; done; } > "$INC/stdbrick_mod.hpp"
# PHY_11a.hpp up to the end of TBB11aMRSelect: the receive bricks behind it need the demodulator's facades, and thread_if.h (the
# thread primitives they use) is left out
sed -n '1,/^TBB11aMRSelect - modulation multi-rate selector/p' "$B11/PHY_11a.hpp" | sed '/^#include "thread_if.h"/d' > "$INC/phy11a_mod.hpp"
sed -n '/^TBB11aMRSelect - modulation multi-rate selector/,/^};/p' "$B11/PHY_11a.hpp" | sed '1d' >> "$INC/phy11a_mod.hpp"
for b in TNoInline TModSink TPackSample16to8 TDropAny; do grep -q "class $b " "$INC/stdbrick_mod.hpp" || { echo "build_ref_mod: stdbrick.hpp cut lost $b" >&2; exit 1; }; done
grep -q 'class TBB11aSrc' "$INC/phy11a_mod.hpp" && grep -q 'class TBB11aMRSelect' "$INC/phy11a_mod.hpp" && ! grep -q 'TBB11aSymSel' "$INC/phy11a_mod.hpp" \
  || { echo "build_ref_mod: PHY_11a.hpp cut did not apply" >&2; exit 1; }
# CRC32.h and func.h are reached through symbolic links, so that their quoted includes find the shims; sora.h then takes ceil_div from
# func.h (mapper11a.hpp includes it for BitReverseN and GrayToBinary) instead of declaring its own
LINKS="CRC32.h func.h"
for h in $LINKS; do ln -s "$CORE/$h" "$INC/$h"; done
sed -i 's/^inline int ceil_div(int x, int mod).*$/#include "func.h"/' "$INC/sora.h"
grep -q '^#include "func.h"' "$INC/sora.h" || { echo "build_ref_mod: sora.h shim rewrite did not apply" >&2; exit 1; }
cat > "$INC/entry.cpp" <<'ENTRY'
#define SORA_EXTERN_C
#include <immintrin.h>
#include <stdio.h>
#include <stdlib.h>
#include <stdint.h>
#include <string.h>
#include <limits.h>
#include <vector>
#include "windef.h"
#include "const.h"
#include "vector128.h"
#include "operator_repeater.h"
#include "complex_ext.h"
#include "tpltrick.h"
#include "sora.h"
#include "soratime.h"
#include "dspcomm.h"
#include "soratypes.h"
#include "demux.h"

namespace sbref {
// [0] TPackSample16to8 lanes that saturated, [1] 9 Mbps frames whose transmitted symbol count is even and one more than the standard's
// N_SYM: the symbol pair of GetPadingByte (Ndbps doubled, PHY_11a.hpp:116), [2] frames at any rate whose transmitted symbol count exceeds
// N_SYM.  [1] and [2] are read from what TModSink wrote (tx_sample_cnt), not from the frame's length and rate.
// IFFT<128>'s own edges (twiddle products the pack truncates, saturating adds that clip) are counted by oracle/build_ref_fft.sh's library,
// whose hill-climbed corpus reaches them; TIFFTx hands it a spectrum whose middle half is zero, and no corpus here was seen to reach them.
static thread_local uint64_t counts[3];
int phase;
void tap_pack(__m128i, int) {} void tap_zero(__m128i) {} void tap_clamp(__m128i, __m128i) {} void tap_madd(__m128i) {}
void tap_spack(__m128i a, __m128i b) {
    const __m128i lo = _mm_set1_epi16(-128), hi = _mm_set1_epi16(127);
    for (__m128i v : {a, b}) {
        const __m128i out = _mm_or_si128(_mm_cmplt_epi16(v, lo), _mm_cmpgt_epi16(v, hi));
        counts[0] += (unsigned)__builtin_popcount((unsigned)_mm_movemask_epi8(out)) / 2;
    }
}
}

#define ulong unsigned int
#define ULONG unsigned int
#define PULONG unsigned int*
#define SB_DECLSPEC_noinline __attribute__((noinline))
static_assert(sizeof(ulong) == 4, "MSVC's unsigned long is 32 bits");
#include "ieee80211facade.hpp"
#include "CRC32.h"
#include "stdbrick_mod.hpp"
#include "scramble.hpp"
#include "conv_enc.hpp"
template<class A, class B> constexpr A max(A a, B b) { return a > (A)b ? a : (A)b; }    // windef.h's max, as interleave.hpp:25 uses it
#include "interleave.hpp"
#include "mapper11a.hpp"
#include "pilot.hpp"
#include "fft.hpp"
#include "preamble11a.hpp"
#include "phy11a_mod.hpp"

// a sink that keeps every burst it is handed
template<class T, size_t B> struct Cap {
    template<class T_CTX> class Sink : public TSink<T_CTX> {
    public:
        DEFINE_IPORT(T, B);
        std::vector<T> got;
        explicit Sink(T_CTX& ctx) : TSink<T_CTX>(ctx) {}
        BOOL_FUNC_PROCESS(ipin) { while (ipin.check_read()) { got.insert(got.end(), ipin.peek(), ipin.peek() + B); ipin.pop(); } return true; }
    };
};

// _tagBB11aModContext (fb11amod_config.hpp:18-58): the facades of TDropAny, TModSink, T11aSc and TBB11aSrc, set_mod_buffer (:24-32) and
// init (:34-57).  The local contexts of TTS11aSrc (CF_Error) and TBB11aMRSelect (CF_11aTxVector) name facades that are already there; they
// are listed because the shim's BIND_CONTEXT casts to the brick's own local context
struct Ctx11a : LOCAL_CONTEXT(TDropAny), LOCAL_CONTEXT(TModSink), LOCAL_CONTEXT(T11aSc), LOCAL_CONTEXT(TBB11aSrc), LOCAL_CONTEXT(TTS11aSrc),
                LOCAL_CONTEXT(TBB11aMRSelect) {
    void set_mod_buffer(COMPLEX8* buf, ulong size) {
        CF_Error::error_code() = E_ERROR_SUCCESS;
        CF_TxSampleBuffer::tx_sample_buf() = buf; CF_TxSampleBuffer::tx_sample_buf_size() = size;
    }
    void init(uint rate_kbps, uchar* buf, ushort len, COMPLEX8* sbuf, ulong sbuf_size) {
        CF_11aTxVector::frame_length() = len; CF_11aTxVector::data_rate_kbps() = rate_kbps; CF_11aTxVector::crc32() = CalcCRC32(buf, len);
        CF_TxFrameBuffer::mpdu_buf0() = buf; CF_TxFrameBuffer::mpdu_buf1() = NULL;
        CF_TxFrameBuffer::mpdu_buf_size0() = len; CF_TxFrameBuffer::mpdu_buf_size1() = 0;
        CF_Error::error_code() = E_ERROR_SUCCESS;
        CF_ScramblerSeed::sc_seed() = 0xFF;
        CF_TxSampleBuffer::tx_sample_buf() = sbuf; CF_TxSampleBuffer::tx_sample_buf_size() = sbuf_size;
    }
    Ctx11a() {
        CF_TxSampleBuffer::tx_sample_buf() = NULL; CF_TxSampleBuffer::tx_sample_buf_size() = 0; CF_TxSampleBuffer::tx_sample_cnt() = 0;
        CF_TxFrameBuffer::mpdu_buf0() = NULL; CF_TxFrameBuffer::mpdu_buf1() = NULL;
        CF_TxFrameBuffer::mpdu_buf_size0() = 0; CF_TxFrameBuffer::mpdu_buf_size1() = 0;
        CF_11aTxVector::frame_length() = 0; CF_11aTxVector::data_rate_kbps() = 6000; CF_11aTxVector::crc32() = 0;
        CF_ScramblerSeed::sc_seed() = 0xFF; CF_ScramblerControl::scramble_ctrl() = CF_ScramblerControl::DO_SCRAMBLE;
        CF_Error::error_code() = E_ERROR_SUCCESS;
    }
};

// CreatePreamble11a_40M (fb11amod_config.hpp:150-158)
static ISource* CreatePreamble11a_40M(Ctx11a& BB11aModCtx) {
    CREATE_BRICK_SINK  (modsink, TModSink, BB11aModCtx);
    CREATE_BRICK_FILTER(pack, TPackSample16to8, BB11aModCtx, modsink);
    CREATE_BRICK_SOURCE(ssrc, TTS11aSrc, BB11aModCtx, pack);
    return ssrc;
}
// CreateModGraph11a_40M (fb11amod_config.hpp:75-118); the unconnected TDropAny it creates is left out
static ISource* CreateModGraph11a_40M(Ctx11a& BB11aModCtx) {
    CREATE_BRICK_SINK  (modsink, TModSink, BB11aModCtx);
    CREATE_BRICK_FILTER(pack, TPackSample16to8, BB11aModCtx, modsink);
    CREATE_BRICK_FILTER(ifft, TIFFTx, BB11aModCtx, pack);
    CREATE_BRICK_FILTER(addpilot1, T11aAddPilot<>::Filter, BB11aModCtx, ifft);
    CREATE_BRICK_FILTER(addpilot, TNoInline, BB11aModCtx, addpilot1);
    CREATE_BRICK_FILTER(map_bpsk, TMap11aBPSK<>::Filter, BB11aModCtx, addpilot);
    CREATE_BRICK_FILTER(map_qpsk, TMap11aQPSK<>::Filter, BB11aModCtx, addpilot);
    CREATE_BRICK_FILTER(map_qam16, TMap11aQAM16<>::Filter, BB11aModCtx, addpilot);
    CREATE_BRICK_FILTER(map_qam64, TMap11aQAM64<>::Filter, BB11aModCtx, addpilot);
    CREATE_BRICK_FILTER(inter_bpsk, T11aInterleaveBPSK::Filter, BB11aModCtx, map_bpsk);
    CREATE_BRICK_FILTER(inter_qpsk, T11aInterleaveQPSK::Filter, BB11aModCtx, map_qpsk);
    CREATE_BRICK_FILTER(inter_qam16, T11aInterleaveQAM16::Filter, BB11aModCtx, map_qam16);
    CREATE_BRICK_FILTER(inter_qam64, T11aInterleaveQAM64::Filter, BB11aModCtx, map_qam64);
    CREATE_BRICK_FILTER(enc6, TConvEncode_12, BB11aModCtx, inter_bpsk);
    CREATE_BRICK_FILTER(enc9, TConvEncode_34, BB11aModCtx, inter_bpsk);
    CREATE_BRICK_FILTER(enc12, TConvEncode_12, BB11aModCtx, inter_qpsk);
    CREATE_BRICK_FILTER(enc18, TConvEncode_34, BB11aModCtx, inter_qpsk);
    CREATE_BRICK_FILTER(enc24, TConvEncode_12, BB11aModCtx, inter_qam16);
    CREATE_BRICK_FILTER(enc36, TConvEncode_34, BB11aModCtx, inter_qam16);
    CREATE_BRICK_FILTER(enc48, TConvEncode_23, BB11aModCtx, inter_qam64);
    CREATE_BRICK_FILTER(enc54, TConvEncode_34, BB11aModCtx, inter_qam64);
    CREATE_BRICK_DEMUX8(mrsel, TBB11aMRSelect, BB11aModCtx, enc6, enc9, enc12, enc18, enc24, enc36, enc48, enc54);
    CREATE_BRICK_FILTER(sc, T11aSc, BB11aModCtx, mrsel);
    CREATE_BRICK_SOURCE(ssrc, TBB11aSrc, BB11aModCtx, sc);
    return ssrc;
}

// one brick on its own from a fresh context: nburst bursts of NI inputs pushed one by one, every output kept
template<class B, class TI, size_t NI, class TO, size_t NO, class C>
static size_t run_brick(C& ctx, const TI* in, size_t nburst, TO* out) {
    typedef typename Cap<TO, NO>::template Sink<C> S;
    S* s = new S(ctx);
    typedef typename B::template Bound<C, S> BB;
    BB* f = new BB(ctx, s);
    TPinQueue<TI, NI, NI>* q = new TPinQueue<TI, NI, NI>();
    for (size_t i = 0; i < nburst; i++) { memcpy(q->append(), in + NI * i, NI * sizeof(TI)); f->Process(*q); }
    const size_t m = s->got.size();
    memcpy(out, s->got.data(), m * sizeof(TO));
    delete q; delete f;
    return m;
}
// binders from the reference's two brick spellings (template<TFILTER_ARGS> class B, and class X { template<TFILTER_ARGS> class Filter })
template<template<class, class> class B> struct Plain { template<class C, class N> using Bound = B<C, N>; };
template<class X> struct Nested { template<class C, class N> using Bound = typename X::template Filter<C, N>; };

static int nbpsc_of(unsigned kbps) {
    switch (kbps) { case 6000: case 9000: return 1; case 12000: case 18000: return 2; case 24000: case 36000: return 4; case 48000: case 54000: return 6; }
    return 0;
}

extern "C" {
void ref_mod_debug_reset() { for (int k = 0; k < 3; k++) sbref::counts[k] = 0; }
// what the tap counted since the last ref_mod_debug_reset on this thread (see sbref::counts)
void ref_mod_debug(uint64_t out[3]) { for (int k = 0; k < 3; k++) out[k] = sbref::counts[k]; }

// one 802.11a frame as Test11A_FB_Mod makes it (fb11a_mod.cpp:27-74) on a fresh context: the preamble graph, then init() with the
// payload (the graph appends its CRC-32), sc_seed, then Reset, Process and Flush of the data graph.  TModSink writes without a bound
// (stdbrick.hpp:318-327), so its buffer is sized here from the frame: the preamble, SIGNAL, the standard's N_SYM and two symbols more
// (GetPadingByte pads to at most a symbol pair, and the tail byte to at most one symbol beyond N_SYM).  out = COMPLEX8 pairs, room for
// cap samples; min(n, cap) are copied.  Returns n, the number of samples the graphs wrote (TS_len + tx_sample_cnt), -1 for an unknown
// rate, or -(error_code) if a graph raised one
int64_t ref_mod11a_frame(const uint8_t* payload, uint32_t len, uint32_t rate_kbps, uint8_t sc_seed, int8_t* out, size_t cap) {
    if (!nbpsc_of(rate_kbps)) return -1;
    const unsigned ndbps = rate_kbps / 250u;                      // N_DBPS: 24 at 6 Mbps .. 216 at 54 Mbps
    const unsigned std_nsym = (16u + 8u * (len + 4u) + 6u + ndbps - 1u) / ndbps;
    const size_t room = 640 + 160 * (size_t)(1 + std_nsym + 2);
    Ctx11a* ctx = new Ctx11a();
    std::vector<uint8_t> data(payload, payload + len);
    std::vector<COMPLEX8> buf(room);
    ISource* ssrc = CreateModGraph11a_40M(*ctx);
    ISource* tssrc = CreatePreamble11a_40M(*ctx);
    COMPLEX8* p = buf.data();
    ctx->set_mod_buffer(p, (ulong)room);
    tssrc->Reset();
    if (ctx->CF_Error::error_code() == E_ERROR_SUCCESS) tssrc->Process();
    const uint ts_len = ctx->CF_TxSampleBuffer::tx_sample_cnt();
    p += ts_len;
    ctx->init(rate_kbps, data.data(), (ushort)len, p, (ulong)(room - ts_len));
    ctx->CF_ScramblerSeed::sc_seed() = sc_seed;
    ssrc->Reset();
    int64_t r;
    if (ctx->CF_Error::error_code() == E_ERROR_SUCCESS) {
        ssrc->Process(); ssrc->Flush();
        const uint cnt = ctx->CF_TxSampleBuffer::tx_sample_cnt(), n = ts_len + cnt;
        memcpy(out, buf.data(), (size_t)(n < cap ? n : cap) * sizeof(COMPLEX8));
        r = (int64_t)n;
        const unsigned nsym = (cnt - 160u) / 160u;                // data symbols, from what TModSink wrote (SIGNAL is the first 160)
        if (rate_kbps == 9000 && nsym == std_nsym + 1u && nsym % 2u == 0u) sbref::counts[1]++;
        if (nsym > std_nsym) sbref::counts[2]++;
    } else r = -(int64_t)ctx->CF_Error::error_code();
    IReferenceCounting::Release(ssrc); IReferenceCounting::Release(tssrc);
    delete ctx;
    return r;
}
// T11aSc alone: n bytes, ctrl[i] the CF_ScramblerControl code in force for byte i (0 NO_SCRAMBLE, 1 DO_SCRAMBLE, 2 TAIL_SCRAMBLE)
void ref_mod11a_scramble(const uint8_t* in, const uint8_t* ctrl, size_t n, uint8_t seed, uint8_t* out) {
    Ctx11a* ctx = new Ctx11a(); ctx->CF_ScramblerSeed::sc_seed() = seed;
    typedef Cap<uchar, 1>::Sink<Ctx11a> S;
    S* s = new S(*ctx);
    T11aSc<Ctx11a, S>* f = new T11aSc<Ctx11a, S>(*ctx, s);
    TPinQueue<uchar, 1, 1>* q = new TPinQueue<uchar, 1, 1>();
    for (size_t i = 0; i < n; i++) { ctx->CF_ScramblerControl::scramble_ctrl() = ctrl[i]; *q->append() = in[i]; f->Process(*q); }
    memcpy(out, s->got.data(), n);
    delete q; delete f; delete ctx;
}
// TConvEncode_12 (cr 0), _23 (cr 1), _34 (cr 2) on n bytes; returns the coded bytes written
size_t ref_mod11a_encode(int cr, const uint8_t* in, size_t n, uint8_t* out) {
    Ctx11a ctx;
    switch (cr) {
    case 0: return run_brick<Plain<TConvEncode_12>, uchar, 1, uchar, 2>(ctx, in, n, out);
    case 1: return run_brick<Plain<TConvEncode_23>, uchar, 2, uchar, 3>(ctx, in, n / 2, out);
    default: return run_brick<Plain<TConvEncode_34>, uchar, 3, uchar, 4>(ctx, in, n / 3, out);
    }
}
// T11aInterleave{BPSK,QPSK,QAM16,QAM64} on nsym symbols of 6 * nbpsc bytes
void ref_mod11a_interleave(int nbpsc, const uint8_t* in, size_t nsym, uint8_t* out) {
    Ctx11a ctx;
    switch (nbpsc) {
    case 1: run_brick<Nested<T11aInterleaveBPSK>, uchar, 6, uchar, 6>(ctx, in, nsym, out); break;
    case 2: run_brick<Nested<T11aInterleaveQPSK>, uchar, 12, uchar, 12>(ctx, in, nsym, out); break;
    case 4: run_brick<Nested<T11aInterleaveQAM16>, uchar, 24, uchar, 24>(ctx, in, nsym, out); break;
    default: run_brick<Nested<T11aInterleaveQAM64>, uchar, 36, uchar, 36>(ctx, in, nsym, out);
    }
}
// TMap11a{BPSK,QPSK,QAM16,QAM64}<> on n input bursts (1, 1, 1, 3 bytes); returns the COMPLEX16 written
size_t ref_mod11a_map(int nbpsc, const uint8_t* in, size_t nburst, int16_t* out) {
    Ctx11a ctx; COMPLEX16* o = (COMPLEX16*)out;
    switch (nbpsc) {
    case 1: return run_brick<Nested<TMap11aBPSK<> >, uchar, 1, COMPLEX16, 8>(ctx, in, nburst, o);
    case 2: return run_brick<Nested<TMap11aQPSK<> >, uchar, 1, COMPLEX16, 4>(ctx, in, nburst, o);
    case 4: return run_brick<Nested<TMap11aQAM16<> >, uchar, 1, COMPLEX16, 2>(ctx, in, nburst, o);
    default: return run_brick<Nested<TMap11aQAM64<> >, uchar, 3, COMPLEX16, 4>(ctx, in, nburst, o);
    }
}
// T11aAddPilot<> on nsym symbols of 48 data carriers (pilot index from 127, as after Reset), 64 carriers out per symbol
void ref_mod11a_add_pilot(const int16_t* in, size_t nsym, int16_t* out) {
    Ctx11a ctx;
    run_brick<Nested<T11aAddPilot<> >, COMPLEX16, 48, COMPLEX16, 64>(ctx, (const COMPLEX16*)in, nsym, (COMPLEX16*)out);
}
// TIFFTx on nsym spectra of 64 carriers, 160 samples out per symbol
void ref_mod11a_ifftx(const int16_t* in, size_t nsym, int16_t* out) {
    Ctx11a ctx;
    run_brick<Plain<TIFFTx>, COMPLEX16, 64, COMPLEX16, 160>(ctx, (const COMPLEX16*)in, nsym, (COMPLEX16*)out);
}
// TPackSample16to8 on n blocks of 8 COMPLEX16
void ref_pack16to8(const int16_t* in, size_t nblk, int8_t* out) {
    Ctx11a ctx;
    run_brick<Plain<TPackSample16to8>, COMPLEX16, 8, COMPLEX8, 8>(ctx, (const COMPLEX16*)in, nblk, (COMPLEX8*)out);
}
}
ENTRY
mkdir -p "$HERE/_ref"
rc=0
${CXX:-g++} -O2 -std=c++17 -fwrapv -ffp-contract=off -mssse3 -msse4.1 -fno-strict-aliasing -fno-operator-names -fpermissive -fPIC -shared \
  -fmax-errors=15 -w -include functional -include memory -I"$INC" -I"$B11" -I"$BINC" -I"$CORE" -I"$HERE/../sora_b200/brick" "$INC/entry.cpp" \
  -o "$HERE/_ref/libmod_ref.so.tmp.$$" || rc=$?
for h in $LINKS stdbrick_mod.hpp phy11a_mod.hpp; do rm -f "$INC/$h"; done
[ $rc -eq 0 ] || { rm -f "$HERE/_ref/libmod_ref.so.tmp.$$"; echo "build_ref_mod: compile failed" >&2; exit 1; }
mv -f "$HERE/_ref/libmod_ref.so.tmp.$$" "$HERE/_ref/libmod_ref.so"
echo "build_ref_mod: oracle/_ref/libmod_ref.so"
