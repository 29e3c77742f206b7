#!/bin/sh
# oracle/_ref/librx11n_ref.so: the reference's PLCP header parsers and the back end both OFDM receivers share, compiled from its own
# headers where they lie and driven brick by brick from a fresh context:
#   T11aPLCPParser (kernel/bb/Brick11/src/PHY_11a.hpp:518-604) with BB11aParseDataRate, BB11aGetCodingRateFromDataRate and
#     B11aGetSymbolCount (ieee80211a_cmn.h);
#   T11nSigParser (PHY_11n.hpp:400-514) with CalcCRC8 (kernel/core/inc/CRC8.h), BB11nGetCodingRateFromMcsIndex and ht_symbol_count
#     (ieee80211n_cmn.h);
#   T11aDesc (scramble.hpp:267-355) into TBB11aFrameSink (PHY_11a.hpp:607-702) with CalcCRC32Incremental (kernel/core/inc/CRC32.h).
# The 802.11n front end (TCCA11n, TFreqEstimator_11n, the SISO / MIMO channel bricks, TPilotTrack_11n, the T11nDemap* and
# T11nDeinterleave* bricks, TStreamConcat) is not compiled here yet; its oracle is still checked only by loop-back (DESIGN §7).
# The facades come from source too (ieee80211facade.hpp: CF_11aRxVector::Reset, the error codes).  The shims are oracle/ref_shim.sh's,
# shared with build_ref_rx11a.sh; thread_if.h, which PHY_11a.hpp includes for bricks not compiled here, is an empty file.
#
# Compile flags, for MSVC semantics where GCC's differ:
#   ulong is `unsigned int` (entry.cpp): MSVC's unsigned long is 32 bits.  TBB11aFrameSink keeps its running CRC in a ulong and compares
#     ~crc32 with the 32-bit FCS; with a 64-bit ulong every frame would fail its FCS check.
#   -fwrapv: MSVC wraps signed overflow.  These bricks compute in unsigned or in int far from overflow; building with and without it gives
#     the same results on the whole corpus of tests/test_cpu_rx11n_reference.py.
#   -ffp-contract=off and no -mfma: GCC must not fuse float operations MSVC evaluates one by one (there are none in these bricks yet).
# A debug tap counts, per entry call, which branches the inputs reach (ref_rx11n_debug below).  _dump_text is the only hook the parsers
# give (SB_DUMP_TEXT_TAP): the HT-SIG stage reports its CRC-8 failure, its MCS refusal and its accepted fields through it.  The L-SIG /
# SIGNAL refusals print nothing, so the tap tells them apart by the fields the parser left (a rate of 0, a length over the limit) and
# otherwise by the input's reserved and tail bits.
# Nothing of the reference is copied into the repository.  TEST INFRASTRUCTURE ONLY.
#   usage: oracle/build_ref_rx11n.sh [reference root, default /root/reference]
set -e
REF="${1:-/root/reference}"
B11="$REF/kernel/bb/Brick11/src"
BINC="$REF/kernel/brick/inc"
CORE="$REF/kernel/core/inc"
HERE="$(cd "$(dirname "$0")" && pwd)"
[ -f "$B11/PHY_11n.hpp" ] || { echo "build_ref_rx11n: $B11/PHY_11n.hpp not found (fine outside the build container: the prebuilt oracle/_ref is used)"; exit 0; }
INC="$HERE/_ref/rx11n_inc"
rm -rf "$INC"
. "$HERE/ref_shim.sh"
ref_shim "$INC"
printf '#pragma once\n' > "$INC/thread_if.h"
# CRC8.h and CRC32.h include the core's const.h by a quoted name, which looks beside the including file first: they are reached through
# symbolic links in the shim directory (removed once the library is built), so that the shim's const.h is the one they find.
LINKS="CRC8.h CRC32.h"
for h in $LINKS; do ln -s "$CORE/$h" "$INC/$h"; done
# PHY_11a.hpp and PHY_11n.hpp also hold the transmit bricks and the rate demultiplexers, whose base classes (TDemux) the shim does not
# give.  The build reads the bricks it compiles out of them by a textual cut into the shim directory, removed once the library is built:
# PHY_11a.hpp from T11aPLCPParser's DEFINE_LOCAL_CONTEXT to the line before TBB11aRxRateSel's (T11aPLCPParser and TBB11aFrameSink), and
# PHY_11n.hpp from T11nSigParser's DEFINE_LOCAL_CONTEXT to its end.  The bodies are the headers' own; entry.cpp includes what the
# headers include before them.
sed -n '/^DEFINE_LOCAL_CONTEXT(T11aPLCPParser,/,/^DEFINE_LOCAL_CONTEXT(TBB11aRxRateSel,/p' "$B11/PHY_11a.hpp" | sed '$d' > "$INC/plcp11a.hpp"
sed -n '/^DEFINE_LOCAL_CONTEXT(T11nSigParser,/,$p' "$B11/PHY_11n.hpp" > "$INC/plcp11n.hpp"
grep -q 'class TBB11aFrameSink' "$INC/plcp11a.hpp" && grep -q 'class T11aPLCPParser' "$INC/plcp11a.hpp" && ! grep -q TDemux "$INC/plcp11a.hpp" \
  && grep -q 'class T11nSigParser' "$INC/plcp11n.hpp" || { echo "build_ref_rx11n: PHY_11a.hpp / PHY_11n.hpp cut did not apply" >&2; exit 1; }
cat > "$INC/entry.cpp" <<'ENTRY'
#include <stdint.h>
#include <string.h>
#include "const.h"
#define ulong unsigned int
#define ULONG unsigned int
#define PULONG unsigned int*
#define PUCHAR unsigned char*
#define UINT unsigned int
#define IN
#define OUT
#define SORA_EXTERN_C
#include "ieee80211facade.hpp"
#include "CRC32.h"
#include "ieee80211a_cmn.h"
#include "ieee80211n_cmn.h"
#include "CRC8.h"
#include "plcp11a.hpp"
#include "plcp11n.hpp"
#include "scramble.hpp"

namespace sbref {
// [0] L-SIG / SIGNAL refused at a reserved or tail bit, [1] at the parity, [2] at the rate nibble, [3] at the length limit (2500 bytes
// for 802.11a, 1500 for the L-SIG), [4] HT-SIG refused at its CRC-8, [5] at the MCS gate, [6] at its 1500-byte limit, [7] headers
// accepted, [8] frames whose FCS matched, [9] frames whose FCS did not.
static thread_local uint64_t counts[10];
static thread_local int htsig_said;       // the last HT-SIG message: 1 CRC-8 failed, 2 MCS refused, 3 fields accepted
}
void _dump_text(const char* fmt, ...) {
    if (strstr(fmt, "crc8 check failed")) sbref::htsig_said = 1;
    else if (strstr(fmt, "MCS index not supported")) sbref::htsig_said = 2;
    else if (strstr(fmt, "ht-sig : mcs")) sbref::htsig_said = 3;
}

// every facade the bricks below bind
struct Ctx : LOCAL_CONTEXT(T11aPLCPParser), LOCAL_CONTEXT(T11nSigParser), LOCAL_CONTEXT(T11aDesc), LOCAL_CONTEXT(TBB11aFrameSink) {
    // CF_HTRxVector has no Reset (ieee80211facade.hpp:269-272); the receiver's context is a static object (BB11nDemodCtx,
    // demod11/fb11ndemod_config.hpp:101), so it starts at zero
    Ctx() { ht_frame_mcs() = 0; ht_frame_length() = 0; CF_Error::error_code() = E_ERROR_SUCCESS; plcp_state() = CF_11RxPLCPSwitch::plcp_header; }
};

// the L-SIG / SIGNAL refusals, told apart for the tap (see the script header)
static void count_lsig_refusal(const Ctx& c, uint32_t word, unsigned max_len) {
    if ((word & 0xFFFFFF) & 0xFC0010) sbref::counts[0]++;
    else if (const_cast<Ctx&>(c).data_rate_kbps() == 0) sbref::counts[2]++;
    else if (const_cast<Ctx&>(c).frame_length() > max_len) sbref::counts[3]++;
    else sbref::counts[1]++;
}

extern "C" {
void ref_rx11n_debug_reset() { for (int k = 0; k < 10; k++) sbref::counts[k] = 0; }
// what the tap counted since the last ref_rx11n_debug_reset on this thread (see sbref::counts)
void ref_rx11n_debug(uint64_t out[10]) { for (int k = 0; k < 10; k++) out[k] = sbref::counts[k]; }

// T11aPLCPParser on each of n SIGNAL words, each from a context whose CF_11aRxVector, CF_11RxPLCPSwitch and CF_Error were just Reset
// (BB11aDemodContext::Reset after every event): 6 uint32 per word: plcp_state (1: accepted), error_code, data_rate_kbps, frame_length,
// total_symbols, code_rate
void ref_plcp11a_parse(const uint32_t* words, size_t n, uint32_t* out) {
    Ctx* ctx = new Ctx();
    T11aPLCPParser<Ctx>* b = new T11aPLCPParser<Ctx>(*ctx);
    TPinQueue<uint, 1, 1>* q = new TPinQueue<uint, 1, 1>();
    for (size_t i = 0; i < n; i++) {
        ctx->CF_11aRxVector::Reset(); ctx->CF_11RxPLCPSwitch::Reset(); ctx->CF_Error::error_code() = E_ERROR_SUCCESS;
        *q->append() = words[i];
        b->Process(*q);
        uint32_t* o = out + 6 * i;
        o[0] = (uint32_t)ctx->plcp_state(); o[1] = (uint32_t)ctx->error_code(); o[2] = ctx->data_rate_kbps(); o[3] = ctx->frame_length();
        o[4] = ctx->total_symbols(); o[5] = ctx->code_rate();
        if (o[0] == CF_11RxPLCPSwitch::plcp_data) sbref::counts[7]++; else count_lsig_refusal(*ctx, words[i], 2500);
    }
    delete q; delete b; delete ctx;
}
// T11nSigParser on n blocks of 9 bytes (what T11nViterbiSig hands it: the L-SIG's 3 then the HT-SIG's 6) in turn, through one context
// whose CF_11aRxVector and CF_Error are Reset before each block as after every event; CF_HTRxVector carries over.  8 uint32 per block:
// accepted, error_code, data_rate_kbps, frame_length, total_symbols, code_rate, ht_frame_mcs, ht_frame_length
void ref_sig11n_parse(const uint8_t* sig9, size_t n, uint32_t* out) {
    Ctx* ctx = new Ctx();
    T11nSigParser<Ctx>* b = new T11nSigParser<Ctx>(*ctx);
    TPinQueue<uchar, 9, 9>* q = new TPinQueue<uchar, 9, 9>();
    for (size_t i = 0; i < n; i++) {
        ctx->CF_11aRxVector::Reset(); ctx->CF_Error::error_code() = E_ERROR_SUCCESS;
        memcpy(q->append(), sig9 + 9 * i, 9);
        sbref::htsig_said = 0;
        bool ok = b->Process(*q);
        uint32_t* o = out + 8 * i;
        o[0] = ok; o[1] = (uint32_t)ctx->error_code(); o[2] = ctx->data_rate_kbps(); o[3] = ctx->frame_length(); o[4] = ctx->total_symbols();
        o[5] = ctx->code_rate(); o[6] = ctx->ht_frame_mcs(); o[7] = ctx->ht_frame_length();
        if (ok) sbref::counts[7]++;
        else if (sbref::htsig_said) sbref::counts[3 + sbref::htsig_said]++;
        else { uint32_t w; memcpy(&w, sig9 + 9 * i, 4); count_lsig_refusal(*ctx, w, 1500); }
    }
    delete q; delete b; delete ctx;
}
// T11aDesc -> TBB11aFrameSink, both fresh, for a frame of frame_length bytes, fed n decoded bytes one at a time as T11aViterbi hands
// them.  Returns CF_Error::error_code; *crc32 = CF_11aRxVector::crc32; out = the frame buffer (frame_length bytes)
uint32_t ref_desc_sink(const uint8_t* in, size_t n, uint16_t frame_length, uint8_t* out, uint32_t* crc32) {
    Ctx* ctx = new Ctx();
    // below 4 bytes, (ulong)(frame_length - 4) is huge and the sink stores every byte it is handed: room for all of them
    std::vector<uint8_t> buf(n + frame_length, 0);
    ctx->CF_RxFrameBuffer::Init(buf.data(), (uint)buf.size()); ctx->frame_length() = frame_length;
    typedef TBB11aFrameSink<Ctx> Sink;
    Sink* s = new Sink(*ctx);
    T11aDesc<Ctx, Sink>* d = new T11aDesc<Ctx, Sink>(*ctx, s);
    TPinQueue<uchar, 1, 1>* q = new TPinQueue<uchar, 1, 1>();
    for (size_t i = 0; i < n; i++) { *q->append() = in[i]; d->Process(*q); }
    uint32_t e = (uint32_t)ctx->error_code(); *crc32 = ctx->CF_11aRxVector::crc32(); memcpy(out, buf.data(), frame_length);
    if (e == E_ERROR_FRAME_OK) sbref::counts[8]++; else if (e == E_ERROR_CRC32_FAIL) sbref::counts[9]++;
    delete q; delete d; delete ctx;
    return e;
}
}
ENTRY
mkdir -p "$HERE/_ref"
rc=0
${CXX:-g++} -O2 -std=c++17 -fwrapv -ffp-contract=off -mssse3 -msse4.1 -fno-strict-aliasing -fno-operator-names -fpermissive -fPIC -shared \
  -fmax-errors=15 -w -DSB_DUMP_TEXT_TAP -I"$INC" -I"$B11" -I"$BINC" -I"$CORE" -I"$HERE/../sora_b200/brick" "$INC/entry.cpp" \
  -o "$HERE/_ref/librx11n_ref.so.tmp.$$" || rc=$?
for h in $LINKS plcp11a.hpp plcp11n.hpp; do rm -f "$INC/$h"; done
[ $rc -eq 0 ] || { rm -f "$HERE/_ref/librx11n_ref.so.tmp.$$"; echo "build_ref_rx11n: compile failed" >&2; exit 1; }
mv -f "$HERE/_ref/librx11n_ref.so.tmp.$$" "$HERE/_ref/librx11n_ref.so"
echo "build_ref_rx11n: oracle/_ref/librx11n_ref.so"
