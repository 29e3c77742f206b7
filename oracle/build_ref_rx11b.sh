#!/bin/sh
# oracle/_ref/librx11b_ref.so: the reference's 802.11b receiver, compiled from its own headers where they lie, brick by brick and as the
# whole graph CreateDemodGraph builds (kernel/bb/demod11/fb11bdemod_config.hpp:123-180):
#   TDCRemove, TDCEstimator (kernel/brick/inc/dc.hpp); TEnergyDetect (cca.hpp:11-98);
#   TSymTiming, TBarkerSync (symtiming.hpp:10-308); TBB11bDespread, TDBPSKDemap, TDQPSKDemap (barkerspread.hpp:227-451);
#   TSFDSync (sfd_sync.hpp); TCCK5P5Decoder, TCCK11Decoder (cck.hpp:9-764) with the demap_dqpsk_bits they call (core/inc/soradsp.h:190-199);
#   TDesc741 (scramble.hpp:93-162); TBB11bRxSwitch, TBB11bRxRateSel, TBB11bPlcpSwitch, TBB11bPlcpParser, TBB11bFrameSink
#   (PHY_11b.hpp:305-747) with CalcCRC16 (core/inc/CRC16.h) and CalcCRC32Incremental (core/inc/CRC32.h).
# The entry restates two things only, each citing the lines it restates: the graph wiring of CreateDemodGraph, and the driver loop of
# MAC11b_Receive (kernel/bb/demod11/fb11b_demod.cpp:26-79) with the TMemSamples source it pulls (kernel/brick/inc/memsource.hpp:87-151).
# The switches route through their own Process and Flush bodies.  The shims are oracle/ref_shim.sh's (TDemux among them).
#
# The width of `long`.  MSVC's long and unsigned long are 32 bits; GCC's on Linux are 64.  The bricks keep the CCK arg-max (cck.hpp:77,
# :144, :271-276) and the DQPSK decisions (barkerspread.hpp:434-438, soradsp.h:192-197) in long and cast to ulong before `>> 31`: with
# 64-bit types re + im never wraps and (ulong)(negative) >> 31 sets 33 bits, so the comparison would be meaningless at full scale.  So:
#   - ulong / ULONG / PULONG are `unsigned int`, as in build_ref_rx11n.sh;
#   - `long` is redefined around the brick includes only, after <immintrin.h>, <stdio.h>, <stdlib.h> and every shim header (a `#define
#     long int` before them would break `long long` in mmintrin.h), and #undef'd after them.  It is `int` around most headers, and
#     sbref::long32 around barkerspread.hpp and cck.hpp: a 4-byte int with the same arithmetic (wrapping + and -, >>=, conversions)
#     whose comparisons and sums feed the debug tap.  A static_assert inside each region checks that the type is 4 bytes.
# -fwrapv: MSVC wraps signed overflow (the CCK products and the DQPSK sums do at full scale).  -ffp-contract=off: as the other libraries.
# Textual cuts into the shim directory, removed once the library is built: PHY_11b.hpp (see below), cck.hpp up to its encoders (which need COMPLEX8 arithmetic the
# shim does not give), and soradsp.h's demap_dqpsk_bits (the rest of soradsp.h needs the radio stream headers).  The bodies are the
# headers' own.  CRC16.h, CRC32.h and dot11_plcp.h are reached through symbolic links, so that their quoted includes find the shims.
# A debug tap counts, per entry call, which edges the inputs reach (ref_rx11b_debug below).
# Nothing of the reference is copied into the repository.  TEST INFRASTRUCTURE ONLY.
#   usage: oracle/build_ref_rx11b.sh [reference root, default /root/reference]
set -e
REF="${1:-/root/reference}"
B11="$REF/kernel/bb/Brick11/src"
BINC="$REF/kernel/brick/inc"
CORE="$REF/kernel/core/inc"
HERE="$(cd "$(dirname "$0")" && pwd)"
[ -f "$B11/PHY_11b.hpp" ] || { echo "build_ref_rx11b: $B11/PHY_11b.hpp not found (fine outside the build container: the prebuilt oracle/_ref is used)"; exit 0; }
INC="$HERE/_ref/rx11b_inc"
rm -rf "$INC"
. "$HERE/ref_shim.sh"
ref_shim "$INC"
# bb/DataRate.h: the rate codes of kernel/inc/bb/bbb.h:47-50 it brings in, cut from there, and a declaration of the transmit side's
# Dot11BDataRate_Kbps2Code (DataRate.h:127; TBB11bSrc is not compiled into anything here)
{ printf '#pragma once\nunsigned char Dot11BDataRate_Kbps2Code(unsigned int kbps);\n'; grep '^#define DOT11B_PLCP_DATA_RATE_' "$REF/kernel/inc/bb/bbb.h"; } \
  > "$INC/bb/DataRate.h"
LINKS="CRC16.h CRC32.h dot11_plcp.h"
ln -s "$CORE/CRC16.h" "$INC/CRC16.h"; ln -s "$CORE/CRC32.h" "$INC/CRC32.h"; ln -s "$REF/kernel/inc/dot11_plcp.h" "$INC/dot11_plcp.h"
sed -n '1,/^const COMPLEX8 DQPSKEncode/p' "$B11/cck.hpp" | sed '$d' > "$INC/cck11b.hpp"
# PHY_11b.hpp whole, with one spelling changed: TBB11bRxSwitch::Reset calls `TDemux::Reset()` (:336), naming its dependent base by the
# injected class name, which MSVC resolves when the template is instantiated and GCC does not; the cut calls the same function
# through the base's typedef.
sed 's/^\([[:space:]]*\)TDemux::Reset();/\1this->TDemuxBase::Reset();/' "$B11/PHY_11b.hpp" > "$INC/phy11b.hpp"
{ printf '#pragma once\n#include "windef.h"\n#include "const.h"\n'; sed -n '/^FINL void demap_dqpsk_bits/,/^}/p' "$CORE/soradsp.h"; } > "$INC/soradsp.h"
grep -q 'TDemuxBase::Reset' "$INC/phy11b.hpp" && ! grep -q '[^>]TDemux::' "$INC/phy11b.hpp" && grep -q 'class TCCK11Decoder' "$INC/cck11b.hpp" && ! grep -q 'TCCK11Encode' "$INC/cck11b.hpp" && grep -q 're >>= 1' "$INC/soradsp.h" \
  || { echo "build_ref_rx11b: PHY_11b.hpp / cck.hpp / soradsp.h cut did not apply" >&2; exit 1; }
cat > "$INC/entry.cpp" <<'ENTRY'
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
// [0] CCK comparisons with an operand equal to INT_MIN (an L.re / L.im of INT_MIN, where -L wraps, reaches ABS and Max: cck.hpp:300-372),
// [1] CCK comparisons between equal values (arg-max ties: equal ABS1 / ABS2, or equal Max between hypotheses),
// [2] DQPSK (TDQPSKDemap) re or im that wrapped (the int products summed to 2^31), [3] DQPSK re + im or re - im that wrapped,
// [4] SFD found, [5] E_ERROR_SFD_FAIL, [6] E_ERROR_SFD_TIMEOUT, [7] E_ERROR_SYNC_TIMEOUT, [8] PLCP header refused at its CRC-16
// (E_ERROR_PLCP_HEADER_FAIL), [9] PLCP header accepted with a SIGNAL that is none of the four rates (rate 0, length 0: no verdict
// follows), [10] PLCP header accepted at a known rate with a frame length below 4 (the sink never reaches its verdict),
// [11] FCS matched (E_ERROR_FRAME_OK), [12] FCS failed (E_ERROR_CRC32_FAIL), [13] E_ERROR_CS_TIMEOUT.
static thread_local uint64_t counts[14];
void tap_pack(__m128i, int) {} void tap_zero(__m128i) {} void tap_clamp(__m128i, __m128i) {} void tap_madd(__m128i) {}
// MSVC's 32-bit long, as the tap sees it
struct long32 {
    int v;
    long32() = default;
    long32(int x) : v(x) { if (x == INT_MIN) counts[2]++; }          // `long re = ...`: a sum of two int16 products is INT_MIN only by wrapping
    long32& operator=(int x) { v = x; return *this; }
    long32& operator>>=(int n) { v >>= n; return *this; }
    operator int() const { return v; }
};
inline int operator+(long32 a, long32 b) { long long s = (long long)a.v + b.v; if (s != (int)s) counts[3]++; return (int)((unsigned)a.v + (unsigned)b.v); }
inline int operator-(long32 a, long32 b) { long long s = (long long)a.v - b.v; if (s != (int)s) counts[3]++; return (int)((unsigned)a.v - (unsigned)b.v); }
inline bool operator>(long32 a, long32 b) {
    if (a.v == INT_MIN || b.v == INT_MIN) counts[0]++;
    if (a.v == b.v) counts[1]++;
    return a.v > b.v;
}
}

#define ulong unsigned int
#define ULONG unsigned int
#define PULONG unsigned int*
#define SORA_EXTERN_C
#define long int
static_assert(sizeof(long) == 4 && sizeof(ulong) == 4, "MSVC's long and unsigned long are 32 bits");
#include "ieee80211facade.hpp"
#include "CRC32.h"
#include "dc.hpp"
#include "cca.hpp"
#include "symtiming.hpp"
#include "sfd_sync.hpp"
#include "scramble.hpp"
#include "phy11b.hpp"
#include "soradsp.h"
#undef long
#define long ::sbref::long32
static_assert(sizeof(long) == 4 && sizeof(ulong) == 4, "MSVC's long and unsigned long are 32 bits");
#include "barkerspread.hpp"
#include "cck11b.hpp"
#undef long

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

// Observation only, between TDCRemove and TBB11bRxSwitch: numbers the 4-sample vectors and notes the one during which TEnergyDetect
// raised cca_state (RaiseEvent(OnPowerDetected) binds CF_11CCA's empty handler through the brick's local context, cca.hpp:82).
struct VecTap { uint32_t count, detect; };
template<class T_CTX, class T_NEXT> class TVecTap : public TFilter<T_CTX, T_NEXT> {
    VecTap& tap;
public:
    DEFINE_IPORT(COMPLEX16, 4);
    DEFINE_OPORT(COMPLEX16, 4);
    TVecTap(T_CTX& ctx, T_NEXT* n) : TFilter<T_CTX, T_NEXT>(ctx, n), tap(ctx.vec_tap) {}
    void Reset() { this->Next()->Reset(); opin().clear(); }
    void Flush() { this->Next()->Flush(); }
    BOOL_FUNC_PROCESS(ipin) {
        while (ipin.check_read()) {
            memcpy(opin().append(), ipin.peek(), 4 * sizeof(COMPLEX16)); ipin.pop();
            tap.count++;
            const bool clear = this->ctx().cca_state() == CF_11CCA::power_clear;
            this->Next()->Process(opin());
            if (clear && this->ctx().cca_state() == CF_11CCA::power_detected) tap.detect = tap.count;
        }
        return true;
    }
};

// TDropAny (kernel/brick/inc/stdbrick.hpp) takes whatever it is handed and drops it
template<class T_CTX> class TDropAny : public TSink<T_CTX> {
public:
    DEFINE_IPORT(COMPLEX16, 4);
    explicit TDropAny(T_CTX& ctx) : TSink<T_CTX>(ctx) {}
    BOOL_FUNC_PROCESS(ipin) { ipin.clear(); return true; }
};

// BB11bDemodCtx (fb11bdemod_config.hpp:17-106): the facades every brick binds, reset() (:64-78) and init() (:80-100)
struct Ctx : LOCAL_CONTEXT(TBB11bFrameSink), LOCAL_CONTEXT(TBB11bPlcpParser), LOCAL_CONTEXT(TBB11bPlcpSwitch), LOCAL_CONTEXT(TDBPSKDemap),
             LOCAL_CONTEXT(TSFDSync), LOCAL_CONTEXT(TBB11bRxRateSel), LOCAL_CONTEXT(TEnergyDetect), LOCAL_CONTEXT(TDCEstimator),
             LOCAL_CONTEXT(TBB11bRxSwitch), LOCAL_CONTEXT(TDCRemove), LOCAL_CONTEXT(TCCK5P5Decoder), LOCAL_CONTEXT(TCCK11Decoder),
             LOCAL_CONTEXT(TDesc741), LOCAL_CONTEXT(TDQPSKDemap), LOCAL_CONTEXT(TBB11bDespread), LOCAL_CONTEXT(TBarkerSync),
             LOCAL_CONTEXT(TSymTiming) {
    VecTap vec_tap;
    std::vector<uint8_t> frame;
    Ctx(size_t frame_cap) : frame(frame_cap, 0) {
        CF_RxFrameBuffer::rx_frame_buf() = frame.data(); CF_RxFrameBuffer::rx_frame_buf_size() = (uint)frame.size();
        set_zero(CF_VecDC::direct_current());
        cca_pwr_threshold() = 1000 * 1000;
        last_symbol().re = last_symbol().im = 0; byte_reg() = 0;
        frame_length() = 0; data_rate_kbps() = 0; CF_11bRxVector::crc32() = 0;
        vec_tap.count = vec_tap.detect = 0;
        reset();
    }
    void reset() {
        CF_Error::error_code() = E_ERROR_SUCCESS; CF_11CCA::cca_state() = CF_11CCA::power_clear;
        rxrate_state() = CF_11bRxMRSel::rate_sync; plcp_state() = CF_11RxPLCPSwitch::plcp_header;
    }
};

// CreateDemodGraph (fb11bdemod_config.hpp:123-180) below TMemSamples, with the vector tap between dc and rxswt
struct Graph {
    Ctx& ctx; IReferenceCounting* root; std::function<void(const COMPLEX16*)> push; std::function<void()> flush, reset;
};
static Graph* make_graph(Ctx& BB11bDemodCtx) {
    CREATE_BRICK_SINK  (drop, TDropAny, BB11bDemodCtx);
    CREATE_BRICK_SINK  (plcphdr, TBB11bPlcpParser, BB11bDemodCtx);
    CREATE_BRICK_SINK  (mpdu, TBB11bFrameSink, BB11bDemodCtx);
    CREATE_BRICK_DEMUX2(plcpswt, TBB11bPlcpSwitch, BB11bDemodCtx, plcphdr, mpdu);
    CREATE_BRICK_FILTER(dsc741, TDesc741, BB11bDemodCtx, plcpswt);
    CREATE_BRICK_FILTER(cck11, TCCK11Decoder, BB11bDemodCtx, dsc741);
    CREATE_BRICK_FILTER(cck5p5, TCCK5P5Decoder, BB11bDemodCtx, dsc741);
    CREATE_BRICK_FILTER(dqpsk, TDQPSKDemap, BB11bDemodCtx, dsc741);
    CREATE_BRICK_FILTER(despread_dqpsk, TBB11bDespread, BB11bDemodCtx, dqpsk);
    CREATE_BRICK_FILTER(dbpsk, TDBPSKDemap, BB11bDemodCtx, dsc741);
    CREATE_BRICK_FILTER(despread_dbpsk, TBB11bDespread, BB11bDemodCtx, dbpsk);
    CREATE_BRICK_SINK  (sfdsync, TSFDSync, BB11bDemodCtx);
    CREATE_BRICK_FILTER(despread_sfd, TBB11bDespread, BB11bDemodCtx, sfdsync);
    CREATE_BRICK_DEMUX5(mrsel, TBB11bRxRateSel, BB11bDemodCtx, despread_sfd, despread_dbpsk, despread_dqpsk, cck5p5, cck11);
    CREATE_BRICK_FILTER(bsync, TBarkerSync, BB11bDemodCtx, mrsel);
    CREATE_BRICK_FILTER(symtime, TSymTiming, BB11bDemodCtx, bsync);
    CREATE_BRICK_FILTER(dcest, TDCEstimator, BB11bDemodCtx, drop);
    CREATE_BRICK_FILTER(pwrdet, TEnergyDetect, BB11bDemodCtx, dcest);
    CREATE_BRICK_DEMUX2(rxswt, TBB11bRxSwitch, BB11bDemodCtx, pwrdet, symtime);
    CREATE_BRICK_FILTER(vtap, TVecTap, BB11bDemodCtx, rxswt);
    CREATE_BRICK_FILTER(dc, TDCRemove, BB11bDemodCtx, vtap);
    IReferenceCounting::AddRef(dc);
    typedef TPinQueue<COMPLEX16, 28, 28> Q;     // TMemSamples' DEFINE_OPORT(COMPLEX16, 28) into TDCRemove's DEFINE_IPORT(COMPLEX16, 28)
    std::shared_ptr<Q> q(new Q());
    Graph* g = new Graph{BB11bDemodCtx, dc};
    g->push = [dc, q](const COMPLEX16* s) { memcpy(q->append(), s, 28 * sizeof(COMPLEX16)); dc->Process(*q); };
    g->flush = [dc]() { dc->Flush(); };
    g->reset = [dc, q]() { q->clear(); dc->Reset(); };
    return g;
}

struct Event { uint32_t status, rate_kbps, length, crc32, sample_index, detect_vec; };

// MAC11b_Receive (fb11b_demod.cpp:26-79) over one capture of n samples from a fresh context (init(), fb11bdemod_config.hpp:80-100), up to
// max_events events other than E_ERROR_CS_TIMEOUT.  TMemSamples::Process (memsource.hpp:87-114) hands the graph one 28-sample block per
// call; the driver polls error_code after each; on an event it Seeks past the last FCS byte after FRAME_OK / CRC32_FAIL (:46-64; Seek
// rounds up to a multiple of 4 and stops at the end, memsource.hpp:136-149), then Flush(), ctx.reset(), Reset() (:66-68).  The capture
// ends at its last whole block: TMemSamples would hand on a shorter tail padded with whatever its pin queue last held.
static int run_chain(const int16_t* iq, size_t n, Event* ev, uint8_t* out, size_t out_stride, int max_events) {
    Ctx* ctx = new Ctx(n / 32 + 65536 + 64);      // the sink writes without a bound (PHY_11b.hpp:714-722): room for every byte a capture can hold
    Graph* g = make_graph(*ctx);
    g->reset();
    const COMPLEX16* s = (const COMPLEX16*)iq;
    size_t pos = 0; uint32_t sample_index = 0; int ne = 0;
    std::vector<COMPLEX16> blk(28);
    while (pos + 28 <= n && ne < max_events) {
        memcpy(blk.data(), s + pos, 28 * sizeof(COMPLEX16)); pos += 28; sample_index += 28;
        g->push(blk.data());
        ulong err = ctx->CF_Error::error_code();
        if (err == E_ERROR_SUCCESS) continue;
        switch (err) {
        case E_ERROR_SFD_FAIL: sbref::counts[5]++; break;          case E_ERROR_SFD_TIMEOUT: sbref::counts[6]++; break;
        case E_ERROR_SYNC_TIMEOUT: sbref::counts[7]++; break;      case E_ERROR_PLCP_HEADER_FAIL: sbref::counts[8]++; break;
        case E_ERROR_FRAME_OK: sbref::counts[11]++; break;         case E_ERROR_CRC32_FAIL: sbref::counts[12]++; break;
        case E_ERROR_CS_TIMEOUT: sbref::counts[13]++; break;
        }
        if (err != E_ERROR_CS_TIMEOUT) {
            Event& e = ev[ne];
            e.status = err; e.rate_kbps = ctx->data_rate_kbps(); e.length = ctx->frame_length();
            e.crc32 = ctx->CF_11bRxVector::crc32() & 0x00FFFFFFu;   // the sink reads 4 bytes; the 4th is the buffer's previous content
            e.sample_index = sample_index; e.detect_vec = ctx->vec_tap.detect;
            if (out) { size_t nb = ctx->frame_length() < out_stride ? ctx->frame_length() : out_stride; memcpy(out + (size_t)ne * out_stride, ctx->frame.data(), nb); }
            ne++;
        }
        if (err == E_ERROR_FRAME_OK || err == E_ERROR_CRC32_FAIL) {
            uint32_t off = 0;
            switch (ctx->data_rate_kbps()) { case 1000: off = 8 * 11 * 4; break; case 2000: off = 4 * 11 * 4; break;
                                             case 5500: off = 8 * 2 * 4; break; case 11000: off = 8 * 1 * 4; break; }
            off = (off + 3) / 4 * 4; if (off > n - pos) off = (uint32_t)(n - pos);
            pos += off; sample_index += off;
        }
        g->flush();
        ctx->reset();
        g->reset();
    }
    IReferenceCounting::Release(g->root); delete g; delete ctx;
    return ne;
}

// one brick on its own: a fresh context, the inputs pushed burst by burst, every output byte kept
template<template<class, class> class B, size_t NI>
static void run_decoder(const int16_t* chips, size_t nburst, int16_t last_re, int16_t last_im, uint8_t* out, int16_t* last_out) {
    Ctx* ctx = new Ctx(16);
    ctx->last_symbol().re = last_re; ctx->last_symbol().im = last_im;
    typedef typename Cap<uchar, 1>::template Sink<Ctx> S;
    S* s = new S(*ctx);
    B<Ctx, S>* f = new B<Ctx, S>(*ctx, s);
    TPinQueue<COMPLEX16, NI, NI>* q = new TPinQueue<COMPLEX16, NI, NI>();
    for (size_t i = 0; i < nburst; i++) { memcpy(q->append(), chips + 2 * NI * i, NI * sizeof(COMPLEX16)); f->Process(*q); }
    memcpy(out, s->got.data(), s->got.size());
    last_out[0] = ctx->last_symbol().re; last_out[1] = ctx->last_symbol().im;
    delete q; delete f; delete ctx;
}

extern "C" {
void ref_rx11b_debug_reset() { for (int k = 0; k < 14; k++) sbref::counts[k] = 0; }
// what the tap counted since the last ref_rx11b_debug_reset on this thread (see sbref::counts)
void ref_rx11b_debug(uint64_t out[14]) { for (int k = 0; k < 14; k++) out[k] = sbref::counts[k]; }

// TCCK11Decoder (one instance: is_even runs from 0 across the symbols) on nsym symbols of 8 chips; one byte per symbol.  last = the
// CF_DifferentialDemap::last_symbol before / after
void ref_cck11_decode(const int16_t* chips, size_t nsym, const int16_t* last, uint8_t* out, int16_t* last_out) {
    run_decoder<TCCK11Decoder, 8>(chips, nsym, last[0], last[1], out, last_out);
}
// TCCK5P5Decoder on nbyte bytes of 16 chips
void ref_cck5_decode(const int16_t* chips, size_t nbyte, const int16_t* last, uint8_t* out, int16_t* last_out) {
    run_decoder<TCCK5P5Decoder, 16>(chips, nbyte, last[0], last[1], out, last_out);
}
// TDQPSKDemap on nbyte bytes of 4 symbols, TDBPSKDemap on nbyte bytes of 8 symbols
void ref_dqpsk_demap(const int16_t* sym, size_t nbyte, const int16_t* last, uint8_t* out, int16_t* last_out) {
    run_decoder<TDQPSKDemap, 4>(sym, nbyte, last[0], last[1], out, last_out);
}
void ref_dbpsk_demap(const int16_t* sym, size_t nbyte, const int16_t* last, uint8_t* out, int16_t* last_out) {
    run_decoder<TDBPSKDemap, 8>(sym, nbyte, last[0], last[1], out, last_out);
}
// TBB11bDespread on nsym blocks of 11 chips: one symbol each
void ref_despread(const int16_t* chips, size_t nsym, int16_t* out) {
    Ctx* ctx = new Ctx(16);
    typedef Cap<COMPLEX16, 1>::Sink<Ctx> S;
    S* s = new S(*ctx);
    TBB11bDespread<Ctx, S>* f = new TBB11bDespread<Ctx, S>(*ctx, s);
    TPinQueue<COMPLEX16, 11, 11>* q = new TPinQueue<COMPLEX16, 11, 11>();
    for (size_t i = 0; i < nsym; i++) { memcpy(q->append(), chips + 22 * i, 11 * sizeof(COMPLEX16)); f->Process(*q); }
    memcpy(out, s->got.data(), s->got.size() * sizeof(COMPLEX16));
    delete q; delete f; delete ctx;
}
// TBB11bPlcpParser on n 6-byte headers in turn through one context whose CF_Error and CF_11RxPLCPSwitch are reset before each (as after
// every event); CF_11bRxVector and CF_11bRxMRSel carry over (CF_11bRxVector has no Reset, ieee80211facade.hpp:72-76).  prev = the
// rxrate_state, data_rate_kbps and frame_length before the first.  5 uint32 per header: error_code, plcp_state, rxrate_state,
// data_rate_kbps, frame_length
void ref_plcp11b_parse(const uint8_t* hdr6, size_t n, const uint32_t* prev, uint32_t* out) {
    Ctx* ctx = new Ctx(16);
    ctx->rxrate_state() = (CF_11bRxMRSel::RxRateState)prev[0]; ctx->data_rate_kbps() = prev[1]; ctx->frame_length() = (ushort)prev[2];
    TBB11bPlcpParser<Ctx>* b = new TBB11bPlcpParser<Ctx>(*ctx);
    TPinQueue<uchar, 6, 6>* q = new TPinQueue<uchar, 6, 6>();
    for (size_t i = 0; i < n; i++) {
        ctx->CF_Error::error_code() = E_ERROR_SUCCESS; ctx->plcp_state() = CF_11RxPLCPSwitch::plcp_header;
        memcpy(q->append(), hdr6 + 6 * i, 6);
        b->Process(*q);
        uint32_t* o = out + 5 * i;
        o[0] = ctx->error_code(); o[1] = ctx->plcp_state(); o[2] = ctx->rxrate_state(); o[3] = ctx->data_rate_kbps(); o[4] = ctx->frame_length();
        if (o[0] == E_ERROR_PLCP_HEADER_FAIL) sbref::counts[8]++;
        else if (o[3] == 0) sbref::counts[9]++;
        else if (o[4] < 4) sbref::counts[10]++;
    }
    delete q; delete b; delete ctx;
}
// TDesc741 -> TBB11bFrameSink, both fresh, CF_Descramber::byte_reg = seed, for a frame of frame_length bytes fed n scrambled bytes one
// at a time.  Returns error_code; *crc32 = the sink's frame_crc32 (low 24 bits); *consumed = bytes handed on before the sink's verdict;
// out = the frame buffer (frame_length bytes)
uint32_t ref_desc_sink(const uint8_t* in, size_t n, uint8_t seed, uint16_t frame_length, uint8_t* out, uint32_t* crc32) {
    Ctx* ctx = new Ctx(n + frame_length + 16);
    ctx->byte_reg() = seed; ctx->frame_length() = frame_length;
    typedef TBB11bFrameSink<Ctx> Sink;
    Sink* s = new Sink(*ctx);
    TDesc741<Ctx, Sink>* d = new TDesc741<Ctx, Sink>(*ctx, s);
    TPinQueue<uchar, 1, 1>* q = new TPinQueue<uchar, 1, 1>();
    for (size_t i = 0; i < n; i++) { *q->append() = in[i]; d->Process(*q); }
    uint32_t e = ctx->error_code(); *crc32 = ctx->CF_11bRxVector::crc32() & 0x00FFFFFFu; memcpy(out, ctx->frame.data(), frame_length);
    if (e == E_ERROR_FRAME_OK) sbref::counts[11]++; else if (e == E_ERROR_CRC32_FAIL) sbref::counts[12]++;
    delete q; delete d; delete ctx;
    return e;
}
// the whole chain (run_chain above) on one capture of n int16 pairs: 6 uint32 per event (status, rate_kbps, length, crc32, sample_index,
// detect_vec), frame bytes at out + k * out_stride.  Returns the number of events
int ref_rx11b_run(const int16_t* iq, size_t n, uint32_t* ev, uint8_t* out, size_t out_stride, int max_events) {
    return run_chain(iq, n, (Event*)ev, out, out_stride, max_events);
}
}
ENTRY
mkdir -p "$HERE/_ref"
rc=0
${CXX:-g++} -O2 -std=c++17 -fwrapv -ffp-contract=off -mssse3 -msse4.1 -fno-strict-aliasing -fno-operator-names -fpermissive -fPIC -shared \
  -fmax-errors=15 -w -include functional -include memory -I"$INC" -I"$B11" -I"$BINC" -I"$CORE" -I"$HERE/../sora_b200/brick" "$INC/entry.cpp" \
  -o "$HERE/_ref/librx11b_ref.so.tmp.$$" || rc=$?
for h in $LINKS phy11b.hpp cck11b.hpp soradsp.h; do rm -f "$INC/$h"; done
[ $rc -eq 0 ] || { rm -f "$HERE/_ref/librx11b_ref.so.tmp.$$"; echo "build_ref_rx11b: compile failed" >&2; exit 1; }
mv -f "$HERE/_ref/librx11b_ref.so.tmp.$$" "$HERE/_ref/librx11b_ref.so"
echo "build_ref_rx11b: oracle/_ref/librx11b_ref.so"
