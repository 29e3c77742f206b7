#!/bin/sh
# oracle/_ref/librx11a_ref.so: the reference's 802.11a receive front end behind the carrier sense, compiled from its own headers where they
# lie and driven brick by brick from a fresh context:
#   T11aLTS (kernel/bb/Brick11/src/channel_11a.hpp:23-230) with FreqOffsetEstimate, BuildFrequencyShiftCoeffs and FrequencyShift
#     (kernel/brick/inc/dspalg.hpp:200-243) and uatan2 / ucos / usin (kernel/core/inc/intalg.h, intalglut.h);
#   per symbol TFreqCompensation and TChannelEqualization (channel_11a.hpp:532-653), TFFT64 (fft.hpp:106-135, FFT<64> of fft_r4dif.h),
#     TPhaseCompensate (freqoffset.hpp), TPilotTrack with its PilotSgn (pilot.hpp:10-28, 121-269);
#   soft bits T11aDemap<1,2,4,6> (demapper11a.hpp, demapper.h with demap_limit<64> and the LUTs), T11aDeinterleaveBPSK / QPSK / QAM16 /
#     QAM64 (deinterleaver.hpp);
#   TDownSample44_40 with Down44to40 (sampling.hpp:33-65, 44MTo40M.hpp);
#   the carrier sense: TDownSample2 (samples.hpp:27-49), TDCRemoveEx<4> and TDCEstimator (kernel/brick/inc/dc.hpp), TCCA11a (cca.hpp:106-441)
#     with CMovingWindow / CAccumulator (dspalg.hpp:5-100) and Generate80211aSTS (sequence.h).
# Nothing of these bricks is restated: their bodies, the facades (ieee80211facade.hpp, kernel/brick/inc/stdfacade.h, so CompCoeffs = 0x7fff
# and symbol_count = 127 come from source), the tables and the integer trigonometry all come from the reference tree.
#
# Include order: the shim directory first, then Brick11/src, kernel/brick/inc and kernel/core/inc.  Quoted includes look beside the
# including file first, so demapper11a.hpp, sampling.hpp and 44MTo40M.hpp are reached through symbolic links in the shim directory
# (removed once the library is built), which lets their quoted includes find the shims.  The shims are oracle/ref_shim.sh's, shared
# with build_ref_rx11n.sh, plus 40MTo44M.hpp: a declaration of up40to44 only.
# A debug tap counts, per entry call, what the edges of these bricks reach (ref_rx11a_debug below): LTS bins whose |Y|^2 >> 8 is 0 (the
# channel estimate's e == 0 branch), channel-estimate packs that wrap, equaliser packs that wrap, mul(vcs, vcs) packs that wrap (the
# rotations of TFreqCompensation, TPhaseCompensate and TPilotTrack), demap_limit lanes that smax / smin clamp, and pmaddwd sums that wrap.
# Nothing of the reference is copied into the repository.  TEST INFRASTRUCTURE ONLY.
#   usage: oracle/build_ref_rx11a.sh [reference root, default /root/reference]
set -e
REF="${1:-/root/reference}"
B11="$REF/kernel/bb/Brick11/src"
BINC="$REF/kernel/brick/inc"
CORE="$REF/kernel/core/inc"
HERE="$(cd "$(dirname "$0")" && pwd)"
[ -f "$B11/channel_11a.hpp" ] || { echo "build_ref_rx11a: $B11/channel_11a.hpp not found (fine outside the build container: the prebuilt oracle/_ref is used)"; exit 0; }
INC="$HERE/_ref/rx11a_inc"
rm -rf "$INC"
. "$HERE/ref_shim.sh"
ref_shim "$INC"
printf '#pragma once\nvoid up40to44(const COMPLEX16*, COMPLEX16*);\n' > "$INC/40MTo44M.hpp"
cat > "$INC/entry.cpp" <<'ENTRY'
#include <stdint.h>
#include "ieee80211facade.hpp"
#include "channel_11a.hpp"
#include "freqoffset.hpp"
#include "fft.hpp"
#include "pilot.hpp"
#include "demapper11a.hpp"
#include "deinterleaver.hpp"
template<> void DemapperCore::Demap<1>(const COMPLEX16& input, uchar* output) { Demap_1(input, output); }
template<> void DemapperCore::Demap<2>(const COMPLEX16& input, uchar* output) { Demap_2(input, output); }
template<> void DemapperCore::Demap<4>(const COMPLEX16& input, uchar* output) { Demap_4(input, output); }
template<> void DemapperCore::Demap<6>(const COMPLEX16& input, uchar* output) { Demap_6(input, output); }
#include "sampling.hpp"
#include "samples.hpp"
#include "dc.hpp"
#include "cca.hpp"

namespace sbref {
// [0] LTS bins whose |Y|^2 >> 8 is 0 (T11aLTS's e == 0 branch), [1] channel-estimate pack lanes outside int16 (the pack wraps them),
// [2] equaliser pack lanes outside int16, [3] mul(vcs, vcs) lanes whose >> 15 lies outside int16, [4] demap_limit lanes smax / smin
// clamped, [5] pmaddwd lanes that wrapped (both products 2^30).  `phase` says which brick runs: 0 the LTS, 1 the symbol bricks.
static thread_local uint64_t counts[6];
int phase;
static inline unsigned lanes16(__m128i ne) { return (unsigned)__builtin_popcount((unsigned)_mm_movemask_epi8(ne)) / 2; }
static inline unsigned lanes32(__m128i ne) { return (unsigned)__builtin_popcount((unsigned)_mm_movemask_epi8(ne)) / 4; }
void tap_pack(__m128i v, int k) {
    unsigned n = 4 - lanes32(_mm_cmpeq_epi32(v, _mm_srai_epi32(_mm_slli_epi32(v, 16), 16)));
    counts[k ? 3 : phase ? 2 : 1] += n;
}
void tap_zero(__m128i v) { if (phase == 0) counts[0] += lanes32(_mm_cmpeq_epi32(v, _mm_setzero_si128())); }
void tap_clamp(__m128i r, __m128i a) { counts[4] += 8 - lanes16(_mm_cmpeq_epi16(r, a)); }
void tap_madd(__m128i v) { counts[5] += lanes32(_mm_cmpeq_epi32(v, _mm_set1_epi32(INT32_MIN))); }
}

// every facade the bricks below bind, as BB11aDemodContext composes them (kernel/bb/demod11/fb11ademod_config.hpp)
struct Ctx : LOCAL_CONTEXT(T11aLTS), LOCAL_CONTEXT(TFreqCompensation), LOCAL_CONTEXT(TFFT64), LOCAL_CONTEXT(TChannelEqualization),
             LOCAL_CONTEXT(TPhaseCompensate), LOCAL_CONTEXT(TPilotTrack), LOCAL_CONTEXT(T11aDemap), LOCAL_CONTEXT(T11aDeinterleaveBPSK),
             LOCAL_CONTEXT(T11aDeinterleaveQPSK), LOCAL_CONTEXT(T11aDeinterleaveQAM16), LOCAL_CONTEXT(T11aDeinterleaveQAM64),
             LOCAL_CONTEXT(TDownSample44_40), LOCAL_CONTEXT(TDownSample2), LOCAL_CONTEXT(TDCRemoveEx), LOCAL_CONTEXT(TCCA11a),
             LOCAL_CONTEXT(TDCEstimator) {
    // BB11aDemodContext::Reset (fb11ademod_config.hpp:68-94), the facades the bricks here bind; CF_VecDC as its own Reset leaves it
    Ctx() {
        CF_Channel_11a::Reset(); CF_FreqCompensate::Reset(); CF_PhaseCompensate::Reset(); CF_PilotTrack::Reset();
        CF_11aSymState::Reset(); CF_CFOffset::Reset(); CF_11aRxVector::Reset(); CF_VecDC::Reset();
        CF_Error::error_code() = E_ERROR_SUCCESS; CF_11CCA::Reset();     // ResetCarrierSense (:96-102)
    }
};

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

// one burst of NI through brick B (a fresh instance: the bricks here keep their state in the context), its NO outputs copied to out
template<template<class, class> class B, class TI, size_t NI, class TO, size_t NO>
static void step(Ctx& ctx, const TI* in, TO* out) {
    typedef typename Cap<TO, NO>::template Sink<Ctx> S;
    S* s = new S(ctx);
    B<Ctx, S>* f = new B<Ctx, S>(ctx, s);
    TPinQueue<TI, NI, NI>* q = new TPinQueue<TI, NI, NI>();
    memcpy(q->append(), in, NI * sizeof(TI));
    f->Process(*q);
    memcpy(out, s->got.data(), NO * sizeof(TO));
    delete q; delete f;
}
template<class C, class N> using Demap1 = T11aDemap<1>::Filter<C, N>;
template<class C, class N> using Demap2 = T11aDemap<2>::Filter<C, N>;
template<class C, class N> using Demap4 = T11aDemap<4>::Filter<C, N>;
template<class C, class N> using Demap6 = T11aDemap<6>::Filter<C, N>;

static void lts(Ctx& ctx, const int16_t* lts144) {
    sbref::phase = 0;
    T11aLTS<Ctx>* b = new T11aLTS<Ctx>(ctx);
    TPinQueue<COMPLEX16, 144, 144>* q = new TPinQueue<COMPLEX16, 144, 144>();
    memcpy(q->append(), lts144, 144 * sizeof(COMPLEX16));
    b->Process(*q);
    delete q; delete b;
}

extern "C" {
// T11aLTS on the 144 samples T11aSymSelEx hands it (the CP of the LTS pair then two LTS), from a fresh context:
// CFO_est, FreqCoeffs [64][2], ChannelCoeffs [64][2]
void ref_rx11a_lts(const int16_t* lts144, int16_t* cfo_est, int16_t* freq, int16_t* chan) {
    for (int k = 0; k < 6; k++) sbref::counts[k] = 0;
    Ctx* ctx = new Ctx();
    lts(*ctx, lts144);
    *cfo_est = ctx->CFO_est(); memcpy(freq, ctx->Coeffs(), 256); memcpy(chan, ctx->ChannelCoeffs(), 256);
    delete ctx;
}
// T11aLTS on lts144, then n 80-sample symbol blocks (the CP and the symbol, as T11aDataSymbol is handed them; it skips skip_cp = 8,
// PHY_11a.hpp:365, 391) through TFreqCompensation, TFFT64, TChannelEqualization, TPhaseCompensate, TPilotTrack, the demapper and the
// de-interleaver.  Symbol 0 is SIGNAL (BPSK); the rest use the modulation of rate_kbps.  Per symbol: fft_in (TFreqCompensation's
// output), fft_out, equalized, phase_comp, tracked [64][2]; demapped and soft [288] (the first N_CBPS meaningful); state: CFO_comp,
// SFO_comp, CFO_tracker, SFO_tracker, symbol_count after the symbol.  Returns 0, or -1 for an unknown rate.
int ref_rx11a_symbols(const int16_t* lts144, size_t n, const int16_t* sym80, unsigned rate_kbps, int16_t* cfo_est, int16_t* freq,
                      int16_t* chan, int16_t* fft_in, int16_t* fft_out, int16_t* equalized, int16_t* phase_comp, int16_t* tracked,
                      uint8_t* demapped, uint8_t* soft, int32_t* state) {
    int nbpsc;
    switch (rate_kbps) { case 6000: case 9000: nbpsc = 1; break; case 12000: case 18000: nbpsc = 2; break;
                         case 24000: case 36000: nbpsc = 4; break; case 48000: case 54000: nbpsc = 6; break; default: return -1; }
    for (int k = 0; k < 6; k++) sbref::counts[k] = 0;
    Ctx* ctx = new Ctx();
    lts(*ctx, lts144);
    *cfo_est = ctx->CFO_est(); memcpy(freq, ctx->Coeffs(), 256); memcpy(chan, ctx->ChannelCoeffs(), 256);
    sbref::phase = 1;
    for (size_t s = 0; s < n; s++) {
        COMPLEX16* fi = (COMPLEX16*)(fft_in + 128 * s); COMPLEX16* fo = (COMPLEX16*)(fft_out + 128 * s);
        COMPLEX16* eq = (COMPLEX16*)(equalized + 128 * s); COMPLEX16* pc = (COMPLEX16*)(phase_comp + 128 * s);
        COMPLEX16* tr = (COMPLEX16*)(tracked + 128 * s);
        uint8_t* dm = demapped + 288 * s; uint8_t* so = soft + 288 * s;
        memset(dm, 0, 288); memset(so, 0, 288);
        step<TFreqCompensation, COMPLEX16, 64, COMPLEX16, 64>(*ctx, (const COMPLEX16*)(sym80 + 160 * s) + 8, fi);
        step<TFFT64, COMPLEX16, 64, COMPLEX16, 64>(*ctx, fi, fo);
        step<TChannelEqualization, COMPLEX16, 64, COMPLEX16, 64>(*ctx, fo, eq);
        step<TPhaseCompensate, COMPLEX16, 64, COMPLEX16, 64>(*ctx, eq, pc);
        step<TPilotTrack, COMPLEX16, 64, COMPLEX16, 64>(*ctx, pc, tr);
        switch (s == 0 ? 1 : nbpsc) {
        case 1: step<Demap1, COMPLEX16, 64, uchar, 48>(*ctx, tr, dm); step<T11aDeinterleaveBPSK, uchar, 48, uchar, 48>(*ctx, dm, so); break;
        case 2: step<Demap2, COMPLEX16, 64, uchar, 96>(*ctx, tr, dm); step<T11aDeinterleaveQPSK, uchar, 96, uchar, 96>(*ctx, dm, so); break;
        case 4: step<Demap4, COMPLEX16, 64, uchar, 192>(*ctx, tr, dm); step<T11aDeinterleaveQAM16, uchar, 192, uchar, 192>(*ctx, dm, so); break;
        default: step<Demap6, COMPLEX16, 64, uchar, 288>(*ctx, tr, dm); step<T11aDeinterleaveQAM64, uchar, 288, uchar, 288>(*ctx, dm, so);
        }
        int32_t* st = state + 5 * s;
        st[0] = ctx->CFO_comp(); st[1] = ctx->SFO_comp(); st[2] = ctx->CFO_tracker(); st[3] = ctx->SFO_tracker(); st[4] = (int32_t)ctx->symbol_count();
    }
    delete ctx;
    return 0;
}
// TDownSample44_40 (one Down44to40 across the stream) fed floor(n / 28) blocks of 28 samples at 44 Msps; returns the 40 Msps samples
// it emitted (whole 28-sample blocks), written to out (room for n samples)
size_t ref_resample_44_40(const int16_t* in, size_t n, int16_t* out) {
    typedef Cap<COMPLEX16, 28>::Sink<Ctx> S;
    Ctx* ctx = new Ctx();
    S* s = new S(*ctx);
    TDownSample44_40<Ctx, S>* f = new TDownSample44_40<Ctx, S>(*ctx, s);
    TPinQueue<COMPLEX16, 28, 28>* q = new TPinQueue<COMPLEX16, 28, 28>();
    for (size_t b = 0; b + 28 <= n; b += 28) { memcpy(q->append(), in + 2 * b, 28 * sizeof(COMPLEX16)); f->Process(*q); }
    size_t m = s->got.size();
    memcpy(out, s->got.data(), m * sizeof(COMPLEX16));
    delete q; delete f; delete ctx;
    return m;
}
// The carrier-sense end of CreateDemodGraph11a_40M (fb11ademod_config.hpp:220-229): TDownSample2 -> TDCRemoveEx<4> -> TCCA11a ->
// TDCEstimator, fed n 40 Msps samples in TMemSamples' 28-sample blocks.  TBB11bRxSwitch hands TDCRemoveEx each 20 Msps vector while
// cca_state is power_clear; the first vector after power_detected would go to the demodulation branch, so the run stops there.  After
// each block an E_ERROR_CS_TIMEOUT is handled as RxThread does (fb11a_demod.cpp:47-50): ResetCarrierSense, then the carrier-sense
// graph's Reset (TCCA11a and TDCEstimator re-initialise; CF_VecDC keeps the DC).  Per vector handed to TDCRemoveEx, 13 int32 after it:
// cca_state, error_code, DC as 8 int16 lanes, cca_peak_index, cca_pwr_reading, the 20 Msps index of the vector.  Returns the number
// of vectors recorded (at most max_vec); *detect is the 20 Msps index of the first vector past the detection, or -1.
}
static const int CS_REC = 13;
struct CsState { Ctx* ctx; int32_t* rec; size_t nrec, max_vec; uint32_t vec20; bool done; };
template<class T_CTX, class T_DC> class CsSwitch : public TSink<T_CTX> {
public:
    DEFINE_IPORT(COMPLEX16, 4);
    T_DC* dc; CsState* st;
    CsSwitch(T_CTX& ctx, T_DC* d, CsState* s) : TSink<T_CTX>(ctx), dc(d), st(s) {}
    BOOL_FUNC_PROCESS(ipin) {
        while (ipin.check_read()) {
            Ctx& c = *st->ctx;
            if (!st->done && c.cca_state() == CF_11CCA::power_clear) {
                TPinQueue<COMPLEX16, 4, 4> q; memcpy(q.append(), ipin.peek(), 16); dc->Process(q);
                if (st->nrec < st->max_vec) {
                    int32_t* r = st->rec + CS_REC * st->nrec++;
                    const short* d = (const short*)&c.direct_current();
                    r[0] = (int32_t)c.cca_state(); r[1] = (int32_t)(uint32_t)c.error_code();
                    for (int k = 0; k < 8; k++) r[2 + k] = d[k];
                    r[10] = (int32_t)c.cca_peak_index(); r[11] = (int32_t)c.cca_pwr_reading(); r[12] = (int32_t)st->vec20;
                }
            } else st->done = true;
            st->vec20++;
            ipin.pop();
        }
        return true;
    }
};
template<class C, class N> using DCRemove4 = TDCRemoveEx<4>::Filter<C, N>;
typedef Cap<COMPLEX16, 4>::Sink<Ctx> DropSink;
typedef TDCEstimator<Ctx, DropSink> DcEst;
typedef TCCA11a<Ctx, DcEst> Cca;
typedef DCRemove4<Ctx, Cca> DcRm;
typedef CsSwitch<Ctx, DcRm> Switch;
extern "C" {
size_t ref_rx11a_carrier_sense(const int16_t* iq, size_t n, unsigned cca_pwr_threshold, int32_t* rec, size_t max_vec, int64_t* detect) {
    Ctx* ctx = new Ctx(); ctx->cca_pwr_threshold() = cca_pwr_threshold;
    CsState st = {ctx, rec, 0, max_vec, 0, false};
    DropSink* drop = new DropSink(*ctx);
    DcEst* dcest = new DcEst(*ctx, drop); Cca* cca = new Cca(*ctx, dcest); DcRm* dc = new DcRm(*ctx, cca);
    Switch* sw = new Switch(*ctx, dc, &st);
    TDownSample2<Ctx, Switch>* ds2 = new TDownSample2<Ctx, Switch>(*ctx, sw);
    TPinQueue<COMPLEX16, 28, 8>* q = new TPinQueue<COMPLEX16, 28, 8>();
    for (size_t b = 0; b + 28 <= n && !st.done; b += 28) {
        memcpy(q->append(), iq + 2 * b, 28 * sizeof(COMPLEX16)); ds2->Process(*q);
        drop->got.clear();
        if (ctx->error_code() == E_ERROR_CS_TIMEOUT) { ctx->CF_Error::error_code() = E_ERROR_SUCCESS; ctx->CF_11CCA::Reset(); dc->Reset(); }
    }
    *detect = st.done || ctx->cca_state() == CF_11CCA::power_detected ? (int64_t)(st.nrec ? rec[CS_REC * (st.nrec - 1) + 12] + 1 : 0) : -1;
    size_t m = st.nrec;
    delete q; delete ds2; delete dc; delete ctx;     // ds2 holds the only reference to sw, dc the chain behind it
    return m;
}
// what the tap counted during the last ref_rx11a_lts / ref_rx11a_symbols call of this thread (see sbref::counts)
void ref_rx11a_debug(uint64_t out[6]) { for (int k = 0; k < 6; k++) out[k] = sbref::counts[k]; }
}
ENTRY
# demapper.h declares DemapperCore::Demap<1, 2, 4, 6> as explicit specialisations inside the class (demapper.h:48-53), which only MSVC
# accepts.  The build reads it through one textual rewrite into the shim directory, removed once the library is built: each
# `template<> static void Demap<N>(` becomes a static member Demap_N with the same body, and the specialisations are declared after
# the class, at namespace scope, each forwarding to Demap_N (entry.cpp).  The bodies, the LUTs and demap_limit stay the header's own.
sed 's/^\([[:space:]]*\)template<> static void Demap<\([0-9]\)>(/\1static void Demap_\2(/' "$B11/demapper.h" > "$INC/demapper.h"
[ "$(grep -c 'static void Demap_[1246](' "$INC/demapper.h")" = 4 ] || { echo "build_ref_rx11a: demapper.h rewrite did not apply" >&2; exit 1; }
# dspalg.hpp:89 calls CAccumulator's inherited Add(datum) unqualified from a class template whose base depends on its parameters; only
# a compiler without two-phase lookup (MSVC) finds it.  The same kind of rewrite makes that one call this->Add(datum).
sed 's/^\([[:space:]]*\)Add ( datum );/\1this->Add ( datum );/' "$BINC/dspalg.hpp" > "$INC/dspalg.hpp"
[ "$(grep -c 'this->Add ( datum );' "$INC/dspalg.hpp")" = 1 ] || { echo "build_ref_rx11a: dspalg.hpp rewrite did not apply" >&2; exit 1; }
LINKS="demapper11a.hpp sampling.hpp 44MTo40M.hpp"
for h in $LINKS; do ln -s "$B11/$h" "$INC/$h"; done
mkdir -p "$HERE/_ref"
rc=0
${CXX:-g++} -O2 -std=c++17 -mssse3 -msse4.1 -fno-strict-aliasing -fno-operator-names -fpermissive -fPIC -shared -fmax-errors=15 -w \
  -I"$INC" -I"$B11" -I"$BINC" -I"$CORE" -I"$HERE/../sora_b200/brick" "$INC/entry.cpp" -o "$HERE/_ref/librx11a_ref.so.tmp.$$" || rc=$?
for h in $LINKS demapper.h dspalg.hpp; do rm -f "$INC/$h"; done
[ $rc -eq 0 ] || { rm -f "$HERE/_ref/librx11a_ref.so.tmp.$$"; echo "build_ref_rx11a: compile failed" >&2; exit 1; }
mv -f "$HERE/_ref/librx11a_ref.so.tmp.$$" "$HERE/_ref/librx11a_ref.so"
echo "build_ref_rx11a: oracle/_ref/librx11a_ref.so"
