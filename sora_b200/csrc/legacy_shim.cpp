// Legacy C baseband interface (include/sora_b200_legacy.h) over the C ABI of include/sora_b200.h.  Host code only.
//
// The legacy driver loop alternates BB11ARxCarrierSense / BB11ARxFrameDemod over an RX stream of RX_BLOCKs (demod11a.cpp:81-200).
// Here the blocks between the scan pointer and the end of the stream are unpacked and decoded once on the device in
// continuous-capture mode (sb200_rxblocks_unpack + sb200_rx11a_stream); the two entry points then walk the resulting event list
// and move the stream's scan pointer exactly as far as the samples they consumed.
#include "../../include/sora_b200_legacy.h"
#include "../../include/sora_b200.h"
#include <cstdlib>
#include <cstring>
#include <vector>

namespace {
struct Event { sb200_frame_result r; uint32_t end_sample; uint32_t start_sample; std::vector<uint8_t> bytes; };
struct Events { const unsigned char* base = nullptr; size_t nblocks = 0; std::vector<Event> ev; size_t next = 0; bool pending = false; };
const uint32_t MAX_EVENTS = 256;

bool decode_from(PBB11A_RX_CONTEXT c, PSORA_RADIO_RX_STREAM s) {
    Events* E = (Events*)c->b200_events; sb200_handle* h = (sb200_handle*)c->b200_engine;
    const size_t nblocks = (size_t)(s->__pEndPt - s->__pScanPt) / SORA_RX_BLOCK_SIZE;
    E->base = s->__pScanPt; E->nblocks = nblocks; E->ev.clear(); E->next = 0; E->pending = false;
    if (!h || nblocks == 0) return false;
    std::vector<int16_t> iq(nblocks * 56);
    if (sb200_rxblocks_unpack(h, s->__pScanPt, nblocks, c->b200_shift, iq.data(), nullptr) != SB200_OK) return false;
    std::vector<sb200_frame_result> res(MAX_EVENTS); std::vector<uint32_t> sidx(MAX_EVENTS); std::vector<uint8_t> out((size_t)MAX_EVENTS * 2560);
    uint32_t n = 0;
    if (sb200_rx11a_stream(h, iq.data(), nblocks * 28, MAX_EVENTS, out.data(), 2560, res.data(), sidx.data(), &n, nullptr) != SB200_OK) return false;
    uint32_t prev = 0;
    for (uint32_t i = 0; i < n; i++) {
        Event e; e.r = res[i]; e.end_sample = sidx[i]; e.start_sample = prev + 2u * res[i].detect_index;
        e.bytes.assign(out.begin() + (size_t)i * 2560, out.begin() + (size_t)i * 2560 + (res[i].length < 2560 ? res[i].length : 2560));
        E->ev.push_back(std::move(e)); prev = sidx[i];
    }
    // a full event list means the capture may hold more: the decoded span ends with the block of the last event, and the next carrier sense
    // behind it decodes again from there (RxThread never stops after a fixed number of frames, fb11a_demod.cpp:29-81)
    if (n == MAX_EVENTS) { const size_t nb = ((size_t)sidx[n - 1] + 27u) / 28u; if (nb < E->nblocks) E->nblocks = nb; }
    return true;
}
}

extern "C" void SoraGenRadioRxStreamOffline(PSORA_RADIO_RX_STREAM s, PUCHAR in, ULONG size) {
    s->__pStartPt = in; s->__nRxBufSize = size / SORA_RX_BLOCK_SIZE * SORA_RX_BLOCK_SIZE; s->__pEndPt = in + s->__nRxBufSize; s->__pScanPt = in; s->__VStreamMask = 1;
}
extern "C" void BB11ARxContextInit(PBB11A_RX_CONTEXT c, unsigned int SampleRate, ULONG thr, ULONG maxBlk, ULONG minBlk, volatile FLAG* work) {
    memset(c, 0, sizeof *c);
    c->SampleRate = SampleRate; c->uiCSCorrThreshold = thr; c->uiCSMaxFetchRxBlock = maxBlk; c->uiCSMinFetchRxBlock = minBlk; c->ri_pbWorkIndicator = work;
    const char* d = getenv("SB200_DEVICE"); sb200_handle* h = nullptr;
    // rxThreshold gates the carrier sense.  The legacy detector asks autocorrelation > threshold (arx_cs.c:60-61), the brick detector this engine
    // runs asks energy > threshold with autocorrelation >= 7/8 energy (cca.hpp:342): same scale (16 samples of x >> 2), so it is handed through.
    sb200_cfg cfg; memset(&cfg, 0, sizeof cfg); cfg.cca_pwr_threshold = (uint32_t)thr;
    if (sb200_create(d ? atoi(d) : 0, &cfg, &h) == SB200_OK) c->b200_engine = h;          // no CPU fallback: every later call fails without it
    c->b200_events = new Events();
}
extern "C" void BB11APrepareRx(PBB11A_RX_CONTEXT c, char* frame, unsigned int max) { c->ri_pbFrame = frame; c->ri_uiFrameMaxSize = max; }
extern "C" BOOLEAN BB11ARxViterbiWorker(void*) { return 0; }
extern "C" void BB11ARxReset(PBB11A_RX_CONTEXT c) { if (c->b200_events) { Events* E = (Events*)c->b200_events; E->base = nullptr; E->ev.clear(); E->next = 0; E->pending = false; } }
extern "C" void BB11ARxContextCleanup(PBB11A_RX_CONTEXT c) {
    sb200_destroy((sb200_handle*)c->b200_engine); delete (Events*)c->b200_events; c->b200_engine = nullptr; c->b200_events = nullptr;
}
extern "C" void BB11ARxSetSampleShift(PBB11A_RX_CONTEXT c, unsigned int s) { c->b200_shift = s; BB11ARxReset(c); }

extern "C" HRESULT BB11ARxCarrierSense(PBB11A_RX_CONTEXT c, PSORA_RADIO_RX_STREAM s) {
    if (!c->b200_engine || !c->b200_events) return BB11A_E_FORCE_STOP;
    if (c->ri_pbWorkIndicator && !*c->ri_pbWorkIndicator) return BB11A_E_FORCE_STOP;
    Events* E = (Events*)c->b200_events;
    const bool inside = E->base && s->__pScanPt >= E->base && s->__pScanPt < E->base + E->nblocks * SORA_RX_BLOCK_SIZE;   // end exclusive: behind the decoded span, decode again
    if (!inside && !decode_from(c, s)) return BB11A_E_FORCE_STOP;
    const size_t pos_blk = (size_t)(s->__pScanPt - E->base) / SORA_RX_BLOCK_SIZE;
    const size_t max_blk = c->uiCSMaxFetchRxBlock ? c->uiCSMaxFetchRxBlock : 150;
    while (E->next < E->ev.size() && E->ev[E->next].end_sample / 28u <= pos_blk) E->next++;       // events the caller skipped over
    if (E->next < E->ev.size()) {
        const size_t det_blk = E->ev[E->next].start_sample / 28u;
        if (det_blk < pos_blk + max_blk) {
            s->__pScanPt = (PUCHAR)E->base + (det_blk > pos_blk ? det_blk : pos_blk) * SORA_RX_BLOCK_SIZE;
            E->pending = true;
            return BB11A_OK_POWER_DETECTED;
        }
    }
    size_t nb = pos_blk + max_blk; if (nb > E->nblocks) nb = E->nblocks;
    s->__pScanPt = (PUCHAR)E->base + nb * SORA_RX_BLOCK_SIZE;
    if (s->__pScanPt >= s->__pEndPt) { s->__pScanPt = s->__pStartPt; E->base = nullptr; }      // ring wrap: decode again from the start
    return BB11A_CHANNEL_CLEAN;
}

extern "C" HRESULT BB11ARxFrameDemod(PBB11A_RX_CONTEXT c, PSORA_RADIO_RX_STREAM s) {
    if (!c->b200_engine || !c->b200_events) return BB11A_E_FORCE_STOP;
    Events* E = (Events*)c->b200_events;
    if (!E->pending || E->next >= E->ev.size()) return BB11A_E_SYNC_FAIL;
    const Event& e = E->ev[E->next++]; E->pending = false;
    size_t end_blk = (e.end_sample + 27u) / 28u; if (end_blk > E->nblocks) end_blk = E->nblocks;
    s->__pScanPt = (PUCHAR)E->base + end_blk * SORA_RX_BLOCK_SIZE;
    if (s->__pScanPt >= s->__pEndPt) { s->__pScanPt = s->__pStartPt; E->base = nullptr; }
    c->ri_uiFrameSize = e.r.length; c->ri_uiDataRate = e.r.rate_kbps;
    if (e.r.status == SB200_FRAME_PLCP_FAIL) return BB11A_E_INVALID_SIG;
    if (e.r.status != SB200_FRAME_OK && e.r.status != SB200_FRAME_CRC32_FAIL) return BB11A_E_SYNC_FAIL;
    if (!c->ri_pbFrame || e.r.length > c->ri_uiFrameMaxSize) return BB11A_E_FRAME_SIZE;
    memcpy(c->ri_pbFrame, e.bytes.data(), e.bytes.size());
    return e.r.status == SB200_FRAME_OK ? BB11A_OK_FRAME : BB11A_E_CRC32;
}

// ---- 802.11b (bbb.h) ---------------------------------------------------------------------------------------------------------------------
// Same idea: everything between the scan pointer and the end of the stream is decoded once in continuous-capture mode
// (sb200_rxblocks_unpack + sb200_rx11b_streams); BB11BSpd and BB11BRx walk the event list like the driver loop of demod11b.cpp:73-174.
namespace {
struct Event11b { sb200_frame_result_11b r; uint32_t start_sample, end_sample; std::vector<uint8_t> bytes; };
struct Events11b { const unsigned char* base = nullptr; size_t nblocks = 0; std::vector<Event11b> ev; size_t next = 0; bool pending = false, abandoned = false; };

bool decode11b_from(PBB11B_RX_CONTEXT c, PSORA_RADIO_RX_STREAM s) {
    Events11b* E = (Events11b*)c->b200_events; sb200_handle* h = (sb200_handle*)c->b200_engine;
    const size_t nblocks = (size_t)(s->__pEndPt - s->__pScanPt) / SORA_RX_BLOCK_SIZE;
    E->base = s->__pScanPt; E->nblocks = nblocks; E->ev.clear(); E->next = 0; E->pending = false; E->abandoned = false;
    if (!h || nblocks == 0) return false;
    std::vector<int16_t> iq(nblocks * 56);
    if (sb200_rxblocks_unpack(h, s->__pScanPt, nblocks, 0, iq.data(), nullptr) != SB200_OK) return false;
    if (c->b_shiftRight) for (auto& v : iq) v = c->b_shiftRight > 0 ? (int16_t)(v >> c->b_shiftRight) : (int16_t)(v << -c->b_shiftRight);   // bbb.h:141 b_shiftRight
    std::vector<sb200_frame_result_11b> res(MAX_EVENTS); std::vector<uint8_t> out((size_t)MAX_EVENTS * 4096);
    const uint64_t off = 0; const uint32_t len = (uint32_t)(nblocks * 28); uint32_t n = 0;
    if (sb200_rx11b_streams(h, iq.data(), nblocks * 28, &off, &len, 1, MAX_EVENTS, out.data(), 4096, res.data(), &n, nullptr) != SB200_OK) return false;
    uint32_t skipped = 0;                                 // samples the source sought over so far: detect_vec counts processed vectors only
    for (uint32_t i = 0; i < n; i++) {
        Event11b e; e.r = res[i]; e.end_sample = res[i].sample_index; e.start_sample = res[i].detect_vec * 4u + skipped;
        const uint32_t nb = res[i].length < 4096u ? res[i].length : 4096u;
        e.bytes.assign(out.begin() + (size_t)i * 4096, out.begin() + (size_t)i * 4096 + nb);
        if (res[i].status == SB200_FRAME_OK || res[i].status == SB200_FRAME_CRC32_FAIL)
            skipped += res[i].rate_kbps == 1000 ? 352u : res[i].rate_kbps == 2000 ? 176u : res[i].rate_kbps == 5500 ? 64u : 32u;
        E->ev.push_back(std::move(e));
    }
    if (n == MAX_EVENTS) { const size_t nb = ((size_t)res[n - 1].sample_index + 27u) / 28u; if (nb < E->nblocks) E->nblocks = nb; }   // as for 802.11a above
    return true;
}
}

extern "C" void BB11BRxSpdContextInit(PBB11B_RX_CONTEXT rx, PBB11B_SPD_CONTEXT spd, PFLAG work, ULONG nRxMax, ULONG nSpdMax, ULONG nSpdMin, ULONG thr, ULONG thrLow, ULONG thrHigh, ULONG shiftRight) {
    memset(rx, 0, sizeof *rx); memset(spd, 0, sizeof *spd);
    rx->b_maxDescCount = nRxMax; rx->b_workIndicator = work; rx->b_shiftRight = (int)shiftRight;
    spd->b_minDescCount = nSpdMin; spd->b_maxDescCount = nSpdMax; spd->b_threshold = thr; spd->b_thresholdLH = thrLow; spd->b_thresholdHL = thrHigh;
    spd->b_workIndicator = work; spd->b200_rx = rx;
    const char* d = getenv("SB200_DEVICE"); sb200_handle* h = nullptr;
    // nSPDThreshold is stored but not handed to the engine: the legacy software power detector compares it with a per-block energy in another
    // scale (bbb_spd.c:204, demod11's default 4000) than TEnergyDetect's 8-vector average (cca.hpp:79, default 1000*1000), which is what runs here.
    if (sb200_create(d ? atoi(d) : 0, nullptr, &h) == SB200_OK) rx->b200_engine = h;    // no CPU fallback: every later call fails without it
    rx->b200_events = new Events11b();
}
extern "C" void BB11BRxSpdContextCleanUp(PBB11B_RX_CONTEXT rx) {
    sb200_destroy((sb200_handle*)rx->b200_engine); delete (Events11b*)rx->b200_events; rx->b200_engine = nullptr; rx->b200_events = nullptr;
}
extern "C" void BB11BPrepareRx(PBB11B_RX_CONTEXT rx, void* buf, ULONG size) { rx->BB11bCommon.b_outputPt = (PUCHAR)buf; rx->BB11bCommon.b_maxOutputSize = size; }

extern "C" HRESULT BB11BSpd(PBB11B_SPD_CONTEXT spd, PSORA_RADIO_RX_STREAM s) {
    PBB11B_RX_CONTEXT c = (PBB11B_RX_CONTEXT)spd->b200_rx;
    if (!c || !c->b200_engine || !c->b200_events) return BB11B_E_FORCE_STOP;
    if (spd->b_workIndicator && !*spd->b_workIndicator) return BB11B_E_FORCE_STOP;
    Events11b* E = (Events11b*)c->b200_events;
    const bool inside = E->base && s->__pScanPt >= E->base && s->__pScanPt < E->base + E->nblocks * SORA_RX_BLOCK_SIZE;
    if (!inside && !decode11b_from(c, s)) return BB11B_E_FORCE_STOP;
    const size_t pos_blk = (size_t)(s->__pScanPt - E->base) / SORA_RX_BLOCK_SIZE;
    const size_t max_blk = spd->b_maxDescCount ? spd->b_maxDescCount : 150;
    while (E->next < E->ev.size() && E->ev[E->next].end_sample / 28u <= pos_blk) E->next++;       // events the caller skipped over
    if (E->next < E->ev.size()) {
        const size_t det_blk = E->ev[E->next].start_sample / 28u;
        if (det_blk < pos_blk + max_blk) {
            s->__pScanPt = (PUCHAR)E->base + (det_blk > pos_blk ? det_blk : pos_blk) * SORA_RX_BLOCK_SIZE;
            E->pending = true; E->abandoned = false;
            return BB11B_OK_POWER_DETECTED;
        }
    }
    size_t nb = pos_blk + max_blk; if (nb > E->nblocks) nb = E->nblocks;
    s->__pScanPt = (PUCHAR)E->base + nb * SORA_RX_BLOCK_SIZE;
    if (s->__pScanPt >= s->__pEndPt) { s->__pScanPt = s->__pStartPt; E->base = nullptr; }      // ring wrap: decode again from the start
    return BB11B_CHANNEL_CLEAN;
}

extern "C" HRESULT BB11BRx(PBB11B_RX_CONTEXT c, PSORA_RADIO_RX_STREAM s) {
    if (!c->b200_engine || !c->b200_events) return BB11B_E_FORCE_STOP;
    if (c->b_workIndicator && !*c->b_workIndicator) return BB11B_E_FORCE_STOP;
    Events11b* E = (Events11b*)c->b200_events;
    if (E->abandoned) { E->abandoned = false; return BB11B_E_ENERGY; }                           // the frame behind a refused header is dropped
    if (!E->pending || E->next >= E->ev.size()) return BB11B_E_ENERGY;
    const Event11b& e = E->ev[E->next++]; E->pending = false;
    size_t end_blk = (e.end_sample + 27u) / 28u; if (end_blk > E->nblocks) end_blk = E->nblocks;
    s->__pScanPt = (PUCHAR)E->base + end_blk * SORA_RX_BLOCK_SIZE;
    if (s->__pScanPt >= s->__pEndPt) { s->__pScanPt = s->__pStartPt; E->base = nullptr; }
    BB11B_COMMON& B = c->BB11bCommon;
    B.b_length = e.r.length; B.b_isLongPreamble = 1; B.b_crc32 = e.r.crc32;
    B.b_dataRate = e.r.rate_kbps == 1000 ? 0x0A : e.r.rate_kbps == 2000 ? 0x14 : e.r.rate_kbps == 5500 ? 0x37 : e.r.rate_kbps == 11000 ? 0x6E : 0;
    switch (e.r.status) {
        case SB200_FRAME_OK: case SB200_FRAME_CRC32_FAIL:
            if (!B.b_outputPt || e.bytes.size() > B.b_maxOutputSize) { B.b_errFrame++; return BB11B_E_DATA; }
            memcpy(B.b_outputPt, e.bytes.data(), e.bytes.size());
            if (e.r.status == SB200_FRAME_OK) { B.b_goodFrameCounter++; return BB11B_OK_FRAME; }
            B.b_errFrame++; return BB11B_E_DATA;
        case SB200_FRAME_PLCP_FAIL: B.b_errPLCPHeader++; E->abandoned = true; return BB11B_E_PLCP_HEADER_CRC;
        case SB200_FRAME_SFD_FAIL: case SB200_FRAME_SFD_TIMEOUT: return BB11B_E_SFD;
        case SB200_FRAME_SYNC_TIMEOUT: E->abandoned = true; return BB11B_E_BARKER;
        default: B.b_errEnergyLoss++; return BB11B_E_ENERGY;
    }
}


// ---- BB11BPMDSpreadFIR4SSE / BB11BPMDSpreadFIR4ASM (bbb.h:188-200): context-free in the reference, so the engine is process-wide here ----
#include <mutex>
static std::mutex g_fir_mu; static sb200_handle* g_fir_engine = nullptr;
static bool fir_engine() {                              // under g_fir_mu
    if (!g_fir_engine) {
        const char* d = getenv("SB200_DEVICE"); sb200_handle* h = nullptr;
        if (sb200_create(d ? atoi(d) : 0, nullptr, &h) != SB200_OK) return false;                  // no CPU fallback
        g_fir_engine = h;
    }
    return true;
}
static HRESULT spread_fir(const SORA_COMPLEX8* src, uint32_t n, SORA_COMPLEX8* dst, ULONG* out_n, uint32_t variant) {
    if (!src || !dst || (n & 7u)) return SORA_E_FAIL;
    std::lock_guard<std::mutex> lk(g_fir_mu);
    if (!fir_engine()) return SORA_E_FAIL;
    const uint64_t off = 0; const uint32_t len = n;
    if (n && sb200_tx11b_fir37(g_fir_engine, (const int8_t*)src, n, &off, &len, 1, variant, (int8_t*)dst, nullptr) != SB200_OK) return SORA_E_FAIL;
    if (out_n) *out_n = n;
    return SORA_S_OK;
}
extern "C" HRESULT BB11BPMDSpreadFIR4SSE(const SORA_COMPLEX8* s, uint32_t n, SORA_COMPLEX8* d, ULONG* on) { return spread_fir(s, n, d, on, 0); }
extern "C" HRESULT BB11BPMDSpreadFIR4ASM(const SORA_COMPLEX8* s, uint32_t n, SORA_COMPLEX8* d, ULONG* on) { return spread_fir(s, n, d, on, 1); }

// ---- the legacy 802.11b transmitter (bbb.h:204-240, bbb_tx.c) over sb200_tx11b_legacy_batch ---------------------------------------------
namespace {
uint32_t kbps_of_code(UCHAR c) { return c == 0x0A ? 1000u : c == 0x14 ? 2000u : c == 0x37 ? 5500u : c == 0x6E ? 11000u : 0u; }
// the samples BB11BPMDBufferTx4X* writes for a PSDU of `size` bytes (FCS included): 4 per chip, TX_FIR_DEPTH zeros rounded up to 128
uint32_t legacy_nsamples(uint32_t size, UCHAR pre, uint32_t kbps) {
    const uint32_t cpb = kbps == 1000 ? (pre ? 0u : 88u) : kbps == 2000 ? 44u : kbps == 5500 ? 16u : 8u;
    return (4u * ((pre ? 1056u : 2112u) + size * cpb) + 37u + 127u) & ~127u;
}
// the scrambler's side effect on the caller's bytes: the stream runs over the PLCP frame first (bbb_tx.c:537-538, :669-670)
void scramble_in_place(const DOT11B_PLCP_TXVECTOR* v, uint32_t kbps, uint32_t size, const std::vector<uint8_t*>& bytes) {
    uint32_t plen, ext = 0;                                                                 // PLCPGetLength (bbb_tx.c:39-65), CCK
    if (kbps == 1000) plen = size << 3; else if (kbps == 2000) plen = size << 2;
    else if (kbps == 5500) plen = ((size << 4) - 1u) / 11u + 1u;
    else { plen = ((size << 3) - 1u) / 11u + 1u; if (plen * 11u - (size << 3) >= 8u) ext = 1; }
    uint8_t hdr[6] = {v->DateRate, (uint8_t)(ext << 7), (uint8_t)plen, (uint8_t)(plen >> 8), 0, 0};
    unsigned c = 0xFFFFu;
    for (int i = 0; i < 4; i++) { c ^= hdr[i]; for (int k = 0; k < 8; k++) c = (c & 1u) ? (c >> 1) ^ 0x8408u : c >> 1; }
    c = ~c & 0xFFFFu; hdr[4] = (uint8_t)c; hdr[5] = (uint8_t)(c >> 8);
    unsigned reg = v->PreambleType ? 0x1Bu : 0x6Cu;
    auto scr = [&](uint8_t x) { uint8_t o = 0; for (int k = 0; k < 8; k++) { const unsigned b = (x ^ reg ^ (reg >> 3)) & 1u; reg = (reg >> 1) | (b << 6); o |= (uint8_t)(b << k); x >>= 1; } reg = o >> 1; return o; };
    const int nsync = v->PreambleType ? 7 : 16;
    for (int i = 0; i < nsync; i++) scr(v->PreambleType ? 0x00 : 0xFF);
    if (v->PreambleType) { scr(0xCF); scr(0x05); } else { scr(0xA0); scr(0xF3); }
    for (int i = 0; i < 6; i++) scr(hdr[i]);
    for (uint8_t* b : bytes) *b = scr(*b);
}
// encode psdu (FCS included) with the filter selected (0 encoder output, 1 SSE filter) into dst; n = samples written
HRESULT legacy_tx(const DOT11B_PLCP_TXVECTOR* v, const std::vector<uint8_t>& psdu, uint32_t filter, void* dst, uint32_t* n) {
    const uint32_t kbps = kbps_of_code(v->DateRate);
    if (!kbps || v->PreambleType > 1 || v->ModSelect != 0 || psdu.size() < 4 || psdu.size() > 4095) return SORA_E_FAIL;
    const uint32_t ns = legacy_nsamples((uint32_t)psdu.size(), v->PreambleType, kbps);
    void* buf = nullptr;
    if (posix_memalign(&buf, 16, (size_t)ns * 2) != 0) return SORA_E_FAIL;
    const uint64_t off = 0; const uint32_t len = (uint32_t)psdu.size(); uint32_t got = 0;
    int rc;
    {   std::lock_guard<std::mutex> lk(g_fir_mu);
        rc = fir_engine() ? sb200_tx11b_legacy_batch(g_fir_engine, psdu.data(), len, &off, &len, 1, kbps, v->PreambleType, SB200_TX11B_LEGACY_FCS_IN_PAYLOAD, filter,
                                                     (int8_t*)buf, ns, &got, nullptr) : SB200_E_NODEVICE; }
    if (rc == SB200_OK && got == ns) memcpy(dst, buf, (size_t)ns * 2);
    free(buf);
    if (rc != SB200_OK || got != ns) return SORA_E_FAIL;
    *n = ns;
    return SORA_S_OK;
}
HRESULT buffer_tx(PDOT11B_PLCP_TXVECTOR v, PUCHAR data, unsigned int dataLength, PUCHAR out, unsigned int* n, UCHAR pre) {
    if (!v || !data || !out || !n) return SORA_E_FAIL;
    DOT11B_PLCP_TXVECTOR w = *v; w.PreambleType = pre;                                   // the entry point, not the vector, picks the preamble
    std::vector<uint8_t> psdu(data, data + dataLength + 4u);
    uint32_t ns = 0;
    const HRESULT r = legacy_tx(&w, psdu, 0, out, &ns);
    if (r != SORA_S_OK) return r;
    std::vector<uint8_t*> bytes; for (unsigned int i = 0; i < dataLength + 4u; i++) bytes.push_back(data + i);
    scramble_in_place(&w, kbps_of_code(w.DateRate), dataLength + 4u, bytes);
    *n = ns;
    return SORA_S_OK;
}
// the MDL chain and Reserved1 as one PSDU; pointers to the bytes in order (for the in-place scramble)
bool packet_bytes(PPACKET_BASE p, std::vector<uint8_t>& psdu, std::vector<uint8_t*>& where) {
    for (PMDL m = p->pMdl; m; m = m->Next)
        for (ULONG i = 0; i < m->ByteCount; i++) { uint8_t* b = (uint8_t*)m->StartVa + m->ByteOffset + i; psdu.push_back(*b); where.push_back(b); }
    if (psdu.size() != p->PacketSize) return false;
    for (int i = 0; i < 4; i++) { uint8_t* b = (uint8_t*)&p->Reserved1 + i; psdu.push_back(*b); where.push_back(b); }   // little endian, as sizeof(ULONG) bytes are read
    return true;
}
HRESULT packet_tx(PDOT11B_PLCP_TXVECTOR v, PPACKET_BASE p, PUCHAR out, ULONG* n, PTXSAMPLE filtered, ULONG* nfiltered) {
    if (!v || !p || !out) return SORA_E_FAIL;
    if (v->PreambleType > 1) return SORA_E_FAIL;                                            // bbb_tx.c:94-97
    std::vector<uint8_t> psdu; std::vector<uint8_t*> where;
    if (!packet_bytes(p, psdu, where)) return SORA_E_FAIL;
    uint32_t ns = 0;
    HRESULT r = legacy_tx(v, psdu, 0, out, &ns);
    if (r == SORA_S_OK && filtered) r = legacy_tx(v, psdu, 1, filtered, &ns);
    if (r != SORA_S_OK) return r;
    scramble_in_place(v, kbps_of_code(v->DateRate), (uint32_t)psdu.size(), where);
    if (n) *n = ns;
    if (nfiltered) *nfiltered = ns;
    return SORA_S_OK;
}
}

extern "C" void BB11BTxVectorInit(PDOT11B_PLCP_TXVECTOR v, UCHAR rate, UCHAR mod, UCHAR pre) { v->DateRate = rate; v->ModSelect = mod; v->PreambleType = pre; }
extern "C" HRESULT BB11BPMDBufferTx4XWithShortHeader(PDOT11B_PLCP_TXVECTOR v, PUCHAR d, unsigned int len, PUCHAR o, unsigned int* n) { return buffer_tx(v, d, len, o, n, 1); }
extern "C" HRESULT BB11BPMDBufferTx4XWithLongHeader(PDOT11B_PLCP_TXVECTOR v, PUCHAR d, unsigned int len, PUCHAR o, unsigned int* n) { return buffer_tx(v, d, len, o, n, 0); }
extern "C" HRESULT BB11BPMDPacketTx4X(PDOT11B_PLCP_TXVECTOR v, PPACKET_BASE p, PUCHAR o, ULONG BufferLength, ULONG* n) {
    (void)BufferLength;                                                                      // unused by the reference too (bbb_tx.c:84)
    return packet_tx(v, p, o, n, nullptr, nullptr);
}
extern "C" void SoraPacketGetTxSampleBuffer(PPACKET_BASE p, PTXSAMPLE* b, ULONG* size) {
    *b = p && p->pTxDesc ? p->pTxDesc->pSampleBuffer : nullptr; *size = p && p->pTxDesc ? p->pTxDesc->SampleBufferSize : 0;
}
extern "C" void SoraPacketSetSignalLength(PPACKET_BASE p, ULONG len) { if (p && p->pTxDesc) p->pTxDesc->SignalLength = len; }
extern "C" HRESULT BB11BPMDPacketGenSignal(PPACKET_BASE p, PDOT11B_PLCP_TXVECTOR v, PUCHAR temp, ULONG temp_len) {
    PTXSAMPLE sb = nullptr; ULONG sb_size = 0;
    if (!p) return SORA_E_FAIL;
    SoraPacketGetTxSampleBuffer(p, &sb, &sb_size);
    if (temp_len < BB11B_MAX_SYMBOL_LENGTH || sb_size < BB11B_MAX_SYMBOL_LENGTH || !sb || !temp) return SORA_E_FAIL;   // bbb_tx.c:133-137
    ULONG n = 0, nf = 0;
    const HRESULT r = packet_tx(v, p, temp, &n, sb, &nf);
    if (r != SORA_S_OK) return r;
    memset(temp + (size_t)n * 2, 0, 64);                                                     // bbb_tx.c:140
    SoraPacketSetSignalLength(p, nf * (ULONG)sizeof(TXSAMPLE));
    return SORA_S_OK;
}

// ---- the legacy 802.11a transmitter (bba.h:201-247, atx_fe.c) over sb200_tx11a_legacy_batch ------------------------------------------------
namespace {
std::mutex g_pre_mu; bool g_pre_set = false; int16_t g_pre[1280];
uint32_t kbps_of_11a(unsigned int c) {
    switch (c) { case 0xB: return 6000; case 0xF: return 9000; case 0xA: return 12000; case 0xE: return 18000;
                 case 0x9: return 24000; case 0xD: return 36000; case 0x8: return 48000; case 0xC: return 54000; default: return 0; }
}
uint32_t nsamples_11a(uint32_t size, uint32_t kbps, unsigned int sr) {   // GetSignalBytes (atx_tpl.h:69-83) / 2, rounded up to 128 bytes
    const uint32_t ndbps = kbps / 250u, nsym = (22u + 8u * size + ndbps - 1u) / ndbps;
    return ((sr == 44 ? 176u : 160u) * (5u + nsym) + 8u + 63u) & ~63u;
}
// modulate psdu (FCS included) into dst, which holds at least cap_bytes; *n = padded samples
bool tx11a(const std::vector<uint8_t>& psdu, uint32_t kbps, unsigned int sr, void* dst, size_t cap_bytes, uint32_t* n) {
    if (!kbps || (sr != 40 && sr != 44) || psdu.size() < 4 || psdu.size() > 4096 || !dst) return false;
    const uint32_t ns = nsamples_11a((uint32_t)psdu.size(), kbps, sr);
    if ((size_t)ns * 2 > cap_bytes) return false;
    void* buf = nullptr;
    if (posix_memalign(&buf, 16, (size_t)ns * 2) != 0) return false;
    int16_t pre[1280];
    {   std::lock_guard<std::mutex> lk(g_pre_mu);
        if (!g_pre_set) { free(buf); return false; }
        memcpy(pre, g_pre, sizeof pre); }
    const uint64_t off = 0; const uint32_t len = (uint32_t)psdu.size(); uint32_t got = 0;
    int rc;
    {   std::lock_guard<std::mutex> lk(g_fir_mu);
        rc = fir_engine() ? sb200_tx11a_legacy_batch(g_fir_engine, psdu.data(), len, &off, &len, 1, kbps, sr, SB200_TX11A_LEGACY_FCS_IN_PAYLOAD, pre,
                                                     (int8_t*)buf, ns, &got, nullptr) : SB200_E_NODEVICE; }
    const bool ok = rc == SB200_OK && got == ns;
    if (ok) memcpy(dst, buf, (size_t)ns * 2);
    free(buf);
    if (ok) *n = ns;
    return ok;
}
}

extern "C" void BB11ATxSetPreamble(const void* p) {
    std::lock_guard<std::mutex> lk(g_pre_mu);
    g_pre_set = p != nullptr;
    if (p) memcpy(g_pre, p, sizeof g_pre);
}
extern "C" void BB11ATxContextInit(PBB11A_TX_VECTOR info, unsigned int SampleRate) {   // a_init.c:61-86: the data rate is left as it is
    if (!info) return;
    info->SampleRate = SampleRate; info->ti_uiBufferLength = 0;
}
extern "C" HRESULT BB11ATxFrameMod(PBB11A_TX_VECTOR info, PPACKET_BASE p) {
    if (!info || !p) return SORA_E_FAIL;
    if (p->PacketSize + 4u > 4096u) return SORA_E_FAIL;                                    // atx_fe.c:23
    const uint32_t kbps = kbps_of_11a(info->ti_uiDataRate);
    if (!kbps) return SORA_E_FAIL;                                                          // atx_fe.c:59-62
    std::vector<uint8_t> psdu; std::vector<uint8_t*> where;
    if (!packet_bytes(p, psdu, where)) return SORA_E_FAIL;                                  // MDL chain + Reserved1 (atx_tpl.h:24-46)
    PTXSAMPLE sb = nullptr; ULONG sb_size = 0;
    SoraPacketGetTxSampleBuffer(p, &sb, &sb_size);
    uint32_t n = 0;
    if (!tx11a(psdu, kbps, info->SampleRate, sb, sb_size, &n)) return SORA_E_FAIL;
    SoraPacketSetSignalLength(p, n * (ULONG)sizeof(TXSAMPLE));
    return SORA_S_OK;
}
extern "C" ULONG BB11AModulateACK(unsigned int SampleRate, const PMAC_ADDRESS ra, void* out) {
    if (!ra || !out) return 0;
    std::vector<uint8_t> ack = {0xD4, 0x00, 0x00, 0x00};                                  // FrameControl: ACK, control; Duration 0 (atx_fe.c:181-184)
    ack.insert(ack.end(), ra->Address, ra->Address + 6);
    uint32_t c = 0xFFFFFFFFu;
    for (uint8_t b : ack) { c ^= b; for (int k = 0; k < 8; k++) c = (c & 1u) ? (c >> 1) ^ 0xEDB88320u : c >> 1; }
    c = ~c;
    for (int i = 0; i < 4; i++) ack.push_back((uint8_t)(c >> (8 * i)));
    // BB11ATxBufferMod6M: 6 Mbps whatever ti_uiDataRate says (the reference sets DOT11A_RATE_24M and never reads it there)
    uint32_t n = 0;
    if (!tx11a(ack, 6000, SampleRate, out, (size_t)nsamples_11a(14, 6000, SampleRate) * 2, &n)) return 0;
    return n * (ULONG)sizeof(TXSAMPLE);
}
