// ORACLE — TEST INFRASTRUCTURE ONLY (see ops.h).
// CPU restatement of the reference's 802.11a brick receive graph
//   kernel/bb/demod11/fb11ademod_config.hpp:169-242 (CreateDemodGraph11a_40M)
//   driven like kernel/bb/demod11/fb11a_demod.cpp:29-81 (RxThread).
#pragma once
#include "viterbi.h"
#include <vector>

namespace sbo {

// error codes (brick/inc/stdfacade.h:10-12, Brick11/src/ieee80211facade.hpp:10-19)
enum : uint32_t {
    E_SUCCESS = 0, E_FRAME_OK = 1, E_FAILED = 0x8000FFFFu, E_PLCP_HEADER_FAIL = 0x80000005u,
    E_CRC32_FAIL = 0x80000006u, E_CS_TIMEOUT = 0x80000007u,
    E_NO_FRAME = 0x8000F001u,   // oracle/engine only: sample buffer exhausted before any frame event
};

struct FrameResult {
    uint32_t status, rate_kbps, length, crc32, nsym;
    uint32_t sample_index;      // CF_MemSamples::mem_sample_index when the event was seen (40 Msps samples)
    uint32_t detect_index;      // 20 Msps index (since start/seek) of the first vector routed to the demod branch
    int16_t  cfo_est;           // CF_CFOffset::CFO_est after the LTS
    uint16_t peak_index;        // CF_11CCA::cca_peak_index
};

// per-frame intermediate taps for stage-level parity tests (symbol 0 = SIGNAL)
struct Taps {
    bool enable = false;
    std::vector<c16> freq_coeffs, chan_coeffs;      // 64 each (after LTS)
    std::vector<c16> fft_in, fft_out, equalized, tracked;    // 64 per symbol (fft_in: what fft64 is handed)
    std::vector<c16> lts_in, sym_in;                 // what on_lts (144) and on_symbol (80 per symbol) are handed
    std::vector<int32_t> cs;                         // per vector cca_process is handed, 13 values after it (see sbo_rx11a_cs_trace)
    std::vector<uint8_t> soft;                       // deinterleaved soft bits, N_CBPS per symbol, concatenated
    std::vector<uint32_t> soft_off;                  // offset of each symbol in `soft`
    void clear() { freq_coeffs.clear(); chan_coeffs.clear(); fft_in.clear(); fft_out.clear(); lts_in.clear(); sym_in.clear(); cs.clear(); equalized.clear(); tracked.clear(); soft.clear(); soft_off.clear(); }
};

class Rx11a {
public:
    Rx11a();
    void init();                               // BB11aDemodContext::Init (fb11ademod_config.hpp:105-121)
    // feed one TMemSamples block of 28 samples (40 Msps).  Returns CF_Error::error_code afterwards.
    uint32_t push_block28(const c16* s);
    void reset_after_event();                  // ssrc->Flush(); ctx.Reset(); ssrc->Reset()  (fb11a_demod.cpp:64-72)
    void reset_carrier_sense();                // ctx.ResetCarrierSense(); scs->Reset()       (fb11a_demod.cpp:47-49)
    // Whole-buffer driver mirroring RxThread: decodes up to max_frames events, returns the count.
    int run(const c16* samples, size_t n, FrameResult* res, uint8_t* out, size_t out_stride, int max_frames);

    uint32_t cca_pwr_threshold = 1000 * 1000;
    Taps taps;
    // Two-thread topology of the reference (TThreadSeparator between the de-interleaver and T11aViterbi, fb11ademod_config.hpp:169-242;
    // stdbrick.hpp:91-248): with `split` set, the front end hands every de-interleaved DATA symbol to it instead of decoding it, and a second
    // Rx11a object on the consumer thread runs back_begin / back_symbol / back_result.
    struct SoftSplit { virtual void begin(int code_rate, uint16_t frame_length) = 0; virtual void symbol(const uint8_t* dsoft, int ncbps) = 0; virtual ~SoftSplit() {} };
    SoftSplit* split = nullptr;
    void back_begin(int code_rate_, uint16_t frame_length_);
    void back_symbol(const uint8_t* dsoft, int ncbps);
    uint32_t back_status() const { return error_code; }
    uint32_t back_crc32() const { return frame_crc32; }
    const uint8_t* frame_bytes() const { return frame_buf; }
    // T11aPLCPParser alone, on a context whose CF_11aRxVector, CF_11RxPLCPSwitch and CF_Error were just Reset (as after every event):
    // out = plcp_state (1: accepted), error_code, data_rate_kbps, frame_length, total_symbols, code_rate
    void plcp_parse_only(uint32_t sig, uint32_t out[6]);
    // T11aDesc -> TBB11aFrameSink alone, both fresh, for a frame of frame_length_ bytes, fed n decoded bytes; returns error_code
    // (frame_bytes() and back_crc32() hold the rest)
    uint32_t desc_sink_only(const uint8_t* in, size_t n, uint16_t frame_length_);

private:
    // ---- context facades ----
    uint32_t error_code;
    int cca_state;                 // 0 power_clear, 1 power_detected
    uint32_t cca_pwr_reading, cca_peak_index;
    v128 DC;                       // CF_VecDC (persists across frames)
    int16_t CFO_est, CFO_comp, SFO_comp, CFO_tracker, SFO_tracker;
    uint32_t symbol_count; int symbol_type, plcp_state;
    alignas(16) c16 ChannelCoeffs[64], FreqCoeffs[64], CompCoeffs[64];
    uint16_t frame_length, total_symbols, remain_symbols, code_rate; uint32_t data_rate_kbps, frame_crc32;
    uint32_t mem_sample_index;
    // ---- TDownSample2 input queue ----
    c16 ds_q[64]; int ds_n;
    // ---- TDCEstimator ----
    uint32_t dc_update_cnt; v128 dc_sum;
    // ---- TCCA11a ----
    v128 his[4]; int his_idx;
    int acr[4], aci[4], eng[4]; int acr_i, aci_i, eng_i; int acr_reg, aci_reg, eng_reg;
    uint32_t auto_count, sense_count, high_count; int sync_state; int peak_corr, peak_index;
    // ---- symbol framing ----
    alignas(16) c16 lts_q[144]; int lts_n;
    alignas(16) c16 sym_q[80]; int sym_n;
    uint32_t vec20_count, detect_index;
    // ---- back end ----
    ViterbiCore vit; uint32_t ob_count;
    uint32_t desc_count; uint8_t desc_reg;
    uint8_t frame_buf[4096]; uint32_t byte_count, crc_run;
    std::vector<uint8_t> vit_out;

    void ctx_reset();
    void rxvector_reset();
    bool plcp_parse(uint32_t sig);
    void cca_init();
    void dcest_init();
    void on_vec20(v128 v);
    void cca_process(v128 pi);
    void dcest_process(v128 pi);
    int  xcorr(int k, const c16* pattern);
    bool establish_sync();
    bool check_sync();
    void on_lts();
    void on_symbol();
    void sink_byte(uint8_t b);
};

// Standalone stage entry points used by the stage-level parity tests and the Viterbi benchmark
void deinterleave(const uint8_t* in, uint8_t* out, int ncbps);
void demap_symbol(const c16* eq /*64*/, uint8_t* out, int nbpsc);
size_t resample_44_40(const c16* in, size_t n_in, c16* out);   // out must hold n_in samples

} // namespace sbo
