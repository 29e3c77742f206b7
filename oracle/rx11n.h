// ORACLE — TEST INFRASTRUCTURE ONLY (see ops.h).
// CPU restatement of the reference's 802.11n 2x2 (HT mixed format, 20 MHz, 2 spatial streams) receive graph: MCS 8..10 as the reference's HT-SIG parser
// admits them (PHY_11n.hpp:496-501), and MCS 11..14 through the 16-QAM / 64-QAM branches the graph already carries (fb11ndemod_config.hpp:206-236,
// demapper11n.hpp:199-309, deinterleaver_11n.hpp) when the parser's gate is opened (ht_mcs_limit; SURVEY.md §8(f) rank 4)
//   kernel/bb/demod11/fb11ndemod_config.hpp:167-262 (CreateDemodGraph11n)
//   driven like kernel/bb/demod11/fb11n_demod.cpp:29-81 (RxThread).
// Written as scalar integer code with the SSE lane semantics (wrapping / saturating / arithmetic shifts) spelled out;
// the one floating point stage (2x2 channel inverse, sora_matrix.h:135-150,296-304) keeps the reference's single
// precision operation order.
#pragma once
#include "viterbi.h"
#include <vector>

namespace sbo {

struct c32 { int32_t re, im; };

struct Tables11n {
    c16      sincos[65536];        // dsp_math.h:214-231
    int16_t  atan_lut[4097];       // dsp_math.h:233-247
    uint8_t  demap[256];           // dsp_demap.h:97-137 lookup_table_bpsk == lookup_table_qpsk (data, run-length coded)
    uint8_t  crc8[256];            // core/inc/CRC8.h:16-26
    uint8_t  demap16[2][256];      // dsp_demap.h lookup_table_16qam1 / 16qam2 (data, run-length coded), indexed by the uint8 of the limited value
    uint8_t  demap64[3][288];      // dsp_demap.h lookup_table_64qam1..3, indexed by value + 144
    uint16_t deint[4][2][312];     // [bpsk, qpsk, 16-qam, 64-qam][stream][k] : out[k] = in[map]   deinterleaver_11n.hpp:6-1618
    uint8_t  lltf_sign[64];        // 1 where L-LTF carrier is +1      channel_11n.hpp:7-32  (_80211_LLTFMask)
    uint8_t  htltf_sign[64];       // 1 where HT-LTF carrier is +1     channel_11n.hpp:300-325 (_80211n_HTLTFMask)
    Tables11n();
};
const Tables11n& tables11n();

int16_t dsp_atan(int x, int y);                                   // dsp_math.h:166-212 atan(int,int)
uint8_t crc8_htsig(const uint8_t* p, unsigned nbytes, unsigned tail_bits);   // CRC8.h:29-50 CalcCRC8
// first MCS index the HT-SIG parser refuses: 11 as the reference ships it (PHY_11n.hpp:497), 15 with the 16-/64-QAM branches enabled
void set_ht_mcs_limit(uint32_t first_refused);
uint32_t ht_mcs_limit();
struct HtMcs { int nbpsc, cr, ndbps, q; };                         // q = table index 0..3 for N_BPSC 1, 2, 4, 6
bool ht_mcs_params(uint32_t mcs, HtMcs& m);                       // MCS 8..14 (ieee80211n_cmn.h:7-26, ieee80211const.h:35-55)

struct FrameResult11n {
    uint32_t status, mcs, length, crc32, nsym;
    uint32_t sample_index;      // CF_MemSamples::mem_sample_index when the event was seen (40 Msps samples)
    uint32_t detect_index;      // 20 Msps index (since start/seek) of the first vector routed to the L-LTF branch
    int16_t  cfo_est;           // CF_CFOffset::CFO_est
    uint16_t lsig_length;       // 2 x L-SIG LENGTH (PHY_11n.hpp:476)
};

struct Taps11n {
    bool enable = false;
    std::vector<c16> siso[2];              // 64 each: dot11a_siso_channel_1/2
    std::vector<c16> hinv;                 // [4][64]: inv h11, h12, h21, h22
    std::vector<c16> fft_in[2], fft_out[2], eq[2];    // 64 per symbol per antenna/stream (data symbols only for eq; fft_in: what fft64 is handed)
    std::vector<uint8_t> soft;             // stream-parsed soft values per data symbol, concatenated
    std::vector<int16_t> theta;            // vfo_theta_i after each data symbol
    uint8_t sig[9] = {0};
    void clear() { for (int i = 0; i < 2; i++) { siso[i].clear(); fft_in[i].clear(); fft_out[i].clear(); eq[i].clear(); } hinv.clear(); soft.clear(); theta.clear(); }
};

class Rx11n {
public:
    Rx11n() { init(); }
    void init();
    uint32_t push_block28(const c16* a, const c16* b);
    void reset_after_event();
    void reset_carrier_sense();
    int run(const c16* s0, const c16* s1, size_t n, FrameResult11n* res, uint8_t* out, size_t out_stride, int max_frames);
    Taps11n taps;
    // T11nSigParser alone, after the CF_11aRxVector::Reset and error code clear of every event; CF_HTRxVector carries over from the
    // call before, as it does between events.  out = accepted, error_code, data_rate_kbps, frame_length, total_symbols, code_rate,
    // ht_frame_mcs, ht_frame_length
    void sig_parse_only(const uint8_t* sig, uint32_t out[8]);
    // T11aDesc -> TBB11aFrameSink alone, both fresh, for a frame of frame_length_ bytes, fed n decoded bytes; returns error_code
    uint32_t desc_sink_only(const uint8_t* in, size_t n, uint16_t frame_length_);
    uint32_t crc32() const { return frame_crc32; }
    const uint8_t* frame_bytes() const { return frame_buf; }

private:
    enum { SYM_L_LTF = 1, SYM_SIG, SYM_HT_STF, SYM_HT_LTF, SYM_DATA };
    // context
    uint32_t error_code; int cca_state; uint32_t symbol_type;
    uint16_t frame_length, total_symbols, remain_symbols, code_rate; uint32_t data_rate_kbps, frame_crc32;
    uint16_t ht_frame_length; uint32_t ht_frame_mcs; uint16_t lsig_len2;
    int16_t vfo_d, vfo_theta, CFO_est; uint16_t vfo_n;      // NCO: lane k of vfo_delta_i == (int16)((n+k)*d)
    uint32_t mem_sample_index, vec20_count, detect_index;
    // TDownSample2 queue
    c16 ds_q[2][64]; int ds_n;
    // TCCA11n + MimoAutoCorr (never reset between frames: cca_11n.hpp:146-163, autocorr.hpp:9-42)
    c16 his_sample[2][8][4]; c32 his_corr[2][8][4]; int32_t his_energy[2][8][4]; int his_idx;
    c32 corr_sum[2]; int32_t energy_sum[2];
    int64_t his_moving_energy[64]; bool his_valid[64]; int his_index;
    uint32_t sense_count; bool peak_found; int peak_count;
    // framing
    c16 lltf_q[2][128]; int lltf_n;
    c16 sym_q[2][80]; int sym_n;
    c16 sig_q[192]; int sig_n;
    c16 htltf_q[2][128]; int htltf_n;
    c16 siso_ch[2][64]; c16 hinv[4][64];
    // back end
    ViterbiCore vit; uint32_t ob_count; std::vector<uint8_t> vit_in, vit_out;
    uint32_t desc_count; uint8_t desc_reg;
    uint8_t frame_buf[4096]; uint32_t byte_count, crc_run;

    void on_vec20(const c16* a, const c16* b);
    void cca_process(const c16* a, const c16* b);
    void on_lltf();
    void on_symbol();
    void on_sig3();
    void on_htltf();
    void on_data(const c16 Y[2][64]);
    void viterbi_feed(bool flush);
    void rxvector_reset();
    bool parse_sig(const uint8_t* sig);
    void sink_byte(uint8_t b);
};

} // namespace sbo
