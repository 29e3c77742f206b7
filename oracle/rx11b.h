// ORACLE — TEST INFRASTRUCTURE ONLY (see ops.h).  802.11b receive chain (see rx11b.cpp).
#pragma once
#include "rx11a.h"

namespace sbo {

enum : uint32_t { E_SFD_FAIL = 0x80000004u, E_SFD_TIMEOUT = 0x80000008u, E_SYNC_TIMEOUT = 0x80000009u };

struct FrameResult11b { uint32_t status, rate_kbps, length, crc32, sample_index, detect_vec; };

uint8_t cck11_decode(const c16* P, c16& last, int& even);
uint8_t cck5_decode(const c16* P, c16& last);
c16 barker_despread(const c16* chips11);
uint8_t dbpsk_demap(const c16* sym8, c16& last);
uint8_t dqpsk_demap(const c16* sym4, c16& last);

class Rx11b {
public:
    Rx11b();
    void init();
    uint32_t push_block28(const c16* s);
    int run(const c16* samples, size_t n, FrameResult11b* res, uint8_t* out, size_t out_stride, int max_frames);
    uint32_t cca_pwr_threshold = 1000 * 1000;
private:
    uint32_t error_code; int cca_state, rate_state, plcp_state;
    c16 DC, last_symbol; uint8_t byte_reg; uint16_t frame_length; uint32_t data_rate_kbps, frame_crc32, mem_sample_index, vec_count, detect_vec;
    uint32_t avg_energy, win[8], win_idx, ed_count;
    uint32_t dc_update_cnt; c16 dc_sum;
    int m_index, m_frag; c16 st_q[28]; int st_n;
    int bs_state, bs_last_peak, bs_max, bs_search; c16 bs_partial[11];
    c16 dsp_q[11]; int dsp_n; c16 sym_q[8]; int sym_n; c16 cck_q[16]; int cck_n; int cck_even;
    bool sfd_one; uint16_t sfd_word; int sfd_err; uint32_t sfd_cnt;
    uint8_t hdr[6]; int hdr_n;
    uint8_t frame_buf[4096]; uint32_t byte_count, crc_run;
    void ctx_reset(); void bricks_reset();
    void dcest(const c16* v); void energy_detect(const c16* v);
    void sym_timing(c16* blk); void barker_sync(c16 in); void on_chip(c16 s); void on_byte(uint8_t b);
};

} // namespace sbo
