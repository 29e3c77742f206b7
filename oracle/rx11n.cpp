// ORACLE — TEST INFRASTRUCTURE ONLY (see ops.h).  802.11n 2x2 receive graph restatement; see rx11n.h.
#include "rx11n.h"
#include "rx11a.h"
#include "tables.h"
#include <cmath>
#include <cstring>
#include <climits>

namespace sbo {

// ---- small lane helpers (vector128.h semantics) --------------------------------------------------------------------
static inline int32_t w32(int64_t x) { return (int32_t)(uint32_t)(uint64_t)x; }
static inline int16_t w16(int32_t x) { return (int16_t)(uint16_t)(uint32_t)x; }
static inline int16_t sat16(int32_t x) { return (int16_t)(x > 32767 ? 32767 : x < -32768 ? -32768 : x); }
static inline int16_t neg16w(int16_t x) { return w16(-(int32_t)x); }                  // psignw / xor-sub negate
// mul(vci,vci,vcs a,vcs b)  vector128.h:1075-1088 : a*b with conj0(b) inside pmaddwd
static inline c32 cmul_s(c16 a, c16 b) {
    c32 r; r.re = w32((int64_t)a.re * b.re + (int64_t)a.im * neg16w(b.im)); r.im = w32((int64_t)a.re * b.im + (int64_t)a.im * b.re); return r;
}
// conj_mul(vci,vci,vcs a,vcs b) vector128.h:1038-1051 : a*conj(b)
static inline c32 cmul_conj(c16 a, c16 b) {
    c32 r; r.re = w32((int64_t)a.re * b.re + (int64_t)a.im * b.im); r.im = w32((int64_t)neg16w(b.im) * a.re + (int64_t)b.re * a.im); return r;
}
static inline c16 shr_pack(c32 v, int n) { c16 r; r.re = sat16(v.re >> n); r.im = sat16(v.im >> n); return r; }

// ---- tables --------------------------------------------------------------------------------------------------------
static const int8_t LLTF[64] = {                        // L-LTF in FFT order (k = 0..31, -32..-1); IEEE 802.11-2007 17.3.3
    0, 1,-1,-1, 1, 1,-1, 1,-1, 1,-1,-1,-1,-1,-1, 1, 1,-1,-1, 1,-1, 1,-1, 1, 1, 1, 1, 0, 0, 0, 0, 0,
    0, 0, 0, 0, 0, 0, 1, 1,-1,-1, 1, 1,-1, 1,-1, 1, 1, 1, 1, 1, 1,-1,-1, 1, 1,-1, 1,-1, 1, 1, 1, 1 };

Tables11n::Tables11n() {
    for (unsigned i = 0; i < 65536; i++) {              // dsp_math.h:214-231
        double r = (double)i * 2.0 * M_PI / 65535.0;
        sincos[i].re = (int16_t)(cos(r) * 32767.5); sincos[i].im = (int16_t)(sin(r) * 32767.5);
    }
    for (int i = 0; i <= 4096; i++) atan_lut[i] = (int16_t)(atan((double)i / 4096.0) / (M_PI / 4.0) * 8192);   // dsp_math.h:233-247
    static const uint8_t rle[8][2] = {{4, 11}, {5, 10}, {6, 10}, {7, 97}, {0, 97}, {1, 10}, {2, 10}, {3, 11}};
    int p = 0; for (auto& r : rle) for (int k = 0; k < r[1]; k++) demap[p++] = r[0];
    for (int b = 0; b < 256; b++) { uint8_t c = (uint8_t)b; for (int k = 0; k < 8; k++) c = (c & 1) ? (uint8_t)((c >> 1) ^ 0xE0) : (uint8_t)(c >> 1); crc8[b] = c; }
    {   // 16-QAM / 64-QAM soft-bit tables (dsp_demap.h, hand-tuned data carried as run lengths; diffed against the header by the tests)
        static const uint8_t r161[][2] = {{4, 5}, {5, 4}, {6, 7}, {7, 112}, {0, 113}, {1, 7}, {2, 4}, {3, 4}};
        static const uint8_t r162[][2] = {{7, 56}, {6, 3}, {5, 3}, {4, 2}, {3, 2}, {2, 2}, {1, 3}, {0, 115}, {1, 3}, {2, 2}, {3, 2}, {4, 2}, {5, 3}, {6, 3}, {7, 55}};
        static const uint8_t r641[][2] = {{0, 138}, {1, 3}, {2, 2}, {3, 1}, {4, 2}, {5, 2}, {6, 3}, {7, 137}};
        static const uint8_t r642[][2] = {{0, 68}, {1, 3}, {2, 2}, {3, 2}, {4, 1}, {5, 2}, {6, 3}, {7, 127}, {6, 3}, {5, 2}, {4, 1}, {3, 2}, {2, 2}, {1, 3}, {0, 67}};
        static const uint8_t r643[][2] = {{0, 34}, {1, 2}, {2, 2}, {3, 2}, {4, 2}, {5, 1}, {6, 3}, {7, 57}, {6, 3}, {5, 2}, {4, 2}, {3, 1}, {2, 2}, {1, 3}, {0, 57},
                                          {1, 3}, {2, 2}, {3, 1}, {4, 2}, {5, 2}, {6, 3}, {7, 57}, {6, 3}, {5, 1}, {4, 2}, {3, 2}, {2, 2}, {1, 2}, {0, 33}};
        auto fill = [](uint8_t* dst, const uint8_t (*r)[2], size_t n) { int p = 0; for (size_t i = 0; i < n; i++) for (int k = 0; k < r[i][1]; k++) dst[p++] = r[i][0]; };
        fill(demap16[0], r161, sizeof r161 / 2); fill(demap16[1], r162, sizeof r162 / 2);
        fill(demap64[0], r641, sizeof r641 / 2); fill(demap64[1], r642, sizeof r642 / 2); fill(demap64[2], r643, sizeof r643 / 2);
    }
    for (int q = 0; q < 4; q++) for (int ss = 0; ss < 2; ss++) {   // IEEE 802.11n-2009 20.3.11.7.3 (== deinterleaver_11n.hpp tables)
        const int nbpsc = q == 3 ? 6 : q == 2 ? 4 : q + 1, ncbpss = 52 * nbpsc, nrow = 4 * nbpsc, ncol = 13, s = nbpsc / 2 > 1 ? nbpsc / 2 : 1;
        for (int k = 0; k < ncbpss; k++) {
            int i = nrow * (k % ncol) + k / ncol;
            int j = s * (i / s) + (i + ncbpss - (ncol * i) / ncbpss) % s;
            int r = ((j - ((ss * 2) % 3 + 3 * (ss / 3)) * 11 * nbpsc) % ncbpss + ncbpss) % ncbpss;
            deint[q][ss][k] = (uint16_t)r;
        }
    }
    for (int i = 0; i < 64; i++) {
        lltf_sign[i] = LLTF[i] == 1;
        int h = LLTF[i]; if (i == 27 || i == 28) h = -1; if (i == 36 || i == 37) h = 1;   // HT-LTF adds carriers +-27, +-28
        htltf_sign[i] = h == 1;
    }
}
const Tables11n& tables11n() { static Tables11n t; return t; }

static uint32_t g_ht_mcs_limit = 11;                    // PHY_11n.hpp:497: `ht_frame_mcs >= 11` is refused
void set_ht_mcs_limit(uint32_t first_refused) { g_ht_mcs_limit = first_refused < 9 ? 9 : first_refused > 15 ? 15 : first_refused; }
uint32_t ht_mcs_limit() { return g_ht_mcs_limit; }
bool ht_mcs_params(uint32_t mcs, HtMcs& m) {
    static const HtMcs P[7] = {{1, CR_12, 52, 0}, {2, CR_12, 104, 1}, {2, CR_34, 156, 1}, {4, CR_12, 208, 2}, {4, CR_34, 312, 2}, {6, CR_23, 416, 3}, {6, CR_34, 468, 3}};
    if (mcs < 8 || mcs > 14) return false;
    m = P[mcs - 8]; return true;
}

int16_t dsp_atan(int x, int y) {                        // dsp_math.h:157-212 (the short overload :90-164 agrees on its range)
    // dsp_math::abs / imax (dsp_math.h:64-88) and the sums are 32-bit int C, which wraps: abs(INT_MIN) = INT_MIN, and
    // tsum = |x| + |y| wraps once either argument passes 2^30
    auto wadd = [](int a, int b) { return (int)((unsigned)a + (unsigned)b); };
    auto wsub = [](int a, int b) { return (int)((unsigned)a - (unsigned)b); };
    auto iabs = [&](int v) { return wsub(v ^ (v >> 31), v >> 31); };
    const int sign = (x ^ y) >> 31;                     // 0 or -1
    const int ax = iabs(x), ay = iabs(y);
    const int tsign = wsub(ax, ay) >> 31;
    const int tsum = wadd(ax, ay), d = iabs(wsub(ax, ay));
    const int tmax = wadd(tsum, d) >> 1, tmin = wsub(tsum, tmax);
    int64_t num = (int64_t)tmin * 65536, den = tmax; if (den == 0) den = 1;
    int idx = (int)((num + (den >> 1)) / den); idx >>= 4;
    if (idx < 0 || idx >= 4097) return 0;
    int16_t srad = tables11n().atan_lut[idx];
    srad = w16((16384 & tsign) + ((srad ^ tsign) - tsign));
    srad = w16((srad ^ sign) - sign);
    return srad;
}

uint8_t crc8_htsig(const uint8_t* p, unsigned nbytes, unsigned tail_bits) {
    uint8_t crc = 0xFF; unsigned i;
    for (i = 0; i < nbytes; i++) crc = tables11n().crc8[crc ^ p[i]];
    if (tail_bits) { crc ^= p[i] & ((1u << tail_bits) - 1); for (unsigned k = 0; k < tail_bits; k++) crc = (crc & 1) ? (uint8_t)((crc >> 1) ^ 0xE0) : (uint8_t)(crc >> 1); }
    return (uint8_t)~crc;
}

// ---- context / graph reset ------------------------------------------------------------------------------------------
void Rx11n::init() {
    memset(his_sample, 0, sizeof his_sample); memset(his_corr, 0, sizeof his_corr); memset(his_energy, 0, sizeof his_energy);
    his_idx = 0; memset(corr_sum, 0, sizeof corr_sum); energy_sum[0] = energy_sum[1] = 0;
    for (int i = 0; i < 64; i++) { his_moving_energy[i] = LLONG_MAX; his_valid[i] = false; }       // cca_11n.hpp:153
    his_index = 0;
    mem_sample_index = 0; vec20_count = 0; detect_index = 0; ds_n = 0;
    vfo_d = 0; vfo_theta = 0; vfo_n = 0; CFO_est = 0; ht_frame_length = 0; ht_frame_mcs = 0;   // CF_HTRxVector has no Reset(): carried across events
    memset(siso_ch, 0, sizeof siso_ch); memset(hinv, 0, sizeof hinv);
    reset_after_event();
}
void Rx11n::reset_carrier_sense() {                    // BB11nDemodContext::ResetCarrierSense + TCCA11n::_reset
    error_code = E_SUCCESS; cca_state = 0; symbol_type = SYM_L_LTF;
    sense_count = 0; peak_found = false; peak_count = 0;
}
void Rx11n::rxvector_reset() {
    frame_length = 0; total_symbols = 0; remain_symbols = 0; data_rate_kbps = 6000; code_rate = CR_12; frame_crc32 = 0;   // CF_11aRxVector::Reset()
    lsig_len2 = 0;                                      // the L-SIG length is frame_length before the HT-SIG overwrites it: zero again when L-SIG is refused
}
void Rx11n::reset_after_event() {                      // ssrc->Flush(); ctx.Reset(); ssrc->Reset()  (fb11n_demod.cpp:64-70)
    reset_carrier_sense();
    rxvector_reset();
    ds_n = 0; lltf_n = sym_n = sig_n = htltf_n = 0;
    vit.max_steps = 5000 * 8; vit.reset(); ob_count = 0; vit_in.clear(); vit_out.assign(256, 0);
    desc_count = 0; desc_reg = 0; byte_count = 0; crc_run = 0xFFFFFFFFu;
}

// ---- TCCA11n (cca_11n.hpp:26-128) over MimoAutoCorr (autocorr.hpp:44-146) ---------------------------------------------
void Rx11n::cca_process(const c16* a, const c16* b) {
    const c16* in[2] = {a, b};
    c32 R[2][4]; int32_t ve[2][4];
    for (int ant = 0; ant < 2; ant++) {
        c32 run = corr_sum[ant]; int32_t es = energy_sum[ant];
        for (int k = 0; k < 4; k++) {
            c32 c = cmul_conj(in[ant][k], his_sample[ant][his_idx][k]); c.re >>= 5; c.im >>= 5;      // vShift = log2(8*4)
            c32 d = { w32((int64_t)c.re - his_corr[ant][his_idx][k].re), w32((int64_t)c.im - his_corr[ant][his_idx][k].im) };
            his_corr[ant][his_idx][k] = c;
            run.re = w32((int64_t)run.re + d.re); run.im = w32((int64_t)run.im + d.im); R[ant][k] = run;
            int32_t e = w32((int64_t)in[ant][k].re * in[ant][k].re + (int64_t)in[ant][k].im * in[ant][k].im) >> 5;
            int32_t de = w32((int64_t)e - his_energy[ant][his_idx][k]); his_energy[ant][his_idx][k] = e;
            es = w32((int64_t)es + de); ve[ant][k] = es;
        }
        for (int k = 0; k < 4; k++) his_sample[ant][his_idx][k] = in[ant][k];
        corr_sum[ant] = run; energy_sum[ant] = es;
    }
    his_idx = (his_idx + 1) % 8;
    for (int k = 0; k < 4; k++) {
        const int32_t cr = w32((int64_t)(R[0][k].re >> 1) + (R[1][k].re >> 1)), ci = w32((int64_t)(R[0][k].im >> 1) + (R[1][k].im >> 1));
        const int64_t acorr = (int64_t)((uint64_t)((int64_t)cr * cr) + (uint64_t)((int64_t)ci * ci));  // SquaredNorm(vci): pmuldq, paddq wraps (vector128.h:922-933)
        const int32_t es = w32((int64_t)(ve[0][k] >> 1) + (ve[1][k] >> 1));
        const int64_t energy = (int64_t)es * es;
        // his + 1 overflows for the LLONG_MAX start value (cca_11n.hpp:153): the quotient is then 0
        const int64_t eb = his_valid[his_index] ? energy / (his_moving_energy[his_index] + 1) : 0;
        if (!peak_found) {
            sense_count++;
            if (eb > 5 && acorr > (energy >> 1)) { sense_count = 0; peak_count++; peak_found = true; }
            else peak_count = 0;
        } else {
            if (acorr < (energy >> 3)) {
                if (peak_count > 96 && peak_count < 160) {
                    peak_found = false; peak_count = 0; cca_state = 1;
                    detect_index = (vec20_count + 1) * 4;
                    break;                                                   // rest of this vector is dropped (ipin.clear())
                }
                peak_found = false; peak_count = 0;
            } else { peak_count++; if (peak_count > 160) { peak_found = false; peak_count = 0; } }
        }
        his_moving_energy[his_index] = energy; his_valid[his_index] = true; his_index = (his_index + 1) % 64;
    }
    if (sense_count >= 84 && cca_state == 0) error_code = E_CS_TIMEOUT;
}

// ---- NCO (freqoffset_11n.hpp:165-216) ------------------------------------------------------------------------------------
static inline c16 nco_rotate(c16 x, uint16_t phase_n_d, int16_t theta) {
    const c16 co = tables11n().sincos[(uint16_t)(phase_n_d - (uint16_t)theta)];
    return shr_pack(cmul_s(x, co), 15);
}

// ---- L-LTF: joint CFO estimate, compensate, FFT, SISO channel (freqoffset_11n.hpp:42-163, channel_11n.hpp:34-218) -------
static void siso_est64(const c16* Y, c16* ch) {
    const Tables11n& T = tables11n();
    for (int v = 0; v < 16; v++) {
        if (v == 7 || v == 8) { for (int j = 0; j < 4; j++) ch[4 * v + j] = c16{0, 0}; continue; }   // not written by the reference
        int32_t sq[4], in[8];
        for (int j = 0; j < 4; j++) { sq[j] = w32((int64_t)Y[4 * v + j].re * Y[4 * v + j].re + (int64_t)Y[4 * v + j].im * Y[4 * v + j].im);
                                      in[2 * j] = w32((int64_t)Y[4 * v + j].re << 16); in[2 * j + 1] = w32((int64_t)Y[4 * v + j].im << 16); }
        for (int j = 0; j < 8; j++) in[j] = w32((int64_t)in[j] + (sq[j & 3] >> 1));     // rounding term added lane-wise (channel_11n.hpp:52-55)
        for (int j = 0; j < 4; j++) {
            int32_t d = sq[j] ? sq[j] : 1;
            c16 o; o.re = sat16((int32_t)((int64_t)in[2 * j] / d)); o.im = sat16((int32_t)((int64_t)in[2 * j + 1] / d));
            if (T.lltf_sign[4 * v + j]) o.im = neg16w(o.im); else o.re = neg16w(o.re);
            ch[4 * v + j] = o;
        }
    }
}

void Rx11n::on_lltf() {
    // v_estimate_i(ip1, ip2, 16, 16)
    int64_t sr = 0, si = 0;
    for (int ant = 0; ant < 2; ant++)
        for (int i = 0; i < 64; i++) { c32 c = cmul_conj(lltf_q[ant][i], lltf_q[ant][i + 64]); sr += c.re >> 7; si += c.im >> 7; }
    int16_t delta = dsp_atan(w32(sr), w32(si)); delta = (int16_t)(delta >> 6);
    CFO_est = delta; vfo_d = delta; vfo_theta = 0; vfo_n = 0;
    alignas(16) c16 x[2][128], F[64], ch1[64], ch2[64];
    for (int i = 0; i < 128; i++) {
        const uint16_t ph = (uint16_t)(vfo_n * (uint16_t)vfo_d); vfo_n++;
        for (int ant = 0; ant < 2; ant++) x[ant][i] = nco_rotate(lltf_q[ant][i], ph, vfo_theta);
    }
    for (int ant = 0; ant < 2; ant++) {
        alignas(16) c16 t[64];
        memcpy(t, x[ant], sizeof t);      if (taps.enable) taps.fft_in[ant].insert(taps.fft_in[ant].end(), t, t + 64);
        fft64((v128*)t, (v128*)F); siso_est64(F, ch1);
        if (taps.enable) taps.fft_out[ant].insert(taps.fft_out[ant].end(), F, F + 64);
        memcpy(t, x[ant] + 64, sizeof t); if (taps.enable) taps.fft_in[ant].insert(taps.fft_in[ant].end(), t, t + 64);
        fft64((v128*)t, (v128*)F); siso_est64(F, ch2);
        if (taps.enable) taps.fft_out[ant].insert(taps.fft_out[ant].end(), F, F + 64);
        for (int i = 0; i < 64; i++) { siso_ch[ant][i].re = (int16_t)(w16(ch1[i].re + ch2[i].re) >> 1); siso_ch[ant][i].im = (int16_t)(w16(ch1[i].im + ch2[i].im) >> 1); }
        if (taps.enable) taps.siso[ant].assign(siso_ch[ant], siso_ch[ant] + 64);
    }
    symbol_type = SYM_SIG;
}

// ---- one 80-sample OFDM symbol of either kind (PHY_11n.hpp:283-354, fb11ndemod_config.hpp:112-129) -----------------------
void Rx11n::on_symbol() {
    alignas(16) c16 Y[2][64];
    for (int ant = 0; ant < 2; ant++) {
        alignas(16) c16 t[64]; memcpy(t, sym_q[ant] + 16, sizeof t);                   // skip_cp = 16
        if (taps.enable) taps.fft_in[ant].insert(taps.fft_in[ant].end(), t, t + 64);
        fft64((v128*)t, (v128*)Y[ant]);
        if (taps.enable) taps.fft_out[ant].insert(taps.fft_out[ant].end(), Y[ant], Y[ant] + 64);
    }
    switch (symbol_type) {
    case SYM_SIG: {                                                                        // TSisoChannelComp + TMrcCombine
        for (int i = 0; i < 64; i++) {
            c16 o1 = shr_pack(cmul_s(Y[0][i], siso_ch[0][i]), 9), o2 = shr_pack(cmul_s(Y[1][i], siso_ch[1][i]), 9);
            sig_q[sig_n + i].re = (int16_t)(w16(o1.re + o2.re) >> 1); sig_q[sig_n + i].im = (int16_t)(w16(o1.im + o2.im) >> 1);
        }
        sig_n += 64; if (sig_n == 192) { on_sig3(); sig_n = 0; }
        break; }
    case SYM_HT_STF: symbol_type = SYM_HT_LTF; break;                                     // dropped
    case SYM_HT_LTF:
        for (int ant = 0; ant < 2; ant++) memcpy(htltf_q[ant] + htltf_n, Y[ant], 64 * sizeof(c16));
        htltf_n += 64; if (htltf_n == 128) { on_htltf(); htltf_n = 0; }
        break;
    default: on_data(Y); break;
    }
    remain_symbols--;
    if (remain_symbols == 0) { viterbi_feed(true); if (error_code == E_SUCCESS) error_code = E_FAILED; }
}

static uint64_t viterbi_sig_bits(const uint8_t* soft, int nbits) {                     // viterbicore.h:36-261 Viterbi_sig11(..., output_bit)
    ViterbiCore v; v.max_steps = 96; v.reset();
    for (int i = 0; i < nbits; i++) { v.step_ab(soft[2 * i], soft[2 * i + 1]); if ((v.steps & 7) == 0) v.normalize(); }
    v.normalize();
    uint8_t out[8] = {0}; v.traceback(out, (uint32_t)nbits, 0);
    uint64_t w = 0; for (int i = 0; i < nbits / 8; i++) w |= (uint64_t)out[i] << (8 * i);
    return w >> 6;
}

void Rx11n::on_sig3() {                                // T11nSigDemap, T11aDeinterleaveBPSK, T11nViterbiSig, T11nSigParser
    const Tables11n& T = tables11n();
    uint8_t soft[144], dsoft[144]; int j = 0;
    for (int s = 0; s < 3; s++)
        for (int pass = 0; pass < 2; pass++)
            for (int i = pass ? 1 : 38; i <= (pass ? 26 : 63); i++) {
                if (i == 43 || i == 57 || i == 7 || i == 21) continue;
                int16_t v = s == 0 ? sig_q[64 * s + i].re : sig_q[64 * s + i].im;
                v = v < -128 ? -128 : v > 127 ? 127 : v;
                soft[j++] = T.demap[(uint8_t)v];
            }
    for (int s = 0; s < 3; s++) deinterleave(soft + 48 * s, dsoft + 48 * s, 48);
    uint8_t sig[12] = {0};
    uint32_t lsig = (uint32_t)viterbi_sig_bits(dsoft, 24); memcpy(sig, &lsig, 4);
    uint64_t ht = viterbi_sig_bits(dsoft + 48, 48); memcpy(sig + 3, &ht, 6);
    if (taps.enable) memcpy(taps.sig, sig, 9);
    if (!parse_sig(sig)) { error_code = E_PLCP_HEADER_FAIL; return; }
    frame_length = ht_frame_length;
    symbol_type = SYM_HT_STF;
}

// T11nSigParser::_parse_plcp and _parse_htsig (PHY_11n.hpp:458-513) on the 9 bytes T11nViterbiSig hands it
bool Rx11n::parse_sig(const uint8_t* sig) {
    uint32_t u; memcpy(&u, sig, 4); u &= 0xFFFFFF;
    bool ok = !(u & 0xFC0010);
    if (ok) { uint32_t p = (u >> 16) ^ u; p ^= p >> 8; p ^= p >> 4; p ^= p >> 2; p ^= p >> 1; ok = !(p & 1); }
    if (ok) { static const uint32_t rates[8] = {48000, 24000, 12000, 6000, 54000, 36000, 18000, 9000};
              data_rate_kbps = (u & 8) ? rates[u & 7] : 0; ok = data_rate_kbps != 0; }
    if (ok) { frame_length = (uint16_t)(((u >> 5) & 0xFFF) * 2); lsig_len2 = frame_length; ok = frame_length <= 1500; }
    if (ok) {                                                                               // _parse_htsig
        const uint8_t* ip = sig + 3;
        uint8_t c = crc8_htsig(ip, 4, 2);
        // compared as int, as PHY_11n.hpp:488 compares its UCHAR with an int: a byte 5 above 3 fails the check.  The SIG decoder's >> 6
        // leaves byte 5 at most 3, so a receiver never gets there; the parser on its own does
        if (c != ((ip[4] >> 2) | (ip[5] << 6))) { ht_frame_mcs = 0; ht_frame_length = 0; ok = false; }
        else {
            ht_frame_mcs = ip[0] & 0x7F;
            if (ht_frame_mcs < 8 || ht_frame_mcs >= ht_mcs_limit()) ok = false;
            else {
                ht_frame_length = (uint16_t)(ip[1] | (ip[2] << 8));
                if (ht_frame_length > 1500) ok = false;
                else {
                    HtMcs m; ht_mcs_params(ht_frame_mcs, m);
                    code_rate = (uint16_t)m.cr;                                            // ieee80211n_cmn.h:7-26
                    total_symbols = (uint16_t)((ht_frame_length * 8 + 16 + 6 + m.ndbps - 1) / m.ndbps + 4); remain_symbols = total_symbols;
                }
            }
        }
    }
    return ok;
}
void Rx11n::sig_parse_only(const uint8_t* sig, uint32_t out[8]) {
    error_code = E_SUCCESS; rxvector_reset();
    if (parse_sig(sig)) frame_length = ht_frame_length; else error_code = E_PLCP_HEADER_FAIL;
    out[0] = error_code == E_SUCCESS; out[1] = error_code; out[2] = data_rate_kbps; out[3] = frame_length; out[4] = total_symbols; out[5] = code_rate;
    out[6] = ht_frame_mcs; out[7] = ht_frame_length;
}
uint32_t Rx11n::desc_sink_only(const uint8_t* in, size_t n, uint16_t frame_length_) {
    error_code = E_SUCCESS; frame_length = frame_length_; frame_crc32 = 0; desc_count = 0; desc_reg = 0; byte_count = 0; crc_run = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; i++) sink_byte(in[i]);
    return error_code;
}

// ---- HT-LTF: 2x2 channel and its inverse (channel_11n.hpp:331-442, sora_matrix.h:135-150,296-304) ------------------------
struct cf { float re, im; };
static inline cf cmulf(cf a, cf b) { cf r; r.re = a.re * b.re - a.im * b.im; r.im = a.im * b.re + a.re * b.im; return r; }
static inline int32_t cvtps(float x) { if (!(x >= -2147483648.0f && x < 2147483648.0f)) return INT_MIN; return (int32_t)lrintf(x); }   // cvtps2dq

void Rx11n::on_htltf() {
    const Tables11n& T = tables11n();
    for (int i = 0; i < 64; i++) {
        c16 h[4];
        for (int ant = 0; ant < 2; ant++) {
            const c16 a = htltf_q[ant][i], b = htltf_q[ant][i + 64];
            c16 d, s;
            d.re = (int16_t)(sat16((int32_t)a.re - b.re) >> 1); d.im = (int16_t)(sat16((int32_t)a.im - b.im) >> 1);
            s.re = (int16_t)(sat16((int32_t)a.re + b.re) >> 1); s.im = (int16_t)(sat16((int32_t)a.im + b.im) >> 1);
            if (!T.htltf_sign[i]) { d.re = neg16w(d.re); d.im = neg16w(d.im); s.re = neg16w(s.re); s.im = neg16w(s.im); }
            h[2 * ant] = d; h[2 * ant + 1] = s;
        }
        const cf a = {(float)h[0].re, (float)h[0].im}, b = {(float)h[1].re, (float)h[1].im}, c = {(float)h[2].re, (float)h[2].im}, d = {(float)h[3].re, (float)h[3].im};
        const cf ad = cmulf(a, d), bc = cmulf(b, c);
        const cf det = {ad.re - bc.re, ad.im - bc.im};
        const float n = (det.re * det.re + det.im * det.im) / 65536.0f;
        const cf ds = {det.re, -det.im};
        const cf nb = {-b.re, -b.im}, nc = {-c.re, -c.im};
        const cf r[4] = {cmulf(d, ds), cmulf(nb, ds), cmulf(nc, ds), cmulf(a, ds)};
        for (int q = 0; q < 4; q++) { hinv[q][i].re = sat16(cvtps(r[q].re / n)); hinv[q][i].im = sat16(cvtps(r[q].im / n)); }
    }
    if (taps.enable) { taps.hinv.clear(); for (int q = 0; q < 4; q++) taps.hinv.insert(taps.hinv.end(), hinv[q], hinv[q] + 64); }
    symbol_type = SYM_DATA;
}

// ---- data symbol: TMimoChannelComp, TPilotTrack_11n, demap, HT deinterleave, stream de-parse -----------------------------
void Rx11n::on_data(const c16 Y[2][64]) {
    const Tables11n& T = tables11n();
    c16 X[2][64];
    for (int i = 0; i < 64; i++)
        for (int s = 0; s < 2; s++) {
            c32 p = cmul_s(hinv[2 * s][i], Y[0][i]), q = cmul_s(hinv[2 * s + 1][i], Y[1][i]);
            c32 t = { w32((int64_t)p.re + q.re), w32((int64_t)p.im + q.im) };
            X[s][i] = shr_pack(t, 9);
        }
    if (taps.enable) for (int s = 0; s < 2; s++) taps.eq[s].insert(taps.eq[s].end(), X[s], X[s] + 64);
    int16_t th[2];
    for (int s = 0; s < 2; s++) {                                                          // pilot_11n.hpp:84-97 (no polarity: atan is pi-periodic)
        int sum = dsp_atan(X[s][43].re, X[s][43].im) + dsp_atan(X[s][57].re, X[s][57].im) + dsp_atan(X[s][7].re, X[s][7].im) + dsp_atan(X[s][21].re, X[s][21].im);
        th[s] = w16(sum >> 2);
    }
    vfo_theta = w16(vfo_theta + w16((th[0] + th[1]) >> 1));
    if (taps.enable) taps.theta.push_back(vfo_theta);
    HtMcs m; ht_mcs_params(ht_frame_mcs, m);
    const int q = m.q, nss = 52 * m.nbpsc;
    uint8_t soft[2][312], dso[2][312];
    for (int s = 0; s < 2; s++) {
        int j = 0;
        for (int pass = 0; pass < 2; pass++)
            for (int i = pass ? 1 : 36; i <= (pass ? 28 : 63); i++) {
                if (i == 43 || i == 57 || i == 7 || i == 21) continue;
                int16_t re = X[s][i].re, im = X[s][i].im;
                re = re < -128 ? -128 : re > 127 ? 127 : re; im = im < -128 ? -128 : im > 127 ? 127 : im;     // demap_limit with DemapMin / DemapMax, all four demappers
                if (q <= 1) { soft[s][j++] = T.demap[(uint8_t)re]; if (q) soft[s][j++] = T.demap[(uint8_t)im]; }
                else if (q == 2) {                                                                             // dsp_demap.h demap_16qam
                    soft[s][j++] = T.demap16[0][(uint8_t)re]; soft[s][j++] = T.demap16[1][(uint8_t)re];
                    soft[s][j++] = T.demap16[0][(uint8_t)im]; soft[s][j++] = T.demap16[1][(uint8_t)im];
                } else {                                                                                       // demap_64qam: tables based at entry 144
                    for (int t = 0; t < 3; t++) soft[s][j++] = T.demap64[t][144 + re];
                    for (int t = 0; t < 3; t++) soft[s][j++] = T.demap64[t][144 + im];
                }
            }
        for (int k = 0; k < nss; k++) dso[s][k] = soft[s][T.deint[q][s][k]];
    }
    const int S = m.nbpsc / 2 > 1 ? m.nbpsc / 2 : 1;                                                            // TStreamJoin<2, N> + TStreamConcat<2, S>: S values of stream 0, S of stream 1, ...
    const size_t base = vit_in.size(); vit_in.resize(base + 2 * nss);
    for (int k = 0; k < nss; k++) { vit_in[base + (2 * (k / S)) * S + k % S] = dso[0][k]; vit_in[base + (2 * (k / S) + 1) * S + k % S] = dso[1][k]; }
    if (taps.enable) taps.soft.insert(taps.soft.end(), vit_in.begin() + base, vit_in.end());
    viterbi_feed(false);
}

// T11aViterbi<5000*8, 312, 192, 36> behind a 312-value pin queue; Flush pads the queue with zeros (brick.h:461, pinqueue.h:133-143)
void Rx11n::viterbi_feed(bool flush) {
    if (flush && !vit_in.empty()) vit_in.resize((vit_in.size() + 311) / 312 * 312, 0);
    size_t pos = 0;
    while (vit_in.size() - pos >= 312) {
        if (error_code != E_SUCCESS) { pos = vit_in.size(); break; }
        size_t n = viterbi_decode_block(vit, vit_in.data() + pos, 312, code_rate, frame_length, 192, 36, vit_out.data(), ob_count);
        for (size_t i = 0; i < n; i++) sink_byte(vit_out[i]);
        pos += 312;
    }
    vit_in.erase(vit_in.begin(), vit_in.begin() + pos);
}

void Rx11n::sink_byte(uint8_t b) {                     // T11aDesc (scramble.hpp:189-260) + TBB11aFrameSink (PHY_11a.hpp:630-711)
    desc_count++;
    if (desc_count == 1) return;
    if (desc_count == 2) { desc_reg = b >> 1; return; }
    desc_reg = tables().scramble_lut[desc_reg];
    uint8_t o = b ^ desc_reg; desc_reg >>= 1;
    if (byte_count < (uint32_t)((int)frame_length - 4)) {
        frame_buf[byte_count++ & 4095] = o;
        crc_run = (crc_run >> 8) ^ tables().crc32_lut[o ^ (crc_run & 0xFF)];
    } else if (byte_count < (uint32_t)frame_length) {
        frame_buf[byte_count++ & 4095] = o;
        if (byte_count == frame_length) {
            uint32_t fcs; memcpy(&fcs, frame_buf + byte_count - 4, 4);
            frame_crc32 = fcs;
            error_code = (~crc_run == fcs) ? E_FRAME_OK : E_CRC32_FAIL;
        }
    }
}

// ---- routing (fb11ndemod_config.hpp:103-115 rx_switch) and the source (memsource.hpp:189-244, samples.hpp:27-49) ----------
void Rx11n::on_vec20(const c16* a, const c16* b) {
    if (cca_state == 0) cca_process(a, b);
    else if (symbol_type == SYM_L_LTF) {
        memcpy(lltf_q[0] + lltf_n, a, 4 * sizeof(c16)); memcpy(lltf_q[1] + lltf_n, b, 4 * sizeof(c16)); lltf_n += 4;
        if (lltf_n == 128) { on_lltf(); lltf_n = 0; }
    } else {
        for (int k = 0; k < 4; k++) {                                                      // TFreqComp_11n in bursts of 8: phase depends on the sample count only
            const uint16_t ph = (uint16_t)(vfo_n * (uint16_t)vfo_d); vfo_n++;
            sym_q[0][sym_n + k] = nco_rotate(a[k], ph, vfo_theta); sym_q[1][sym_n + k] = nco_rotate(b[k], ph, vfo_theta);
        }
        sym_n += 4;
        if (sym_n == 80) { sym_n = 0; on_symbol(); }
    }
    vec20_count++;
}

uint32_t Rx11n::push_block28(const c16* a, const c16* b) {
    memcpy(ds_q[0] + ds_n, a, 28 * sizeof(c16)); memcpy(ds_q[1] + ds_n, b, 28 * sizeof(c16)); ds_n += 28; mem_sample_index += 28;
    int r = 0;
    while (ds_n - r >= 8) {
        c16 va[4], vb[4];
        for (int k = 0; k < 4; k++) { va[k] = ds_q[0][r + 2 * k]; vb[k] = ds_q[1][r + 2 * k]; }
        on_vec20(va, vb);
        r += 8;
    }
    memmove(ds_q[0], ds_q[0] + r, (size_t)(ds_n - r) * sizeof(c16)); memmove(ds_q[1], ds_q[1] + r, (size_t)(ds_n - r) * sizeof(c16)); ds_n -= r;
    return error_code;
}

int Rx11n::run(const c16* s0, const c16* s1, size_t n, FrameResult11n* res, uint8_t* out, size_t out_stride, int max_frames) {
    init();
    int nf = 0;
    const size_t nblk = n / 28;
    for (size_t b = 0; b < nblk && nf < max_frames; b++) {
        uint32_t err = push_block28(s0 + 28 * b, s1 + 28 * b);
        if (err == E_SUCCESS) continue;
        if (err == E_CS_TIMEOUT) { reset_carrier_sense(); continue; }
        FrameResult11n& r = res[nf];
        r.status = err; r.mcs = ht_frame_mcs; r.length = frame_length; r.crc32 = frame_crc32; r.nsym = total_symbols;
        r.sample_index = mem_sample_index; r.detect_index = detect_index; r.cfo_est = CFO_est; r.lsig_length = lsig_len2;
        if (out) { size_t nb = frame_length < out_stride ? frame_length : out_stride; memcpy(out + (size_t)nf * out_stride, frame_buf, nb); }
        nf++;
        reset_after_event();
    }
    return nf;
}

} // namespace sbo
