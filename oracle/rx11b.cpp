// ORACLE — TEST INFRASTRUCTURE ONLY (see ops.h).
// 802.11b (DSSS / CCK) receive chain, restated from the reference bricks of
//   kernel/bb/demod11/fb11bdemod_config.hpp:123-180 (CreateDemodGraph), driven like MAC11b_Receive
//   (kernel/bb/demod11/fb11b_demod.cpp:26-79).  44 Msps input, 4 samples per chip.
#include "rx11b.h"
#include <stdlib.h>

namespace sbo {

static inline int16_t w16(int v) { return (int16_t)v; }
static inline c16 csub(c16 a, c16 b) { return c16{w16(a.re - b.re), w16(a.im - b.im)}; }     // complex_ext.h:106-108 (short results)
static inline c16 cadd(c16 a, c16 b) { return c16{w16(a.re + b.re), w16(a.im + b.im)}; }
static inline c16 csra(c16 a, int n) { return c16{w16(a.re >> n), w16(a.im >> n)}; }
static inline int cnorm2(c16 a) { return a.re * a.re + a.im * a.im; }
// int32 arithmetic of the reference's scalar C and SSE code, which wraps (two's complement, paddd / pmaddwd / psubd)
static inline int32_t wadd(int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); }
static inline int32_t wsub(int32_t a, int32_t b) { return (int32_t)((uint32_t)a - (uint32_t)b); }
static inline int32_t wneg(int32_t a) { return (int32_t)(0u - (uint32_t)a); }

static uint16_t g_crc16_lut[256];
static bool build_crc16() {                 // CCITT CRC-16 reflected (0x8408), core/inc/CRC16.h:37-48
    for (unsigned i = 0; i < 256; i++) { unsigned c = i; for (int k = 0; k < 8; k++) c = (c & 1) ? 0x8408u ^ (c >> 1) : c >> 1; g_crc16_lut[i] = (uint16_t)c; }
    return true;
}
static uint16_t crc16(const uint8_t* p, unsigned n) {
    uint16_t c = 0xFFFF;
    for (unsigned i = 0; i < n; i++) c = (uint16_t)((c >> 8) ^ g_crc16_lut[(c & 0xFF) ^ p[i]]);
    return (uint16_t)~c;
}

Rx11b::Rx11b() { tables(); static const bool crc_ready = build_crc16(); (void)crc_ready; init(); }

void Rx11b::bricks_reset() {               // every brick's Reset(): queues cleared, local state re-initialised
    // TEnergyDetect (cca.hpp:35-40)
    avg_energy = 0; memset(win, 0, sizeof win); win_idx = 0; ed_count = 0;
    // TDCEstimator (dc.hpp:119-122)
    dc_update_cnt = 8; dc_sum = c16{0, 0};
    // TSymTiming (symtiming.hpp:21-24)
    m_index = 2; m_frag = 0; st_n = 0;
    // TBarkerSync (symtiming.hpp:208-214)
    bs_state = 0; bs_last_peak = -1; bs_max = 0; bs_search = 0; memset(bs_partial, 0, sizeof bs_partial);
    // despreaders / demappers / decoders: pin queues
    dsp_n = 0; sym_n = 0; cck_n = 0; cck_even = 0;
    // TSFDSync (sfd_sync.hpp:30-35)
    sfd_one = false; sfd_word = 0; sfd_err = 0; sfd_cnt = 0;
    hdr_n = 0;
    // TBB11bFrameSink (PHY_11b.hpp:672-682)
    byte_count = 0; crc_run = 0xFFFFFFFFu;
}
void Rx11b::ctx_reset() {                  // fb11bdemod_config.hpp:64-77 reset()
    error_code = E_SUCCESS; cca_state = 0; rate_state = 0; plcp_state = 0;
}
void Rx11b::init() {                       // fb11bdemod_config.hpp:79-98 init()
    DC = c16{0, 0}; last_symbol = c16{0, 0}; byte_reg = 0; frame_length = 0; data_rate_kbps = 0; frame_crc32 = 0;
    mem_sample_index = 0; vec_count = 0; detect_vec = 0;
    ctx_reset(); bricks_reset();
}

// ---- TDCEstimator (dc.hpp:101-166) on one 4-sample vector (scalar DC: all four vcs lanes are equal) ----
void Rx11b::dcest(const c16* v) {
    int hr = 0, hi = 0;
    for (int k = 0; k < 4; k++) { hr += v[k].re >> 5; hi += v[k].im >> 5; }
    dc_sum = c16{w16(dc_sum.re + w16(hr)), w16(dc_sum.im + w16(hi))};
    if (dc_update_cnt == 0) { DC = c16{w16(DC.re + (dc_sum.re >> 2)), w16(DC.im + (dc_sum.im >> 2))}; dc_update_cnt = 8; dc_sum = c16{0, 0}; }
    dc_update_cnt--;
}

// ---- TEnergyDetect (cca.hpp:13-98) ----
void Rx11b::energy_detect(const c16* v) {
    if (error_code == E_CS_TIMEOUT) return;            // `ipin.clear(); return 0`: later vectors of the block still arrive, see below
    uint32_t p = 0;
    // hadd(shift_right(SquaredNorm(pi), 5)) (cca.hpp:65): pmaddwd wraps (-32768, -32768) to INT_MIN, psrad 5 keeps the sign, the hadd wraps
    for (int k = 0; k < 4; k++) p += (uint32_t)(wadd(v[k].re * v[k].re, v[k].im * v[k].im) >> 5);
    avg_energy = avg_energy - win[win_idx] + p; win[win_idx] = p; win_idx = (win_idx + 1) & 7;
    ed_count++;
    if (ed_count >= 32) {
        if (ed_count >= 100) { error_code = E_CS_TIMEOUT; return; }
        if (avg_energy >= cca_pwr_threshold) { cca_state = 1; detect_vec = vec_count + 1; }
    }
    if (cca_state != 1) dcest(v);
}

// ---- CCK correlators (cck.hpp:71-780) ----
struct Pick { int32_t max; uint8_t val; };
static inline int32_t mul32(int32_t a, int32_t b) { return (int32_t)((uint32_t)a * (uint32_t)b); }
// best of the four phi3/phi4 hypotheses for one phi2 module (cck.hpp:283-372: B butterflies, L products, arg-max)
static Pick cck11_module(int32_t a1r, int32_t a1i, int32_t a2r, int32_t a2i, int32_t a3r, int32_t a3i, int32_t a4r, int32_t a4i) {
    int32_t b0r[2], b0i[2], b1r[2], b1i[2], b2r[2], b2i[2], b3r[2], b3i[2];
    b0r[0] = a2r + a1r; b0i[0] = a2i + a1i; b1r[0] = a2r - a1r; b1i[0] = a2i - a1i;
    b0r[1] = a2r - a1i; b0i[1] = a2i + a1r; b1r[1] = a2r + a1i; b1i[1] = a2i - a1r;
    b2r[0] = a4r + a3r; b2i[0] = a4i + a3i; b3r[0] = a4r - a3r; b3i[0] = a4i - a3i;
    b2r[1] = a4r - a3i; b2i[1] = a4i + a3r; b3r[1] = a4r + a3i; b3i[1] = a4i - a3r;
    for (int k = 0; k < 2; k++) { b0r[k] >>= 2; b0i[k] >>= 2; b1r[k] >>= 2; b1i[k] >>= 2; b2r[k] >>= 2; b2i[k] >>= 2; b3r[k] >>= 2; b3i[k] >>= 2; }
    int32_t Lr[4], Li[4];
    // cck.hpp:300-307 and the abs / negations below are 32-bit int C: full-scale chips wrap them
    Lr[0] = wadd(mul32(b0r[0], b2r[0]), mul32(b0i[0], b2i[0])); Li[0] = wsub(mul32(b0r[0], b2i[0]), mul32(b0i[0], b2r[0]));
    Lr[1] = wadd(mul32(b0r[1], b2r[1]), mul32(b0i[1], b2i[1])); Li[1] = wsub(mul32(b0r[1], b2i[1]), mul32(b0i[1], b2r[1]));
    Lr[2] = wadd(mul32(b1r[0], b3r[0]), mul32(b1i[0], b3i[0])); Li[2] = wsub(mul32(b1r[0], b3i[0]), mul32(b1i[0], b3r[0]));
    Lr[3] = wadd(mul32(b1r[1], b3r[1]), mul32(b1i[1], b3i[1])); Li[3] = wsub(mul32(b1r[1], b3i[1]), mul32(b1i[1], b3r[1]));
    static const uint8_t base[4] = {0x00, 0x30, 0x10, 0x20};
    int32_t mx[4]; uint8_t vl[4];
    for (int k = 0; k < 4; k++) {
        int32_t ar = Lr[k] < 0 ? wneg(Lr[k]) : Lr[k], ai = Li[k] < 0 ? wneg(Li[k]) : Li[k];
        if (ar > ai) { if (Lr[k] > 0) { mx[k] = Lr[k]; vl[k] = base[k] | 0x00; } else { mx[k] = wneg(Lr[k]); vl[k] = base[k] | 0x40; } }
        else         { if (Li[k] > 0) { mx[k] = Li[k]; vl[k] = base[k] | 0xC0; } else { mx[k] = wneg(Li[k]); vl[k] = base[k] | 0x80; } }
    }
    Pick p;
    if (mx[0] > mx[1]) { p.max = mx[0]; p.val = vl[0]; } else { p.max = mx[1]; p.val = vl[1]; }
    if (mx[2] > mx[3]) { if (mx[2] > p.max) { p.max = mx[2]; p.val = vl[2]; } }
    else               { if (mx[3] > p.max) { p.max = mx[3]; p.val = vl[3]; } }
    return p;
}
static inline void dqpsk_bits(uint8_t& r, int pos, c16 ref, c16 s) {       // TDQPSKDemap::demap_dqpsk_bits (barkerspread.hpp:432-439)
    // MSVC's 32-bit long: re + im and re - im wrap when both products are near 2^30 (the despread symbols of the chain stay below that)
    int32_t re = wadd(ref.re * s.re, ref.im * s.im), im = wsub(ref.re * s.im, ref.im * s.re);
    r |= (uint8_t)(((uint32_t)wadd(re, im) >> 31) << pos);
    r |= (uint8_t)(((uint32_t)wsub(re, im) >> 31) << (pos + 1));
}
static inline void cck_dqpsk_bits(uint8_t& r, int pos, c16 ref, c16 s) {   // the free demap_dqpsk_bits the CCK decoders call (soradsp.h:190-199)
    // it halves re and im before the sums (:194-195), so re + im and re - im never wrap; re itself wraps to INT_MIN when both products
    // are 2^30 (a raw chip of -32768, -32768 against its like: after a CCK symbol `ref` is a raw chip)
    int32_t re = wadd(ref.re * s.re, ref.im * s.im) >> 1, im = wsub(ref.re * s.im, ref.im * s.re) >> 1;
    r |= (uint8_t)(((uint32_t)(re + im) >> 31) << pos);
    r |= (uint8_t)(((uint32_t)(re - im) >> 31) << (pos + 1));
}
uint8_t cck11_decode(const c16* P, c16& last, int& even) {                  // cck.hpp:262-769 CCK11_DECODER
    int32_t p[8][2]; for (int i = 0; i < 8; i++) { p[i][0] = P[i].re; p[i][1] = P[i].im; }
#define R(i) p[i][0]
#define I(i) p[i][1]
    Pick m1 = cck11_module(R(0) + R(1), I(0) + I(1), R(2) - R(3), I(2) - I(3), R(4) + R(5), I(4) + I(5), R(7) - R(6), I(7) - I(6));
    Pick m2 = cck11_module(I(0) + R(1), I(1) - R(0), I(2) - R(3), -(R(2) + I(3)), I(4) + R(5), I(5) - R(4), R(7) - I(6), R(6) + I(7));
    m2.val |= 0x08;
    uint8_t out;
    if (m1.max > m2.max) {                                                  // lable4 (cck.hpp:622-746)
        Pick m4 = cck11_module(R(1) - I(0), R(0) + I(1), -(I(2) + R(3)), R(2) - I(3), R(5) - I(4), R(4) + I(5), I(6) + R(7), I(7) - R(6));
        m4.val |= 0x0C;
        out = m1.max > m4.max ? m1.val : m4.val;
    } else {
        Pick m3 = cck11_module(R(1) - R(0), I(1) - I(0), -(R(2) + R(3)), -(I(2) + I(3)), R(5) - R(4), I(5) - I(4), R(6) + R(7), I(6) + I(7));
        m3.val |= 0x04;
        out = m2.max > m3.max ? m2.val : m3.val;
    }
#undef R
#undef I
    cck_dqpsk_bits(out, 0, last, P[7]);
    out ^= (uint8_t)((even << 1) | even);
    even ^= 1;
    last = P[7];
    return out;
}
// one CCK-5.5 half byte (cck.hpp:71-205); hi = second half of the byte
static void cck5_half(uint8_t& out, const c16* P, c16& last, bool hi) {
    int32_t p[8][2]; for (int i = 0; i < 8; i++) { p[i][0] = P[i].re; p[i][1] = P[i].im; }
#define R(i) p[i][0]
#define I(i) p[i][1]
    auto corr = [&](int32_t a00r, int32_t a00i, int32_t a01r, int32_t a01i, int32_t a10r, int32_t a10i, int32_t a11r, int32_t a11i) -> int32_t {
        int32_t b0r = a00r + a01r, b0i = a00i + a01i, b1r = a10r + a11r, b1i = a10i + a11i;
        b0i = -b0i;
        b0r >>= 2; b0i >>= 2; b1r >>= 2; b1i >>= 2;
        return wsub(mul32(b0r, b1r), mul32(b0i, b1i));                     // L1.re
    };
    int32_t l1 = corr(I(0) + R(1), I(1) - R(0), I(2) - R(3), -(R(2) + I(3)), I(4) + R(5), I(5) - R(4), R(7) - I(6), R(6) + I(7));
    int32_t l2 = corr(R(1) - I(0), R(0) + I(1), -(I(2) + R(3)), R(2) - I(3), R(5) - I(4), R(4) + I(5), I(6) + R(7), I(7) - R(6));
#undef R
#undef I
    int32_t max1, max2; uint8_t v1, v2;
    const uint8_t b3 = hi ? 0x80 : 0x08, b2 = hi ? 0x40 : 0x04;
    if (l1 > 0) { max1 = l1; v1 = 0; } else { max1 = wneg(l1); v1 = b3; }
    if (l2 > 0) { max2 = l2; v2 = b2; } else { max2 = wneg(l2); v2 = (uint8_t)(b2 | b3); }
    const uint8_t pick = max1 > max2 ? v1 : v2;
    if (!hi) { out = pick; cck_dqpsk_bits(out, 0, last, P[7]); }
    else { out |= pick; cck_dqpsk_bits(out, 4, last, P[7]); out ^= 0x30; }
    last = P[7];
}
uint8_t cck5_decode(const c16* P, c16& last) {                             // TCCK5P5Decoder (cck.hpp:26-45): two half bytes per 16 chips
    uint8_t b = 0; cck5_half(b, P, last, false); cck5_half(b, P + 8, last, true);
    return b;
}

// ---- the Barker branches: TBB11bDespread, TDBPSKDemap, TDQPSKDemap ----
c16 barker_despread(const c16* q) {                                         // QuickBarkerDespread (barkerspread.hpp:276-304), 11 chips
    int sr = 0, si = 0;
    static const int sgn[11] = {1, -1, 1, 1, -1, 1, 1, 1, -1, -1, -1};
    for (int i = 0; i < 11; i++) {
        int16_t re, im;
        if (i == 1 || i == 4) { re = w16(w16(-q[i].re) >> 4); im = w16(w16(-q[i].im) >> 4); }                   // negate, then >> 4
        else if (sgn[i] < 0) { re = w16(-(q[i].re >> 4)); im = w16(-(q[i].im >> 4)); }                          // >> 4, then subtract
        else { re = w16(q[i].re >> 4); im = w16(q[i].im >> 4); }
        sr += re; si += im;
    }
    return c16{w16(sr), w16(si)};                                           // the hadd of int16 lanes wraps
}
uint8_t dbpsk_demap(const c16* sym, c16& last) {                            // TDBPSKDemap::DemapDBPSK (barkerspread.hpp:353-371), 8 symbols
    uint8_t r = 0; c16 ref = last;
    for (int i = 0; i < 8; i++) { r |= (uint8_t)(((uint32_t)wadd(ref.re * sym[i].re, ref.im * sym[i].im) >> 31) << i); ref = sym[i]; }
    last = sym[7];
    return r;
}
uint8_t dqpsk_demap(const c16* sym, c16& last) {                            // TDQPSKDemap::DemapDQPSK (barkerspread.hpp:441-450), 4 symbols
    uint8_t r = 0; c16 ref = last;
    for (int i = 0; i < 4; i++) { dqpsk_bits(r, 2 * i, ref, sym[i]); ref = sym[i]; }
    last = sym[3];
    return r;
}

// ---- byte path: TDesc741 -> TBB11bPlcpSwitch -> parser | frame sink ----
void Rx11b::on_byte(uint8_t b) {
    // TDesc741 (scramble.hpp:95-162): self-synchronising descrambler, 8 bits at a time
    uint8_t x = b, s = byte_reg, o = 0;
    for (int k = 0; k < 8; k++) { uint8_t o1 = (x ^ s ^ (s >> 3)) & 1; s = (uint8_t)((s >> 1) | ((x & 1) << 6)); o = (uint8_t)((o >> 1) | (o1 << 7)); x >>= 1; }
    byte_reg = b >> 1;
    if (plcp_state == 0) {                                                 // TBB11bPlcpParser (PHY_11b.hpp:504-652)
        hdr[hdr_n++] = o;
        if (hdr_n < 6) return;
        hdr_n = 0;
        uint16_t c = crc16(hdr, 4), got = (uint16_t)(hdr[4] | (hdr[5] << 8));
        if (c != got) { error_code = E_PLCP_HEADER_FAIL; return; }
        const uint8_t signal = hdr[0], service = hdr[1]; uint16_t len = (uint16_t)(hdr[2] | (hdr[3] << 8));
        switch (signal) {                                                  // dot11_plcp.h: 0x0A, 0x14, 0x37, 0x6E
        case 0x0A: data_rate_kbps = 1000; frame_length = (uint16_t)(len >> 3); rate_state = 1; break;
        case 0x14: data_rate_kbps = 2000; frame_length = (uint16_t)(len >> 2); rate_state = 2; break;
        case 0x37: data_rate_kbps = 5500; frame_length = (uint16_t)(((len * 11) >> 4) - (service >> 7) - ((service >> 3) & 1)); rate_state = 3; break;
        case 0x6E: data_rate_kbps = 11000; frame_length = (uint16_t)(((len * 11) >> 3) - (service >> 7) - ((service >> 3) & 1)); rate_state = 4; break;
        default: data_rate_kbps = 0; frame_length = 0;                     // unknown rate: rxrate_state unchanged (parser has no default case)
        }
        plcp_state = 1;
        return;
    }
    // TBB11bFrameSink (PHY_11b.hpp:657-747)
    if (error_code != E_SUCCESS) return;                                    // sink returned false: the decoder stops pumping (cck.hpp:44,247)
    if (byte_count < (uint32_t)((int)frame_length - 4)) {
        frame_buf[byte_count++ & 4095] = o;
        crc_run = (crc_run >> 8) ^ tables().crc32_lut[o ^ (crc_run & 0xFF)];
    } else if (byte_count < (uint32_t)frame_length) {
        frame_buf[byte_count++ & 4095] = o;
        if (byte_count == (uint32_t)frame_length - 1) {                      // verdict on the first three FCS bytes (:728-739)
            uint32_t fcs = frame_buf[(byte_count - 3) & 4095] | (frame_buf[(byte_count - 2) & 4095] << 8) | (frame_buf[(byte_count - 1) & 4095] << 16);
            frame_crc32 = fcs;                                               // the 4th byte the reference reads here is stale buffer content
            error_code = ((~crc_run & 0x00FFFFFFu) == fcs) ? E_FRAME_OK : E_CRC32_FAIL;
        }
    }
}

// ---- symbol path behind TBB11bRxRateSel ----
void Rx11b::on_chip(c16 s) {
    if (error_code != E_SUCCESS && error_code != E_CS_TIMEOUT) return;
    if (rate_state <= 2) {                                                  // Barker branches: TBB11bDespread (barkerspread.hpp:229-304)
        dsp_q[dsp_n++] = s;
        if (dsp_n < 11) return;
        dsp_n = 0;
        const c16 sym = barker_despread(dsp_q);
        if (rate_state == 0) {                                              // TSFDSync (sfd_sync.hpp:12-133)
            unsigned bit = (uint32_t)(last_symbol.re * sym.re + last_symbol.im * sym.im) >> 31;
            last_symbol = sym;
            byte_reg &= 0x7f;
            unsigned sbit = (bit ^ byte_reg ^ (byte_reg >> 3)) & 1;
            byte_reg = (uint8_t)((byte_reg >> 1) | (bit << 6));
            sfd_word = (uint16_t)((sfd_word >> 1) | (sbit << 15));
            sfd_cnt++;
            if (!sfd_one) { if (sfd_word == 0xFFFF) sfd_one = true; }
            else {
                if (sfd_word == 0xF3A0) rate_state = 1;
                else if (sfd_word != 0xFFFF) { if (sfd_err++ > 32) { error_code = E_SFD_FAIL; return; } }
            }
            if (sfd_cnt > 128 + 16) { error_code = E_SFD_TIMEOUT; return; }
            return;
        }
        sym_q[sym_n++] = sym;
        if (rate_state == 1 && sym_n == 8) {                                // TDBPSKDemap (barkerspread.hpp:314-390)
            const uint8_t r = dbpsk_demap(sym_q, last_symbol);
            sym_n = 0; on_byte(r);
        } else if (rate_state == 2 && sym_n == 4) {                         // TDQPSKDemap (barkerspread.hpp:398-451)
            const uint8_t r = dqpsk_demap(sym_q, last_symbol);
            sym_n = 0; on_byte(r);
        }
        return;
    }
    cck_q[cck_n++] = s;
    if (rate_state == 3 && cck_n == 16) {                                   // TCCK5P5Decoder (cck.hpp:11-69)
        uint8_t b = cck5_decode(cck_q, last_symbol);
        cck_n = 0; on_byte(b);
    } else if (rate_state == 4 && cck_n == 8) {                             // TCCK11Decoder (cck.hpp:210-260)
        uint8_t b = cck11_decode(cck_q, last_symbol, cck_even);
        cck_n = 0; on_byte(b);
    }
}

// ---- TBarkerSync (symtiming.hpp:177-308) ----
void Rx11b::barker_sync(c16 in) {
    if (bs_state == 4) { on_chip(in); return; }
    bs_search++;
    if (bs_search >= 44) { error_code = E_SYNC_TIMEOUT; return; }
    c16 ss = csra(in, 4);
    c16 o = csub(bs_partial[0], ss);
    bs_partial[0] = csub(bs_partial[1], ss); bs_partial[1] = csub(bs_partial[2], ss); bs_partial[2] = cadd(bs_partial[3], ss);
    bs_partial[3] = cadd(bs_partial[4], ss); bs_partial[4] = cadd(bs_partial[5], ss); bs_partial[5] = csub(bs_partial[6], ss);
    bs_partial[6] = cadd(bs_partial[7], ss); bs_partial[7] = cadd(bs_partial[8], ss); bs_partial[8] = csub(bs_partial[9], ss);
    bs_partial[9] = ss;
    int corr = cnorm2(o);
    if (bs_state == 0) {
        if (corr > bs_max) { bs_max = corr; bs_last_peak = 1; }
        else { bs_last_peak++; if (bs_last_peak == 11) bs_state = 1; }
    } else if (bs_state == 1) { bs_max = corr / 2; bs_last_peak = 1; bs_state = 2; }
    else if (bs_state == 2) {
        if (corr > bs_max) { bs_max = corr; bs_last_peak = 0; bs_state = 0; }
        else { bs_last_peak++; if (bs_last_peak == 11) bs_state = 3; }
    } else bs_state = 4;
}

// ---- TSymTiming (symtiming.hpp:12-169): one 28-sample block ----
void Rx11b::sym_timing(c16* blk) {
    int idx = m_index;
    while (idx < 28) {                                                     // Decimation
        c16 out;
        if (idx < 0) { out = blk[0]; m_index += 4; } else out = blk[idx];
        idx += 4;
        if (error_code == E_SUCCESS) barker_sync(out);                      // TBarkerSync returns false on timeout; later samples are dropped with the reset
    }
    if (m_index >= 4) m_index = 0;
    int sum[4] = {0, 0, 0, 0};                                              // AdjustTiming: energy of (x >> 3) per sampling phase
    for (int i = 0; i < 28; i++) { c16 v = csra(blk[i], 3); sum[i & 3] += v.re * v.re + v.im * v.im; }
    int early = m_index == 0 ? 3 : m_index - 1, late = m_index == 3 ? 0 : m_index + 1;
    if (sum[early] < sum[late]) {
        if (sum[m_index] < sum[early]) { m_index++; m_frag = 0; }
        else if (sum[m_index] < sum[late]) m_frag++;
    } else {
        if (sum[m_index] < sum[late]) { m_index--; m_frag = 0; }
        else if (sum[m_index] < sum[early]) m_frag--;
    }
    if (m_frag >= 4) { m_index++; m_frag = -3; } else if (m_frag <= -4) { m_index--; m_frag = 3; }
}

uint32_t Rx11b::push_block28(const c16* s) {                                // TMemSamples -> TDCRemove (dc.hpp:8-43) -> TBB11bRxSwitch
    mem_sample_index += 28;
    for (int v = 0; v < 7; v++) {
        c16 x[4]; for (int k = 0; k < 4; k++) x[k] = csub(s[4 * v + k], DC);
        if (cca_state == 0) energy_detect(x);
        else {
            memcpy(st_q + st_n, x, sizeof x); st_n += 4;
            if (st_n == 28) { sym_timing(st_q); st_n = 0; }
        }
        vec_count++;
    }
    return error_code;
}

int Rx11b::run(const c16* samples, size_t n, FrameResult11b* res, uint8_t* out, size_t out_stride, int max_frames) {
    init();
    int nf = 0; size_t pos = 0;
    while (pos + 28 <= n && nf < max_frames) {
        uint32_t err = push_block28(samples + pos); pos += 28;
        if (err == E_SUCCESS) continue;
        if (err != E_CS_TIMEOUT) {
            FrameResult11b& r = res[nf];
            r.status = err; r.rate_kbps = data_rate_kbps; r.length = frame_length; r.crc32 = frame_crc32;
            r.sample_index = mem_sample_index; r.detect_vec = detect_vec;
            if (out) { size_t nb = frame_length < out_stride ? frame_length : out_stride; memcpy(out + (size_t)nf * out_stride, frame_buf, nb); }
            nf++;
            if (err == E_FRAME_OK || err == E_CRC32_FAIL) {                 // skip the last FCS byte (fb11b_demod.cpp:43-61), Seek rounds up to 4
                size_t skip = data_rate_kbps == 1000 ? 352 : data_rate_kbps == 2000 ? 176 : data_rate_kbps == 5500 ? 64 : 32;
                pos += skip; mem_sample_index += (uint32_t)skip;
            }
        }
        ctx_reset(); bricks_reset();                                        // Flush(); ctx.reset(); Reset()  (fb11b_demod.cpp:63-65)
    }
    return nf;
}

} // namespace sbo
