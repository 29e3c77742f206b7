// ORACLE — TEST INFRASTRUCTURE ONLY (see ops.h).
#include "tables.h"
#include <math.h>
#include "demap_lut.inc"

namespace sbo {

static void expand_rle(const unsigned char (*rle)[2], size_t n, uint8_t* out) {
    size_t k = 0;
    for (size_t i = 0; i < n; i++) for (int c = 0; c < rle[i][1]; c++) out[k++] = rle[i][0];
}

// 802.11a-1999 17.3.5.6: k = coded-bit index, j = index after both permutations (position on air);
// the receiver reads out[k] = in[j].
static void gen_deint(uint16_t* map, int ncbps, int nbpsc) {
    int s = nbpsc / 2 > 1 ? nbpsc / 2 : 1;
    for (int k = 0; k < ncbps; k++) {
        int i = (ncbps / 16) * (k % 16) + k / 16;
        int j = s * (i / s) + (i + ncbps - (16 * i) / ncbps) % s;
        map[k] = (uint16_t)j;
    }
}

Tables::Tables() {
    const double P = 3.141593;   // the constant the reference tables were generated with (SURVEY.md §7-1)
    for (int i = 0; i < 65536; i++) {
        sin_lut[i] = (int16_t)lround(32767.0 * sin(2 * P * i / 65536));
        cos_lut[i] = (int16_t)lround(32767.0 * cos(2 * P * i / 65536));
    }
    for (int y = 0; y < 256; y++) for (int x = 0; x < 256; x++)
        atan2_lut[y * 256 + x] = (int16_t)trunc(atan2((double)(int8_t)y, (double)(int8_t)x) / P * 32768.0);
    for (int m = 1; m <= 3; m++) {
        for (int j = 0; j < 16; j++) {
            tw64[m - 1][j].re = (int16_t)trunc(32767.0 * cos(2 * M_PI * j * m / 64));
            tw64[m - 1][j].im = (int16_t)trunc(-32767.0 * sin(2 * M_PI * j * m / 64));
        }
        for (int j = 0; j < 4; j++) {
            tw16[m - 1][j].re = (int16_t)trunc(32767.0 * cos(2 * M_PI * j * m / 16));
            tw16[m - 1][j].im = (int16_t)trunc(-32767.0 * sin(2 * M_PI * j * m / 16));
        }
        for (int j = 0; j < 32; j++) { tw128[m - 1][j].re = (int16_t)trunc(32767.0 * cos(2 * M_PI * j * m / 128)); tw128[m - 1][j].im = (int16_t)trunc(-32767.0 * sin(2 * M_PI * j * m / 128)); }
        for (int j = 0; j < 8; j++) { tw32[m - 1][j].re = (int16_t)trunc(32767.0 * cos(2 * M_PI * j * m / 32)); tw32[m - 1][j].im = (int16_t)trunc(-32767.0 * sin(2 * M_PI * j * m / 32));
        }
    }
    // Viterbi branch metrics (SURVEY.md §7-1; viterbilut.h:51-185): new state n = 16*(g>>1)+lane,
    // predecessor p = (n>>1) + 32*(g&1), expected coded bits from g0=133o, g1=171o.
    for (int s = 0; s < 8; s++) for (int g = 0; g < 8; g++) for (int lane = 0; lane < 16; lane++) {
        int n = 16 * (g >> 1) + lane, p = (n >> 1) + 32 * (g & 1), b = n & 1;
        int p0 = p & 1, p1 = (p >> 1) & 1, p2 = (p >> 2) & 1, p4 = (p >> 4) & 1, p5 = (p >> 5) & 1;
        int ea = b ^ p1 ^ p2 ^ p4 ^ p5, eb = b ^ p0 ^ p1 ^ p2 ^ p5;
        vit_ma[s * 8 + g][lane] = (uint8_t)(ea ? 14 - 2 * s : 2 * s);
        vit_mb[s * 8 + g][lane] = (uint8_t)(eb ? 14 - 2 * s : 2 * s);
    }
    gen_deint(deint48, 48, 1); gen_deint(deint96, 96, 2); gen_deint(deint192, 192, 4); gen_deint(deint288, 288, 6);
    expand_rle(SB_RLE_M_BPSK_LUT, sizeof(SB_RLE_M_BPSK_LUT) / 2, demap_bpsk);
    expand_rle(SB_RLE_M_QAM16_LUT2, sizeof(SB_RLE_M_QAM16_LUT2) / 2, demap_q16_2);
    expand_rle(SB_RLE_M_QAM64_LUT2, sizeof(SB_RLE_M_QAM64_LUT2) / 2, demap_q64_2);
    expand_rle(SB_RLE_M_QAM64_LUT3, sizeof(SB_RLE_M_QAM64_LUT3) / 2, demap_q64_3);
    // x^7+x^4+1 advanced 8 steps (scramble.hpp:279-296): index = 7-bit state, entry = next output byte
    for (int i = 0; i < 128; i++) {
        uint8_t x = (uint8_t)(i << 1);
        for (int k = 0; k < 8; k++) { uint8_t o = ((x >> 1) ^ (x >> 4)) & 1; x = (uint8_t)((x >> 1) | (o << 7)); }
        scramble_lut[i] = x;
    }
    for (uint32_t i = 0; i < 256; i++) {      // IEEE 802.3 CRC-32, reflected (core/inc/CRC32.h:76)
        uint32_t c = i; for (int k = 0; k < 8; k++) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
        crc32_lut[i] = c;
    }
    tw8[0] = c16{32767, 0}; tw8[1] = c16{23169, -23169}; tw8[2] = c16{32767, 0}; tw8[3] = c16{-23169, -23169};   // trunc(32767 e^{-j pi k/4}), k = 0,1,0,3
    // STS correlation patterns: IFFT<64> of the frequency-domain STS, 16 cyclic shifts
    // (brick/inc/sequence.h:5-33, cca.hpp:266-276).  tw tables above must be ready first.
}

static void build_sts(Tables& t);
static thread_local const Tables* tl_building = nullptr;   // build_sts() runs the IFFT, which asks for the (twiddle) tables: only the building thread sees them early
const Tables& tables() {   // a function-local static: built once, and complete before any other batch thread can see it
    if (tl_building) return *tl_building;
    static const Tables* g_tables = [] { Tables* t = new Tables(); tl_building = t; build_sts(*t); tl_building = nullptr; return t; }();
    return *g_tables;
}

int16_t uatan2(int y, int x) {
    auto scope = [](int v) -> int {      // floor(log2|v|), 0 for |v|<=1 (intalglut.h:7312 bit_high_pos_lut)
        uint32_t u = v > 0 ? (uint32_t)v : (uint32_t)0 - (uint32_t)v;
        int n = 0; while (u > 1) { n++; u >>= 1; } return n;
    };
    int ys = scope(y), xs = scope(x);
    int shift = (xs > ys ? xs : ys) - 6;
    const int16_t* lut = tables().atan2_lut;
    if (shift > 0) return lut[(uint8_t)(y >> shift) * 256 + (uint8_t)(x >> shift)];
    return lut[(uint8_t)y * 256 + (uint8_t)x];
}

// ---------------------------------------------------------------------------------------------
// Radix-4 DIF fixed-point FFT/IFFT (core/inc/fft_r4dif.h:12-139, ifft_r4dif.h:12-140)
// ---------------------------------------------------------------------------------------------
template <bool INV>
static inline void r4_stage(v128* p, int q, const c16* t1, const c16* t2, const c16* t3) {
    for (int n = 0; n < q; n++) {
        v128 a = _mm_srai_epi16(p[n], 2), b = _mm_srai_epi16(p[n + q], 2);
        v128 c = _mm_srai_epi16(p[n + 2 * q], 2), d = _mm_srai_epi16(p[n + 3 * q], 2);
        v128 ac = _mm_adds_epi16(a, c), bd = _mm_adds_epi16(b, d);
        v128 a_c = _mm_subs_epi16(a, c), b_d = _mm_subs_epi16(b, d);
        p[n] = _mm_adds_epi16(ac, bd);
        v128 x2 = _mm_subs_epi16(ac, bd);
        v128 jbd = mulj_xor(b_d);
        v128 w1 = ld(t1 + 4 * n), w2 = ld(t2 + 4 * n), w3 = ld(t3 + 4 * n);
        if (!INV) {
            p[n + q] = cmul_shift_fft(x2, w2, 15);
            p[n + 2 * q] = cmul_shift_fft(_mm_subs_epi16(a_c, jbd), w1, 15);
            p[n + 3 * q] = cmul_shift_fft(_mm_adds_epi16(a_c, jbd), w3, 15);
        } else {
            p[n + q] = cmul_conj_shift(x2, w2, 15);
            p[n + 2 * q] = cmul_conj_shift(_mm_adds_epi16(a_c, jbd), w1, 15);
            p[n + 3 * q] = cmul_conj_shift(_mm_subs_epi16(a_c, jbd), w3, 15);
        }
    }
}

// 4-point DFT inside one vector, negations done as one's complement (fft_r4dif.h:62-86)
template <bool INV>
static inline v128 dft4(v128 v) {
    const v128 HI64 = _mm_set_epi32(-1, -1, 0, 0);
    const v128 TOP16 = _mm_set_epi32((int)0xFFFF0000, 0, 0, 0);
    const v128 ODD32 = _mm_set_epi32(-1, 0, -1, 0);
    v128 x = _mm_srai_epi16(v, 2);
    v128 y = _mm_shuffle_epi32(x, 0x4e);
    x = _mm_adds_epi16(_mm_xor_si128(x, HI64), y);        // [x0+x2, x1+x3, x0-x2, x1-x3] (approx. negation)
    if (!INV) { x = _mm_shufflehi_epi16(x, 0xb4); x = _mm_xor_si128(x, TOP16); }   // lane3 *= -j
    else      { x = _mm_xor_si128(x, TOP16); x = _mm_shufflehi_epi16(x, 0xb4); }   // lane3 *= +j
    v128 z = _mm_shuffle_epi32(x, 0xb1);
    return _mm_adds_epi16(_mm_xor_si128(x, ODD32), z);
}

template <bool INV>
static void xform64(v128* p, v128* out) {
    const Tables& T = tables();
    r4_stage<INV>(p, 4, T.tw64[0], T.tw64[1], T.tw64[2]);
    for (int s = 0; s < 4; s++) {
        v128* q = p + 4 * s;
        r4_stage<INV>(q, 1, T.tw16[0], T.tw16[1], T.tw16[2]);
        for (int k = 0; k < 4; k++) q[k] = dft4<INV>(q[k]);
    }
    const uint32_t* src = (const uint32_t*)p; uint32_t* dst = (uint32_t*)out;
    for (int i = 0; i < 64; i++) {
        int r = ((i & 1) << 5) | ((i & 2) << 3) | ((i & 4) << 1) | ((i & 8) >> 1) | ((i & 16) >> 3) | ((i & 32) >> 5);
        dst[i] = src[r];                                   // fft_lut_bitreversal.h:76 FFT64LUTMap
    }
}
// IFFTSSEEx<8> (ifft_r4dif.h:90-139): two vectors = eight points, input shift 3, one twiddle vector [1, W8, 1, W8^3]
static inline void ifft8(v128* p) {
    const Tables& T = tables();
    const v128 HI64 = _mm_set_epi32(-1, -1, 0, 0), TOP16 = _mm_set_epi32((int)0xFFFF0000, 0, 0, 0), ODD32 = _mm_set_epi32(-1, 0, -1, 0);
    const v128 HI_IM = _mm_set_epi32((int)0xFFFF0000, (int)0xFFFF0000, 0, 0);
    v128 a = _mm_srai_epi16(p[0], 3), b = _mm_srai_epi16(p[1], 3);
    v128 d = _mm_subs_epi16(a, b); a = _mm_adds_epi16(a, b);
    d = _mm_xor_si128(d, HI_IM); d = _mm_shufflehi_epi16(d, 0xb1);           // upper two elements times j (approximate negation)
    v128 e = _mm_shuffle_epi32(d, 0x4e);
    d = _mm_adds_epi16(_mm_xor_si128(d, HI64), e);
    v128 lo = cmul_conj_shift(d, ld(T.tw8), 15);
    v128 f = _mm_shuffle_epi32(lo, 0xb1);
    lo = _mm_adds_epi16(_mm_xor_si128(lo, ODD32), f);
    e = _mm_shuffle_epi32(a, 0x4e);
    a = _mm_adds_epi16(_mm_xor_si128(a, HI64), e);
    a = _mm_xor_si128(a, TOP16); a = _mm_shufflehi_epi16(a, 0xb4);
    f = _mm_shuffle_epi32(a, 0xb1);
    a = _mm_adds_epi16(_mm_xor_si128(a, ODD32), f);
    p[0] = a; p[1] = lo;
}
thread_local std::vector<c16>* ifft128_log = nullptr;
void ifft128(v128* p, v128* out) {
    const Tables& T = tables();
    if (ifft128_log) ifft128_log->insert(ifft128_log->end(), (const c16*)p, (const c16*)p + 128);
    r4_stage<true>(p, 8, T.tw128[0], T.tw128[1], T.tw128[2]);
    for (int s = 0; s < 4; s++) {
        v128* q = p + 8 * s;
        r4_stage<true>(q, 2, T.tw32[0], T.tw32[1], T.tw32[2]);
        for (int k = 0; k < 4; k++) ifft8(q + 2 * k);
    }
    const uint32_t* src = (const uint32_t*)p; uint32_t* dst = (uint32_t*)out;
    for (int i = 0; i < 128; i++) { int r = 0; for (int b = 0; b < 7; b++) r |= ((i >> b) & 1) << (6 - b); dst[i] = src[r]; }   // FFT128LUTMap
}
void fft64(v128* inout, v128* out) { xform64<false>(inout, out); }
void ifft64(v128* inout, v128* out) { xform64<true>(inout, out); }

static void build_sts(Tables& t) {
    alignas(16) c16 f[64]; memset(f, 0, sizeof f);
    const int16_t A = 10000;                               // sequence.h:3 ONE_MOD
    auto set = [&](int k, int16_t v) { f[k].re = v; f[k].im = v; };
    set(4, -A); set(8, -A); set(12, A); set(16, A); set(20, A); set(24, A);
    set(64 - 24, A); set(64 - 20, -A); set(64 - 16, A); set(64 - 12, -A); set(64 - 8, -A); set(64 - 4, A);
    alignas(16) c16 td[64 + 16];
    ifft64((v128*)f, (v128*)td);
    // cca.hpp:271-275 copies 16 samples starting at temp[i], i=0..15: i+15 <= 30 < 64, no wrap needed
    for (int i = 0; i < 16; i++) memcpy(t.sts_pattern[i], &td[i], 16 * sizeof(c16));
}

} // namespace sbo
