// sora_b200 — device lookup tables.
// Closed-form regeneration of the reference's LUT data (diffed against the headers in the build container by
// tests/test_tables_vs_reference.py; the formulas are the ones SURVEY.md §7-1 established):
//   usin/ucos/uatan2  kernel/core/inc/intalglut.h:4,3648,7332      (constant P = 3.141593)
//   FFT twiddles      kernel/core/inc/fft_lut_twiddle.h:61434-61583
//   de-interleaver    kernel/bb/Brick11/src/deinterleaver.hpp:9-860 (802.11a 17.3.5.6)
//   pilot polarity    kernel/bb/Brick11/src/pilot.hpp:10-28
//   LTS signs         kernel/bb/Brick11/src/channel_11a.hpp:13-18
//   STS patterns      kernel/brick/inc/sequence.h:5-33 + kernel/bb/Brick11/src/cca.hpp:266-276
//   soft demap        kernel/bb/Brick11/src/demapper.h:56-130 (data; tables/demap_lut.inc)
#pragma once
#include "fixed.cuh"
#include <math.h>
#include <string.h>
#include <vector>
#include "tables/demap_lut.inc"

namespace sb {

struct DevTables {
    const int16_t* sin_lut;      // [65536]
    const int16_t* cos_lut;      // [65536]
    const int16_t* atan2_lut;    // [256*256]
    const uint32_t* rot;         // [65536] packed (ucos(th), -usin(th)): one load per rotation instead of two
    const uint32_t* tw64;        // [3][16] packed c16
    const uint32_t* tw16;        // [3][4]
    const uint32_t* sts;         // [16][16] packed c16
    const uint16_t* deint;       // [48 | 96 | 192 | 288] concatenated: offsets 0,48,144,336
    const uint8_t* demap;        // [4][256]: bpsk, qam16_2, qam64_2, qam64_3
    const uint8_t* pilot_neg;    // [128]
    const uint8_t* lts_pos;      // [64] 1 -> +1600
    const uint8_t* scramble;     // [128]
    const uint32_t* crc32;       // [256]
};

struct DevTablesTx {             // 802.11a transmit (tx11a_kernels.cuh)
    const uint32_t* tw128;     // [3][32] packed c16
    const uint32_t* tw32;      // [3][8]
    const uint8_t*  scr_seq;   // [127] scrambler output from the all-ones state
    const uint8_t*  scr_phase; // [128] phase of state s (7 bits, bit 0 = oldest) in that sequence; 255 for the zero state
    uint32_t*       preamble;  // [640] packed c16 (before the 16 -> 8 bit pack), filled by k_tx11a_preamble
};

struct DevTablesTx11n {          // 802.11n transmit (tx11n_kernels.cuh)
    const uint32_t* pre;       // [2][1120] packed c16: per stream L-STF + L-LTF (640) then HT-STF + HT-LTF x 2 (480), cyclic shifts applied
    const uint8_t*  inv;       // [2 (BPSK, QPSK)][2 (stream)][104]: air position -> bit index inside the stream's share of the symbol
    const uint16_t* inv16;     // [2 (16-QAM, 64-QAM)][2 (stream)][312]: the same for the 16-QAM / 64-QAM interleavers
};

struct DevTables11n {            // 802.11n receive (rx11n_kernels.cuh)
    const uint32_t* sincos;     // [65536] packed (cos, sin)            dsp_math.h:214-231
    const int16_t*  atan_lut;   // [4097]                               dsp_math.h:233-247
    const uint8_t*  demap;      // [256]  BPSK == QPSK table (data)     dsp_demap.h:97-137
    const uint8_t*  crc8;       // [256]                                core/inc/CRC8.h:16-26
    const uint8_t*  pos;        // [2 qpsk][2 stream][104] position, in the stream-parsed symbol, of demap output j of stream s
    const uint8_t*  lltf_pos;   // [64] 1 where the L-LTF carrier is +1  channel_11n.hpp:7-32
    const uint8_t*  htltf_pos;  // [64] 1 where the HT-LTF carrier is +1 channel_11n.hpp:300-325
    const uint16_t* pos16;      // [2: 16-QAM, 64-QAM][2 stream][312] the same position map for the 16-QAM / 64-QAM branches (stream parser blocks of 2 / 3)
    const uint8_t*  demap16;    // [2][256] dsp_demap.h lookup_table_16qam1 / 16qam2 (data)
    const uint8_t*  demap64;    // [3][288] dsp_demap.h lookup_table_64qam1..3, entry 144 = value 0 (data)
    uint32_t mcs_limit;         // first MCS index the HT-SIG parser refuses: 11 as the reference ships it (PHY_11n.hpp:497), 15 with the QAM branches enabled
};

struct HostTables {
    std::vector<int16_t> sin_lut, cos_lut, atan2_lut;
    uint32_t tw64[3][16], tw16[3][4], sts[16][16];
    uint16_t deint[48 + 96 + 192 + 288];
    uint8_t demap[4][256], pilot_neg[128], lts_pos[64], scramble[128];
    uint32_t crc32[256];
};

static inline void rle_expand(const unsigned char (*rle)[2], size_t n, uint8_t* out) {
    size_t k = 0; for (size_t i = 0; i < n; i++) for (int c = 0; c < rle[i][1]; c++) out[k++] = rle[i][0];
}
static inline void gen_deint_map(uint16_t* map, int ncbps, int nbpsc) {
    int s = nbpsc / 2 > 1 ? nbpsc / 2 : 1;
    for (int k = 0; k < ncbps; k++) {
        int i = (ncbps / 16) * (k % 16) + k / 16;
        map[k] = (uint16_t)(s * (i / s) + (i + ncbps - (16 * i) / ncbps) % s);
    }
}

// host-side FFT/IFFT 64 built from the same device primitives (used once, for the STS patterns)
static inline void host_ifft64(cs16* x, const HostTables& T) {
    auto tw = [&](const uint32_t* t, int j) { return unpack(t[j]); };
    auto conj_tw = [](cs16 a, cs16 w) {            // vector128.h:1215-1231 conj_mul_shift(a, w, 15)
        int re = wadd(a.re * w.re, a.im * w.im);
        int im = wadd(a.im * w.re, neg16(a.re) * w.im);
        return mk(sx16(re >> 15), sx16(im >> 15));
    };
    auto stage = [&](cs16* p, int q, const uint32_t* t1, const uint32_t* t2, const uint32_t* t3) {   // ifft_r4dif.h:12-47
        for (int e = 0; e < q; e++) {
            cs16 a = sra(p[e], 2), b = sra(p[e + q], 2), c = sra(p[e + 2 * q], 2), d = sra(p[e + 3 * q], 2);
            cs16 ac = adds(a, c), bd = adds(b, d), a_c = subs(a, c), b_d = subs(b, d), jbd = mulj(b_d);
            p[e] = adds(ac, bd);
            p[e + q] = conj_tw(subs(ac, bd), tw(t2, e));
            p[e + 2 * q] = conj_tw(adds(a_c, jbd), tw(t1, e));
            p[e + 3 * q] = conj_tw(subs(a_c, jbd), tw(t3, e));
        }
    };
    stage(x, 16, T.tw64[0], T.tw64[1], T.tw64[2]);
    for (int s = 0; s < 4; s++) {
        cs16* q = x + 16 * s;
        stage(q, 4, T.tw16[0], T.tw16[1], T.tw16[2]);
        for (int k = 0; k < 4; k++) {               // ifft_r4dif.h:62-85 IFFTSSEEx<4>
            cs16* v = q + 4 * k;
            cs16 x0 = sra(v[0], 2), x1 = sra(v[1], 2), x2 = sra(v[2], 2), x3 = sra(v[3], 2);
            cs16 s0 = adds(x0, x2), s1 = adds(x1, x3), s2 = adds(cnot(x2), x0), s3 = adds(cnot(x3), x1);
            cs16 t3 = mk(~s3.im, s3.re);            // lane 3 times +j
            v[0] = adds(s0, s1); v[1] = adds(cnot(s1), s0); v[2] = adds(s2, t3); v[3] = adds(cnot(t3), s2);
        }
    }
    cs16 y[64];
    for (int i = 0; i < 64; i++) {
        int r = ((i & 1) << 5) | ((i & 2) << 3) | ((i & 4) << 1) | ((i & 8) >> 1) | ((i & 16) >> 3) | ((i & 32) >> 5);
        y[i] = x[r];
    }
    memcpy(x, y, sizeof y);
}

static inline void build_host_tables(HostTables& T) {
    const double P = 3.141593;
    T.sin_lut.resize(65536); T.cos_lut.resize(65536); T.atan2_lut.resize(65536);
    for (int i = 0; i < 65536; i++) {
        T.sin_lut[i] = (int16_t)lround(32767.0 * sin(2 * P * i / 65536));
        T.cos_lut[i] = (int16_t)lround(32767.0 * cos(2 * P * i / 65536));
    }
    for (int y = 0; y < 256; y++) for (int x = 0; x < 256; x++)
        T.atan2_lut[y * 256 + x] = (int16_t)trunc(atan2((double)(int8_t)y, (double)(int8_t)x) / P * 32768.0);
    for (int m = 1; m <= 3; m++) {
        for (int j = 0; j < 16; j++)
            T.tw64[m - 1][j] = pack(mk((int)trunc(32767.0 * cos(2 * M_PI * j * m / 64)), (int)trunc(-32767.0 * sin(2 * M_PI * j * m / 64))));
        for (int j = 0; j < 4; j++)
            T.tw16[m - 1][j] = pack(mk((int)trunc(32767.0 * cos(2 * M_PI * j * m / 16)), (int)trunc(-32767.0 * sin(2 * M_PI * j * m / 16))));
    }
    gen_deint_map(T.deint, 48, 1); gen_deint_map(T.deint + 48, 96, 2); gen_deint_map(T.deint + 144, 192, 4); gen_deint_map(T.deint + 336, 288, 6);
    rle_expand(SB_RLE_M_BPSK_LUT, sizeof(SB_RLE_M_BPSK_LUT) / 2, T.demap[0]);
    rle_expand(SB_RLE_M_QAM16_LUT2, sizeof(SB_RLE_M_QAM16_LUT2) / 2, T.demap[1]);
    rle_expand(SB_RLE_M_QAM64_LUT2, sizeof(SB_RLE_M_QAM64_LUT2) / 2, T.demap[2]);
    rle_expand(SB_RLE_M_QAM64_LUT3, sizeof(SB_RLE_M_QAM64_LUT3) / 2, T.demap[3]);
    {   // pilot polarity: scrambler x^7+x^4+1 from the all-ones state gives p_0..p_126; table[i] = (p_{i+1} == -1)
        uint8_t seq[127]; unsigned st = 0x7F;
        for (int i = 0; i < 127; i++) { unsigned b = ((st >> 6) ^ (st >> 3)) & 1; st = ((st << 1) | b) & 0x7F; seq[i] = (uint8_t)b; }
        for (int i = 0; i < 127; i++) T.pilot_neg[i] = seq[(i + 1) % 127];
        T.pilot_neg[127] = 0;
    }
    {
        static const int8_t L[53] = {1,1,-1,-1,1,1,-1,1,-1,1,1,1,1,1,1,-1,-1,1,1,-1,1,-1,1,1,1,1,0,
                                     1,-1,-1,1,1,-1,1,-1,1,-1,-1,-1,-1,-1,1,1,-1,-1,1,-1,1,-1,1,1,1,1};
        for (int i = 0; i < 64; i++) { int k = i < 32 ? i : i - 64; T.lts_pos[i] = (k >= -26 && k <= 26 && L[k + 26] > 0) ? 1 : 0; }
    }
    for (int i = 0; i < 128; i++) {
        uint8_t x = (uint8_t)(i << 1);
        for (int k = 0; k < 8; k++) { uint8_t o = ((x >> 1) ^ (x >> 4)) & 1; x = (uint8_t)((x >> 1) | (o << 7)); }
        T.scramble[i] = x;
    }
    for (uint32_t i = 0; i < 256; i++) { uint32_t c = i; for (int k = 0; k < 8; k++) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1; T.crc32[i] = c; }
    {   // STS cross-correlation patterns
        cs16 f[64]; for (int i = 0; i < 64; i++) f[i] = mk(0, 0);
        const int A = 10000;
        auto set = [&](int k, int v) { f[k] = mk(v, v); };
        set(4, -A); set(8, -A); set(12, A); set(16, A); set(20, A); set(24, A);
        set(64 - 24, A); set(64 - 20, -A); set(64 - 16, A); set(64 - 12, -A); set(64 - 8, -A); set(64 - 4, A);
        host_ifft64(f, T);
        for (int i = 0; i < 16; i++) for (int j = 0; j < 16; j++) T.sts[i][j] = pack(f[i + j]);
    }
}

} // namespace sb
