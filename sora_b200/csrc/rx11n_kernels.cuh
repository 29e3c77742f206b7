// sora_b200 — 802.11n 2x2 (HT mixed format, 20 MHz, 2 spatial streams, MCS 8..10) receive kernels (sm_90a).
//
//   k_sync11n    one thread per slot (a slot = the same sample range of both antenna captures): 2:1 decimation and the
//                joint two-antenna carrier sense — 32-lag autocorrelation^2 against energy^2 in int64, energy step against
//                the value 64 samples earlier, plateau length 97..159.  The reference's history rings are running sums of
//                a function of the input, so the kernel re-reads x[n-32], x[n-64], x[n-96] (L1 hits) instead of keeping
//                1.5 KB of per-thread state.
//                Reference: samples.hpp:27-49, cca_11n.hpp:26-163, autocorr.hpp:44-146, fb11n_demod.cpp:29-81.
//   k_front11n   one warp per slot: joint CFO from the L-LTF (64-lag), NCO, per-antenna FFT64 (the two half-warps run the
//                two antennas' transforms side by side), legacy channel estimate with the reference's lane-wise rounding
//                term, L-SIG + HT-SIG (MRC, BPSK/QBPSK demap, two in-warp K=7 Viterbi runs, parity/CRC-8 parse), HT-LTF
//                2x2 channel with the single-precision inverse in the reference's operation order (no FMA), then per data
//                symbol: H^-1 y, pilot phase into the NCO, soft demap, HT de-interleave and stream de-parse straight into
//                the Viterbi input order.
//                Reference: freqoffset_11n.hpp:42-279, dsp_math.h:90-247, fft.hpp:110-135, channel_11n.hpp:34-521,
//                sora_matrix.h:135-150,296-304, PHY_11n.hpp:283-514, demapper11n.hpp:8-171, dsp_demap.h:38-137,
//                deinterleaver_11n.hpp:6-620, stdbrick.hpp:639-720, pilot_11n.hpp:84-141, viterbicore.h:36-261.
//   The K=7 Viterbi / descrambler / CRC-32 stage is the 802.11a one (k_viterbi_re or k_viterbi_lane, then k_sink11a) with the 11n window 192/36
//   (fb11ndemod_config.hpp:189); the brick's 312-value bursts and zero padding at Flush never reach a decision that is
//   delivered, because the final traceback fires inside the last real symbol.
#pragma once
#include "rx11a_kernels.cuh"

namespace sb {

struct DevTables11n {
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
// FrameInfo::rate_kbps of an event whose HT-SIG was never parsed.  CF_HTRxVector has no Reset() (ieee80211facade.hpp:269-272), so the
// reference then still holds the previous event's ht_frame_mcs: the stream driver substitutes it, a batch slot (a fresh context) reports 0.
constexpr uint32_t MCS11N_UNPARSED = 0xFFFFFFFFu;
struct HostTables11n {
    uint32_t sincos[65536]; int16_t atan_lut[4097]; uint8_t demap[256], crc8[256], pos[2][2][104], lltf_pos[64], htltf_pos[64];
    uint16_t pos16[2][2][312]; uint8_t demap16[2][256], demap64[3][288];
};
static inline void build_host_tables11n(HostTables11n& H) {
    for (unsigned i = 0; i < 65536; i++) {
        double r = (double)i * 2.0 * M_PI / 65535.0;
        H.sincos[i] = pack(mk((int)(short)(cos(r) * 32767.5), (int)(short)(sin(r) * 32767.5)));
    }
    for (int i = 0; i <= 4096; i++) H.atan_lut[i] = (int16_t)(atan((double)i / 4096.0) / (M_PI / 4.0) * 8192);
    static const unsigned char rle[8][2] = {{4, 11}, {5, 10}, {6, 10}, {7, 97}, {0, 97}, {1, 10}, {2, 10}, {3, 11}};
    rle_expand(rle, 8, H.demap);
    for (int b = 0; b < 256; b++) { uint8_t c = (uint8_t)b; for (int k = 0; k < 8; k++) c = (c & 1) ? (uint8_t)((c >> 1) ^ 0xE0) : (uint8_t)(c >> 1); H.crc8[b] = c; }
    for (int q = 0; q < 2; q++) for (int ss = 0; ss < 2; ss++) {        // IEEE 802.11n-2009 20.3.11.7.3; N_COL 13, N_ROW 4 N_BPSC, N_ROT 11, s = 1
        const int nbpsc = q + 1, n = 52 * nbpsc;
        for (int k = 0; k < n; k++) {
            const int i = 4 * nbpsc * (k % 13) + k / 13;
            const int r = ((i - ((ss * 2) % 3 + 3 * (ss / 3)) * 11 * nbpsc) % n + n) % n;        // out[k] = in[r]
            H.pos[q][ss][r] = (uint8_t)(2 * k + ss);                                             // TStreamJoin + TStreamConcat<2,1>
        }
    }
    for (int q = 0; q < 2; q++) for (int ss = 0; ss < 2; ss++) {        // 16-QAM (s = 2) and 64-QAM (s = 3): deinterleaver_11n.hpp T11nDeinterleaveQAM16/64_S0/S1
        const int nbpsc = q ? 6 : 4, n = 52 * nbpsc, sb = nbpsc / 2;
        for (int k = 0; k < n; k++) {
            const int i = 4 * nbpsc * (k % 13) + k / 13;
            const int j = sb * (i / sb) + (i + n - (13 * i) / n) % sb;
            const int r = ((j - ((ss * 2) % 3 + 3 * (ss / 3)) * 11 * nbpsc) % n + n) % n;        // out[k] = in[r]
            H.pos16[q][ss][r] = (uint16_t)((2 * (k / sb) + ss) * sb + k % sb);                   // TStreamJoin + TStreamConcat<2, 2 | 3> (fb11ndemod_config.hpp:196-213)
        }
    }
    {   static const unsigned char r161[8][2] = {{4, 5}, {5, 4}, {6, 7}, {7, 112}, {0, 113}, {1, 7}, {2, 4}, {3, 4}};
        static const unsigned char r162[15][2] = {{7, 56}, {6, 3}, {5, 3}, {4, 2}, {3, 2}, {2, 2}, {1, 3}, {0, 115}, {1, 3}, {2, 2}, {3, 2}, {4, 2}, {5, 3}, {6, 3}, {7, 55}};
        static const unsigned char r641[8][2] = {{0, 138}, {1, 3}, {2, 2}, {3, 1}, {4, 2}, {5, 2}, {6, 3}, {7, 137}};
        static const unsigned char r642[15][2] = {{0, 68}, {1, 3}, {2, 2}, {3, 2}, {4, 1}, {5, 2}, {6, 3}, {7, 127}, {6, 3}, {5, 2}, {4, 1}, {3, 2}, {2, 2}, {1, 3}, {0, 67}};
        static const unsigned char r643[29][2] = {{0, 34}, {1, 2}, {2, 2}, {3, 2}, {4, 2}, {5, 1}, {6, 3}, {7, 57}, {6, 3}, {5, 2}, {4, 2}, {3, 1}, {2, 2}, {1, 3}, {0, 57},
                                                  {1, 3}, {2, 2}, {3, 1}, {4, 2}, {5, 2}, {6, 3}, {7, 57}, {6, 3}, {5, 1}, {4, 2}, {3, 2}, {2, 2}, {1, 2}, {0, 33}};
        rle_expand(r161, 8, H.demap16[0]); rle_expand(r162, 15, H.demap16[1]);
        rle_expand(r641, 8, H.demap64[0]); rle_expand(r642, 15, H.demap64[1]); rle_expand(r643, 29, H.demap64[2]); }
    static const int8_t L[53] = {1,1,-1,-1,1,1,-1,1,-1,1,1,1,1,1,1,-1,-1,1,1,-1,1,-1,1,1,1,1,0,
                                 1,-1,-1,1,1,-1,1,-1,1,-1,-1,-1,-1,-1,1,1,-1,-1,1,-1,1,-1,1,1,1,1};
    for (int i = 0; i < 64; i++) {
        const int k = i < 32 ? i : i - 64; int l = (k >= -26 && k <= 26) ? L[k + 26] : 0;
        H.lltf_pos[i] = l == 1;
        if (k == 27 || k == 28) l = -1; if (k == -28 || k == -27) l = 1;
        H.htltf_pos[i] = l == 1;
    }
}

// dsp_math::atan(x, y) (dsp_math.h:157-212; the short overload :90-164 agrees wherever it does not overflow).  abs, imax and the sums are
// 32-bit int C there (dsp_math.h:64-88), which wraps: abs(INT_MIN) = INT_MIN, |x| + |y| wraps past 2^31.
// SMALL: both arguments are int16 values (the pilot carriers), so (tmin << 16) + tmax / 2 fits 32 unsigned bits and the
// quotient is the same as the reference's 64-bit one at a fifth of the instructions.
template <bool SMALL = false>
__device__ __forceinline__ int d_atan11n(const DevTables11n& N, int x, int y) {
    const int sign = (x ^ y) >> 31;
    const int ax = wsub(x ^ (x >> 31), x >> 31), ay = wsub(y ^ (y >> 31), y >> 31);
    const int tsign = wsub(ax, ay) >> 31;
    const int tsum = wadd(ax, ay); int d = wsub(ax, ay); d = wsub(d ^ (d >> 31), d >> 31);
    const int tmax = wadd(tsum, d) >> 1, tmin = wsub(tsum, tmax);
    int idx;
    if (SMALL) { const unsigned den = tmax ? (unsigned)tmax : 1u; idx = (int)((((unsigned)tmin << 16) + (den >> 1)) / den); }
    else { long long num = (long long)tmin * 65536, den = tmax; if (den == 0) den = 1; idx = (int)((num + (den >> 1)) / den); }
    idx >>= 4;
    if (idx < 0 || idx >= 4097) return 0;
    int srad = __ldg(N.atan_lut + idx);
    srad = sx16((16384 & tsign) + ((srad ^ tsign) - tsign));
    return sx16((srad ^ sign) - sign);
}
__device__ __forceinline__ cs16 shr_sat(int re, int im, int n) { return mk(sat16(re >> n), sat16(im >> n)); }      // psrad + packssdw

// ------------------------------------------------------------------------------------------------
// carrier sense (TCCA11n over MimoAutoCorr)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_sync11n(const uint32_t* __restrict__ iq0, const uint32_t* __restrict__ iq1, const uint64_t* __restrict__ off,
                                                  const uint32_t* __restrict__ len, uint32_t nframes, FrameInfo* __restrict__ info) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nframes) return;
    const uint32_t* x[2] = {iq0 + off[f], iq1 + off[f]};
    const bool al16 = ((((uintptr_t)x[0]) | ((uintptr_t)x[1])) & 15u) == 0;   // a vector = 8 words = two aligned 128-bit loads then
    const uint32_t nvec = (len[f] / 28u) * 28u / 8u;
    int Rre[2] = {0, 0}, Rim[2] = {0, 0}, es[2] = {0, 0}, es64[2] = {0, 0};
    unsigned sense = 0; bool peak_found = false; int peak_count = 0;
    bool timeout = false; uint32_t cur_blk = 0, detect = 0xFFFFFFFFu;
    for (uint32_t v = 0; v < nvec && detect == 0xFFFFFFFFu; v++) {
        const uint32_t blk = (8u * v + 7u) / 28u;
        if (blk != cur_blk) {                          // RxThread polls error_code once per 28-sample block (fb11n_demod.cpp:35-58)
            if (timeout) { sense = 0; peak_found = false; peak_count = 0; timeout = false; }
            cur_blk = blk;
        }
        // the four samples of this vector and of the vectors 32, 64 and 96 samples back, both antennas: sixteen 128-bit loads issued together
        uint32_t w[2][4][4];
#pragma unroll
        for (int a = 0; a < 2; a++)
#pragma unroll
            for (int tp = 0; tp < 4; tp++) {
                if (4u * v >= 32u * tp) {
                    const uint32_t* p = x[a] + 2u * (4u * v - 32u * tp);
                    if (al16) { const uint4 lo = __ldg((const uint4*)p), hi = __ldg((const uint4*)p + 1); w[a][tp][0] = lo.x; w[a][tp][1] = lo.z; w[a][tp][2] = hi.x; w[a][tp][3] = hi.z; }
                    else { w[a][tp][0] = __ldg(p); w[a][tp][1] = __ldg(p + 2); w[a][tp][2] = __ldg(p + 4); w[a][tp][3] = __ldg(p + 6); }
                } else w[a][tp][0] = w[a][tp][1] = w[a][tp][2] = w[a][tp][3] = 0;
            }
#pragma unroll
        for (uint32_t k = 0; k < 4; k++) {
            if (detect != 0xFFFFFFFFu) break;
            const uint32_t n = 4u * v + k;
#pragma unroll
            for (int a = 0; a < 2; a++) {
                const cs16 c0 = unpack(w[a][0][k]), c1 = unpack(w[a][1][k]), c2 = unpack(w[a][2][k]), c3 = unpack(w[a][3][k]);
                int pr, pi, qr, qi; cmul_conj32(pr, pi, c0, c1); cmul_conj32(qr, qi, c1, c2);      // autocorr.hpp:110-131 (vShift = 5)
                Rre[a] = wadd(Rre[a], wadd(pr >> 5, -(qr >> 5))); Rim[a] = wadd(Rim[a], wadd(pi >> 5, -(qi >> 5)));
                const int e0 = wadd(c0.re * c0.re, c0.im * c0.im) >> 5, e1 = wadd(c1.re * c1.re, c1.im * c1.im) >> 5;
                const int e2 = wadd(c2.re * c2.re, c2.im * c2.im) >> 5, e3 = wadd(c3.re * c3.re, c3.im * c3.im) >> 5;
                es[a] = wadd(es[a], wadd(e0, -e1)); es64[a] = wadd(es64[a], wadd(e2, -e3));        // autocorr.hpp:133-146; es64 = es as it was 64 samples ago
            }
            const long long cr = wadd(Rre[0] >> 1, Rre[1] >> 1), ci = wadd(Rim[0] >> 1, Rim[1] >> 1);
            const long long acorr = (long long)((unsigned long long)(cr * cr) + (unsigned long long)(ci * ci));    // SquaredNorm(vci): paddq wraps (vector128.h:922-933)
            const long long e = wadd(es[0] >> 1, es[1] >> 1), energy = e * e;
            const long long h = wadd(es64[0] >> 1, es64[1] >> 1), hise = h * h;
            // eb = energy / (his_moving_energy + 1) > 5  <=>  energy / 6 >= his + 1; the first 64 entries hold LLONG_MAX (eb = 0)
            const bool step = n >= 64 && energy / 6 >= hise + 1;
            if (!peak_found) {
                sense++;
                if (step && acorr > (energy >> 1)) { sense = 0; peak_count++; peak_found = true; } else peak_count = 0;
            } else if (acorr < (energy >> 3)) {
                if (peak_count > 96 && peak_count < 160) { detect = v + 1; continue; }
                peak_found = false; peak_count = 0;
            } else { peak_count++; if (peak_count > 160) { peak_found = false; peak_count = 0; } }
        }
        if (sense >= 84 && detect == 0xFFFFFFFFu) timeout = true;                                   // cca_11n.hpp:120-124
    }
    FrameInfo fi;
    fi.status = detect == 0xFFFFFFFFu ? (uint32_t)E_NO_FRAME : (uint32_t)E_SUCCESS;
    fi.detect_vec = detect; fi.rate_kbps = 0; fi.length = 0; fi.nsym_total = 0; fi.code_rate = CR_12; fi.ncbps = 104;
    fi.soft_bytes = 0; fi.cfo_est = 0; fi.peak_index = 0; fi.dc_re = 0; fi.dc_im = 0;
    info[f] = fi;
}

// Continuous-capture carrier sense (SURVEY.md §8(f) rank 1 for 802.11n).  TCCA11n and MimoAutoCorr are never reset between frames
// (cca_11n.hpp:146-163, autocorr.hpp:9-42) and do not see the samples the demodulator consumed, so across a frame their history is
// the stretch of samples in front of the previous detection — and the energy ring lags the sample history by the lanes dropped in the
// detection vector.  Rather than re-derive that from the input, this variant keeps the bricks' own state per capture in device memory
// (1.6 KB) and runs the reference's recurrences on it; one thread per capture, resumed pass after pass.
struct Cca11nState {
    uint32_t his_sample[2][32];                        // autocorr.hpp:14-18: 8 vectors of 4 samples per antenna
    int his_corr_re[2][32], his_corr_im[2][32], his_energy[2][32];
    int corr_re[2], corr_im[2], energy_sum[2];
    uint32_t his_idx;                                  // vector slot 0..7 the next input replaces
    uint32_t his_index, ring_written;                  // cca_11n.hpp:150-156: 64 moving energies; entries are valid once written (saturates at 64)
    long long ring[64];
};
__global__ void __launch_bounds__(64) k_sync11n_stream(const uint32_t* __restrict__ iq0, const uint32_t* __restrict__ iq1, const uint64_t* __restrict__ off,
                                                       const uint32_t* __restrict__ len, uint32_t nframes, const uint32_t* __restrict__ state_idx,
                                                       Cca11nState* __restrict__ states, FrameInfo* __restrict__ info) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nframes) return;
    const uint32_t* x[2] = {iq0 + off[f], iq1 + off[f]};
    Cca11nState& S = states[state_idx[f]];
    const uint32_t nvec = (len[f] / 28u) * 28u / 8u;
    int Rre[2] = {S.corr_re[0], S.corr_re[1]}, Rim[2] = {S.corr_im[0], S.corr_im[1]}, es[2] = {S.energy_sum[0], S.energy_sum[1]};
    uint32_t hidx = S.his_idx, rindex = S.his_index, written = S.ring_written;
    unsigned sense = 0; bool peak_found = false; int peak_count = 0;                   // BB11nDemodContext::ResetCarrierSense ran at the last event
    bool timeout = false; uint32_t cur_blk = 0, detect = 0xFFFFFFFFu;
    for (uint32_t v = 0; v < nvec && detect == 0xFFFFFFFFu; v++) {
        const uint32_t blk = (8u * v + 7u) / 28u;
        if (blk != cur_blk) {                          // the driver polls error_code once per 28-sample block (fb11n_demod.cpp:35-58)
            if (timeout) { sense = 0; peak_found = false; peak_count = 0; timeout = false; }
            cur_blk = blk;
        }
        int R_re[2][4], R_im[2][4], ve[2][4];
#pragma unroll
        for (int a = 0; a < 2; a++) {
#pragma unroll
            for (int k = 0; k < 4; k++) {                                               // autocorr.hpp:110-146
                const uint32_t w = __ldg(x[a] + 2u * (4u * v + k)); const cs16 c0 = unpack(w), c1 = unpack(S.his_sample[a][4u * hidx + k]);
                int pr, pi; cmul_conj32(pr, pi, c0, c1); pr >>= 5; pi >>= 5;
                Rre[a] = wadd(Rre[a], wadd(pr, -S.his_corr_re[a][4u * hidx + k])); Rim[a] = wadd(Rim[a], wadd(pi, -S.his_corr_im[a][4u * hidx + k]));
                S.his_corr_re[a][4u * hidx + k] = pr; S.his_corr_im[a][4u * hidx + k] = pi; R_re[a][k] = Rre[a]; R_im[a][k] = Rim[a];
                const int e = wadd(c0.re * c0.re, c0.im * c0.im) >> 5;
                es[a] = wadd(es[a], wadd(e, -S.his_energy[a][4u * hidx + k])); S.his_energy[a][4u * hidx + k] = e; ve[a][k] = es[a];
                S.his_sample[a][4u * hidx + k] = w;
            }
        }
        hidx = (hidx + 1u) & 7u;
        for (int k = 0; k < 4; k++) {                                                   // cca_11n.hpp:62-118
            const long long cr = wadd(R_re[0][k] >> 1, R_re[1][k] >> 1), ci = wadd(R_im[0][k] >> 1, R_im[1][k] >> 1);
            const long long acorr = (long long)((unsigned long long)(cr * cr) + (unsigned long long)(ci * ci));    // SquaredNorm(vci): paddq wraps
            const long long e = wadd(ve[0][k] >> 1, ve[1][k] >> 1), energy = e * e;
            const bool step = written >= 64u && energy / 6 >= S.ring[rindex] + 1;       // eb = energy / (his + 1) > 5; the ring starts at LLONG_MAX (eb = 0)
            if (!peak_found) {
                sense++;
                if (step && acorr > (energy >> 1)) { sense = 0; peak_count++; peak_found = true; } else peak_count = 0;
            } else if (acorr < (energy >> 3)) {
                if (peak_count > 96 && peak_count < 160) { detect = v + 1; break; }     // the rest of the vector never reaches the ring (ipin.clear())
                peak_found = false; peak_count = 0;
            } else { peak_count++; if (peak_count > 160) { peak_found = false; peak_count = 0; } }
            S.ring[rindex] = energy; rindex = (rindex + 1u) & 63u; if (written < 64u) written++;
        }
        if (sense >= 84 && detect == 0xFFFFFFFFu) timeout = true;                       // cca_11n.hpp:120-124
    }
    S.corr_re[0] = Rre[0]; S.corr_re[1] = Rre[1]; S.corr_im[0] = Rim[0]; S.corr_im[1] = Rim[1]; S.energy_sum[0] = es[0]; S.energy_sum[1] = es[1];
    S.his_idx = hidx; S.his_index = rindex; S.ring_written = written;
    FrameInfo fi;
    fi.status = detect == 0xFFFFFFFFu ? (uint32_t)E_NO_FRAME : (uint32_t)E_SUCCESS;
    fi.detect_vec = detect; fi.rate_kbps = 0; fi.length = 0; fi.nsym_total = 0; fi.code_rate = CR_12; fi.ncbps = 104;
    fi.soft_bytes = 0; fi.cfo_est = 0; fi.peak_index = 0; fi.dc_re = 0; fi.dc_im = 0;
    info[f] = fi;
}

// ------------------------------------------------------------------------------------------------
// L-SIG / HT-SIG Viterbi: N trellis steps from the zero state, full traceback (Viterbi_sig11(..., output_bit))
// ------------------------------------------------------------------------------------------------
template <int N>
__device__ __forceinline__ unsigned long long warp_viterbi_sig_n(const uint8_t* soft, int lane, uint32_t* dec /* [2N] warp-private shared */) {
    const unsigned FULL = 0xFFFFFFFFu;
    const int cA = ((lane >> 1) ^ (lane >> 2) ^ (lane >> 4)) & 1, cB = (lane ^ (lane >> 1) ^ (lane >> 2)) & 1;
    int m0 = lane == 0 ? 0x00 : 0x30, m1 = 0x30;
    for (int t = 0; t < N; t++) {
        const int tA = 2 * soft[2 * t], tB = 2 * soft[2 * t + 1];
        const int alpha = (cA ? 14 - tA : tA) + (cB ? 14 - tB : tB), beta = 28 - alpha;
        const int n0 = min((m0 + alpha) & 0xFE, ((m1 + beta) & 0xFF) | 1);
        const int n1 = min((m0 + beta) & 0xFE, ((m1 + alpha) & 0xFF) | 1);
        const uint32_t e = __ballot_sync(FULL, n0 & 1), o = __ballot_sync(FULL, n1 & 1);
        if (lane == 0) { dec[2 * t] = e; dec[2 * t + 1] = o; }
        const int w = n0 | (n1 << 8);
        const int wa = __shfl_sync(FULL, w, lane >> 1), wb = __shfl_sync(FULL, w, 16 + (lane >> 1));
        const int sh = 8 * (lane & 1);
        m0 = (wa >> sh) & 0xFF; m1 = (wb >> sh) & 0xFF;
        if (((t + 1) & 7) == 0) { const int mn = __reduce_min_sync(FULL, min(m0, m1)) & 0xFE; m0 = (m0 - mn) & 0xFF; m1 = (m1 - mn) & 0xFF; }
    }
    __syncwarp();
    unsigned key = min(((unsigned)m0 << 8) | ((unsigned)lane << 2), ((unsigned)m1 << 8) | ((unsigned)(lane + 32) << 2));
    key = __reduce_min_sync(FULL, key);
    int pos = (int)(key >> 2) & 0x7F;
    unsigned long long word = 0;
    for (int i = 0; i < N; i++) {
        word |= (unsigned long long)((pos >> 6) & 1) << (N - 1 - i);
        pos = (pos >> 1) & 0x3F;
        const int col = N - 1 - i; int bit = 0;
        if (col >= 1) { const uint32_t wsel = dec[2 * (col - 1) + (pos & 1)]; bit = (wsel >> (pos >> 1)) & 1; }
        pos |= bit << 6;
    }
    __syncwarp();
    return word >> 6;
}

struct Taps11n {              // optional stage taps (device pointers, nullptr = off)
    uint32_t* siso;           // [slot][2][64]
    uint32_t* hinv;           // [slot][4][64]
    uint32_t* eq;             // [slot][2][max_sym][64]   data symbols
    int16_t*  theta;          // [slot][max_sym]
    uint8_t*  sig;            // [slot][16]
    uint32_t  max_sym;
};

__device__ __forceinline__ int ht_data_index(int bin) {     // demapper11n.hpp:110-131: -28..-1 then 1..28 without the pilots
    if (bin >= 36) { if (bin == 43 || bin == 57) return -1; return bin - 36 - (bin > 43) - (bin > 57); }
    if (bin >= 1 && bin <= 28) { if (bin == 7 || bin == 21) return -1; return 26 + bin - 1 - (bin > 7) - (bin > 21); }
    return -1;
}
__device__ __forceinline__ int cvt_x86(float x) {           // cvtps2dq: round to nearest even, "integer indefinite" when out of range / NaN
    if (!(x >= -2147483648.0f && x < 2147483648.0f)) return (int)0x80000000;
    return __float2int_rn(x);
}
struct cfl { float re, im; };
__device__ __forceinline__ cfl cmulf(cfl a, cfl b) {        // vector128.h:1106-1116 mul(vcf, vcf): separate multiplies, then addsub
    cfl r; r.re = __fsub_rn(__fmul_rn(a.re, b.re), __fmul_rn(a.im, b.im)); r.im = __fadd_rn(__fmul_rn(a.im, b.re), __fmul_rn(a.re, b.im)); return r;
}

#define SB_FRONT11N_WARPS 4
// T11nDemapQAM16 / QAM64 (demapper11n.hpp:199-309) for the two carriers of a lane, both streams: limit to [-128, 127], per-bit tables, then the
// position map (HT de-interleaver + stream joiner).  Kept out of line so that the BPSK / QPSK symbol loop keeps its register allocation.
__device__ __noinline__ void demap_qam11n(uint8_t* sb, const uint16_t* __restrict__ pos16, const uint8_t* __restrict__ demap16, const uint8_t* __restrict__ demap64,
                                          int nbpsc, int dh0, int dh1, uint32_t x00, uint32_t x01, uint32_t x10, uint32_t x11) {
#pragma unroll
    for (int w = 0; w < 2; w++) {
        const int d = w ? dh1 : dh0;
        if (d < 0) continue;
#pragma unroll
        for (int s = 0; s < 2; s++) {
            const cs16 x = unpack(s ? (w ? x11 : x10) : (w ? x01 : x00));
            const int re = min(max(x.re, -128), 127), im = min(max(x.im, -128), 127);
            const uint16_t* pp = pos16 + (((nbpsc == 6 ? 2 : 0) + s) * 312 + d * nbpsc);
            if (nbpsc == 4) {
                sb[__ldg(pp + 0)] = __ldg(demap16 + (re & 0xFF)); sb[__ldg(pp + 1)] = __ldg(demap16 + 256 + (re & 0xFF));
                sb[__ldg(pp + 2)] = __ldg(demap16 + (im & 0xFF)); sb[__ldg(pp + 3)] = __ldg(demap16 + 256 + (im & 0xFF));
            } else {
#pragma unroll
                for (int t = 0; t < 3; t++) { sb[__ldg(pp + t)] = __ldg(demap64 + 288 * t + 144 + re); sb[__ldg(pp + 3 + t)] = __ldg(demap64 + 288 * t + 144 + im); }
            }
        }
    }
}

#ifndef SB_FRONT11N_MINB
#define SB_FRONT11N_MINB 6         // resident CTAs per SM the register allocation aims at (tools/front_sweep.sh: 4 and 5 are no faster)
#endif
__global__ void __launch_bounds__(32 * SB_FRONT11N_WARPS, SB_FRONT11N_MINB) k_front11n(const uint32_t* __restrict__ iq0, const uint32_t* __restrict__ iq1,
        const uint64_t* __restrict__ off, const uint32_t* __restrict__ len, uint32_t nframes, DevTables T, DevTables11n N, const uint16_t* __restrict__ inv_deint48,
        FrameInfo* __restrict__ info, uint8_t* __restrict__ soft_out, uint64_t soft_stride, Taps11n taps) {
    __shared__ uint32_t s_fft[SB_FRONT11N_WARPS][2][64];
    __shared__ __align__(16) uint8_t s_soft[SB_FRONT11N_WARPS][624];       // one stream-parsed symbol: 2 x 52 x N_BPSC soft values (SIG phase: 3 x 48)
    __shared__ uint32_t s_dec[SB_FRONT11N_WARPS][96];
    __shared__ uint8_t s_demap[256];
    const unsigned FULL = 0xFFFFFFFFu;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_demap[i] = __ldg(N.demap + i);
    __syncthreads();
    const uint32_t f = blockIdx.x * SB_FRONT11N_WARPS + wib;
    if (f >= nframes) return;
    FrameInfo fi = info[f];
    if (fi.status != E_SUCCESS) return;
    uint8_t* sb = s_soft[wib];
    const uint32_t* xa[2] = {iq0 + off[f], iq1 + off[f]};
    const uint32_t nvec = (len[f] / 28u) * 28u / 8u;
    const uint32_t s0 = fi.detect_vec * 4u;            // first 20 Msps sample of the 128-sample L-LTF block
    if (fi.detect_vec + 32u > nvec) { if (lane == 0) info[f].status = E_NO_FRAME; return; }
    const int half = lane >> 4, hl = lane & 15;
    const int b0 = lane, b1 = lane + 32;
    const int r0 = bitrev6(b0), r1 = bitrev6(b1);
    const cs16 w64_1 = unpack(__ldg(T.tw64 + hl)), w64_2 = unpack(__ldg(T.tw64 + 16 + hl)), w64_3 = unpack(__ldg(T.tw64 + 32 + hl));
    const cs16 w16_1 = unpack(__ldg(T.tw16 + (hl & 3))), w16_2 = unpack(__ldg(T.tw16 + 4 + (hl & 3))), w16_3 = unpack(__ldg(T.tw16 + 8 + (hl & 3)));
    auto fft_from_regs = [&](cs16 a, cs16 b, cs16 c, cs16 d) {             // fft.hpp:110-135 / fft_r4dif.h FFT<64>, one transform per half-warp
        uint32_t* xb = s_fft[wib][half];
        r4_butterfly(a, b, c, d, w64_1, w64_2, w64_3);
        xb[hl] = pack(a); xb[hl + 16] = pack(b); xb[hl + 32] = pack(c); xb[hl + 48] = pack(d);
        __syncwarp();
        {   const int base = (hl >> 2) * 16 + (hl & 3);
            cs16 p = unpack(xb[base]), q = unpack(xb[base + 4]), r = unpack(xb[base + 8]), t = unpack(xb[base + 12]);
            r4_butterfly(p, q, r, t, w16_1, w16_2, w16_3);
            xb[base] = pack(p); xb[base + 4] = pack(q); xb[base + 8] = pack(r); xb[base + 12] = pack(t); }
        __syncwarp();
        {   cs16 p = unpack(xb[4 * hl]), q = unpack(xb[4 * hl + 1]), r = unpack(xb[4 * hl + 2]), t = unpack(xb[4 * hl + 3]);
            dft4(p, q, r, t);
            xb[4 * hl] = pack(p); xb[4 * hl + 1] = pack(q); xb[4 * hl + 2] = pack(r); xb[4 * hl + 3] = pack(t); }
        __syncwarp();
    };
    // ---- TFreqEstimator_11n: joint 64-lag estimate over both antennas (freqoffset_11n.hpp:42-84) ----
    int vfo_d, vfo_theta = 0;
    {
        int sr = 0, si = 0;
#pragma unroll
        for (int a = 0; a < 2; a++)
#pragma unroll
            for (int j = 0; j < 2; j++) {
                const uint32_t i = s0 + lane + 32u * j;
                int re, im; cmul_conj32(re, im, unpack(__ldg(xa[a] + 2u * i)), unpack(__ldg(xa[a] + 2u * (i + 64u))));
                sr = wadd(sr, re >> 7); si = wadd(si, im >> 7);
            }
        for (int o = 16; o; o >>= 1) { sr = wadd(sr, __shfl_xor_sync(FULL, sr, o)); si = wadd(si, __shfl_xor_sync(FULL, si, o)); }
        vfo_d = d_atan11n(N, sr, si) >> 6;
        fi.cfo_est = vfo_d;
    }
    // TFreqComp_11n (freqoffset_11n.hpp:165-216): sample n since the estimate is turned by sincos[(n d - theta) mod 2^16], product >> 15, saturating pack
    auto nco = [&](cs16 s, uint32_t n) -> cs16 {
        const cs16 co = unpack(__ldg(N.sincos + (((n * (uint32_t)vfo_d) - (uint32_t)vfo_theta) & 0xFFFFu)));
        int re, im; cmul32(re, im, s, co); return shr_sat(re, im, 15);
    };
    // 64 samples of antenna `a` starting at 20 Msps index `first` (NCO count nbase): this lane's four FFT inputs hl + 16 j
    auto load4 = [&](int a, uint32_t first, uint32_t nbase, cs16 (&v)[4]) {
#pragma unroll
        for (int j = 0; j < 4; j++) v[j] = nco(unpack(__ldg(xa[a] + 2u * (first + hl + 16u * j))), nbase + hl + 16u * j);
    };
    // ---- L-LTF: per antenna two transforms (half-warp 0: first long symbol, half-warp 1: second), legacy channel (channel_11n.hpp:34-218) ----
    cs16 ch[2][2];                                     // [antenna][b0 | b1]
    {
        auto est = [&](cs16 y, int bin) -> cs16 {      // v_siso_channel_estimation_64 for one carrier; neighbours' |y|^2 come from the lanes of the same SSE vector
            const int sq = wadd(y.re * y.re, y.im * y.im);
            const int base = lane & ~3, j = lane & 3;
            const int sa = __shfl_sync(FULL, sq, base + ((2 * j) & 3)), sbq = __shfl_sync(FULL, sq, base + ((2 * j + 1) & 3));
            if (bin >= 28 && bin <= 35) return mk(0, 0);                     // SSE vectors 7 and 8 are never written by the reference
            const int ire = wadd((int)((unsigned)y.re << 16), sa >> 1), iim = wadd((int)((unsigned)y.im << 16), sbq >> 1);
            const int d = sq ? sq : 1;
            cs16 o = mk(sat16((int)((long long)ire / d)), sat16((int)((long long)iim / d)));
            if (__ldg(N.lltf_pos + bin)) o.im = neg16(o.im); else o.re = neg16(o.re);
            return o;
        };
#pragma unroll
        for (int a = 0; a < 2; a++) {
            cs16 v[4]; load4(a, s0 + 64u * half, 64u * half, v); fft_from_regs(v[0], v[1], v[2], v[3]);
            const uint32_t* x0 = s_fft[wib][0]; const uint32_t* x1 = s_fft[wib][1];
            const cs16 e00 = est(unpack(x0[r0]), b0), e01 = est(unpack(x0[r1]), b1), e10 = est(unpack(x1[r0]), b0), e11 = est(unpack(x1[r1]), b1);
            ch[a][0] = mk(sx16(e00.re + e10.re) >> 1, sx16(e00.im + e10.im) >> 1);
            ch[a][1] = mk(sx16(e01.re + e11.re) >> 1, sx16(e01.im + e11.im) >> 1);
            __syncwarp();
            if (taps.siso) { taps.siso[((size_t)f * 2 + a) * 64 + b0] = pack(ch[a][0]); taps.siso[((size_t)f * 2 + a) * 64 + b1] = pack(ch[a][1]); }
        }
    }
    // ---- symbol machinery ----
    uint32_t status = E_SUCCESS;
    auto sym_ready = [&](uint32_t sym) { return (s0 + 128u + 80u * sym + 80u) / 4u <= nvec; };
    // FFT of symbol `sym` (0 = L-SIG) for both antennas: half-warp a transforms antenna a (T11nDataSymbol skips 16 CP samples)
    auto fft_symbol = [&](uint32_t sym) {
        cs16 v[4]; const uint32_t n0 = 128u + 80u * sym + 16u;
        load4(half, s0 + n0, n0, v); fft_from_regs(v[0], v[1], v[2], v[3]);
    };
    // ---- L-SIG, HT-SIG1, HT-SIG2 (TSisoChannelComp, TMrcCombine, T11nSigDemap, T11aDeinterleaveBPSK) ----
    const int ds0 = data_index(b0), ds1 = data_index(b1);
    for (uint32_t s = 0; s < 3 && status == E_SUCCESS; s++) {
        if (!sym_ready(s)) { status = E_NO_FRAME; break; }
        fft_symbol(s);
        auto comb = [&](int r, int w) -> cs16 {
            int re, im; cmul32(re, im, unpack(s_fft[wib][0][r]), ch[0][w]); const cs16 o1 = shr_sat(re, im, 9);
            cmul32(re, im, unpack(s_fft[wib][1][r]), ch[1][w]); const cs16 o2 = shr_sat(re, im, 9);
            return mk(sx16(o1.re + o2.re) >> 1, sx16(o1.im + o2.im) >> 1);
        };
        const cs16 m0 = comb(r0, 0), m1 = comb(r1, 1);
        auto put = [&](cs16 m, int d) {
            if (d < 0) return;
            const int v = s == 0 ? m.re : m.im;
            sb[48 * s + __ldg(inv_deint48 + d)] = s_demap[(unsigned)min(max(v, -128), 127) & 0xFF];
        };
        put(m0, ds0); put(m1, ds1);
        __syncwarp();
    }
    uint32_t mcs = MCS11N_UNPARSED, frame_length = 0, total_symbols = 0, lsig_len2 = 0, code_rate = CR_12;
    if (status == E_SUCCESS) {                         // T11nViterbiSig (viterbi.hpp:53-99) + T11nSigParser (PHY_11n.hpp:402-514)
        const uint32_t lsig = (uint32_t)warp_viterbi_sig_n<24>(sb, lane, s_dec[wib]);
        const unsigned long long ht = warp_viterbi_sig_n<48>(sb + 48, lane, s_dec[wib]);
        uint8_t sg[9];
        sg[0] = lsig & 0xFF; sg[1] = (lsig >> 8) & 0xFF; sg[2] = (lsig >> 16) & 0xFF;
#pragma unroll
        for (int i = 0; i < 6; i++) sg[3 + i] = (uint8_t)(ht >> (8 * i));
        if (taps.sig && lane < 9) taps.sig[(size_t)f * 16 + lane] = sg[lane];
        const uint32_t u = lsig & 0xFFFFFFu;
        bool ok = !(u & 0xFC0010u);
        uint32_t par = (u >> 16) ^ u; par ^= par >> 8; par ^= par >> 4; par ^= par >> 2; par ^= par >> 1;
        ok = ok && !(par & 1);
        if (ok) ok = (u & 8u) != 0;                    // BB11aParseDataRate: the eight legal codes all have bit 3 set
        if (ok) { frame_length = ((u >> 5) & 0xFFFu) * 2u; lsig_len2 = frame_length; ok = frame_length <= 1500u; }
        if (ok) {
            uint8_t c = 0xFF;
#pragma unroll
            for (int i = 0; i < 4; i++) c = __ldg(N.crc8 + (c ^ sg[3 + i]));
            c ^= sg[7] & 3;
#pragma unroll
            for (int k = 0; k < 2; k++) c = (c & 1) ? (uint8_t)((c >> 1) ^ 0xE0) : (uint8_t)(c >> 1);
            c = (uint8_t)~c;
            if (c != ((sg[7] >> 2) | (sg[8] << 6))) { mcs = 0; ok = false; }     // as int, as PHY_11n.hpp:488 compares its UCHAR
            else {
                mcs = sg[3] & 0x7F;
                if (mcs < 8 || mcs >= N.mcs_limit) ok = false;
                else {
                    const uint32_t hl16 = (uint32_t)sg[4] | ((uint32_t)sg[5] << 8);
                    if (hl16 > 1500u) ok = false;
                    else {
                        const uint32_t m8 = mcs & 7u;                                     // ieee80211n_cmn.h:7-26, ieee80211const.h:46-54
                        code_rate = m8 == 5u ? CR_23 : (m8 == 2u || m8 == 4u || m8 == 6u) ? CR_34 : CR_12;
                        const uint32_t ndbps = mcs == 8 ? 52u : mcs == 9 ? 104u : mcs == 10 ? 156u : mcs == 11 ? 208u : mcs == 12 ? 312u : mcs == 13 ? 416u : 468u;
                        total_symbols = (hl16 * 8u + 16u + 6u + ndbps - 1u) / ndbps + 4u;
                        frame_length = hl16;
                    }
                }
            }
        }
        if (!ok) status = E_PLCP_HEADER_FAIL;
    }
    fi.rate_kbps = mcs; fi.length = frame_length; fi.nsym_total = total_symbols; fi.code_rate = code_rate; fi.peak_index = lsig_len2;
    uint32_t soft_bytes = 0;
    if (status == E_SUCCESS) {
        // ---- HT-STF (dropped), HT-LTF x2: TMimoChannelEst (channel_11n.hpp:331-442) ----
        cs16 hv[4][2];                                 // inverse channel [h11^-1.. order inv11, inv12, inv21, inv22][b0 | b1]
        {
            cs16 y1[2][2];                             // first HT-LTF: [antenna][b0 | b1]
            if (!sym_ready(5)) status = E_NO_FRAME;
            else {
                fft_symbol(4);
#pragma unroll
                for (int a = 0; a < 2; a++) { y1[a][0] = unpack(s_fft[wib][a][r0]); y1[a][1] = unpack(s_fft[wib][a][r1]); }
                __syncwarp();
                fft_symbol(5);
#pragma unroll
                for (int w = 0; w < 2; w++) {
                    const int bin = w ? b1 : b0, r = w ? r1 : r0;
                    const bool plus = __ldg(N.htltf_pos + bin) != 0;
                    cs16 h[4];
#pragma unroll
                    for (int a = 0; a < 2; a++) {
                        const cs16 p = y1[a][w], q = unpack(s_fft[wib][a][r]);
                        cs16 d = sra(subs(p, q), 1), s = sra(adds(p, q), 1);
                        if (!plus) { d = mk(neg16(d.re), neg16(d.im)); s = mk(neg16(s.re), neg16(s.im)); }
                        h[2 * a] = d; h[2 * a + 1] = s;
                    }
                    const cfl A = {(float)h[0].re, (float)h[0].im}, B = {(float)h[1].re, (float)h[1].im}, C = {(float)h[2].re, (float)h[2].im}, D = {(float)h[3].re, (float)h[3].im};
                    const cfl ad = cmulf(A, D), bc = cmulf(B, C);
                    const cfl det = {__fsub_rn(ad.re, bc.re), __fsub_rn(ad.im, bc.im)};
                    const float nn = __fdiv_rn(__fadd_rn(__fmul_rn(det.re, det.re), __fmul_rn(det.im, det.im)), 65536.0f);
                    const cfl dsx = {det.re, -det.im}, nb = {-B.re, -B.im}, nc = {-C.re, -C.im};
                    const cfl rr[4] = {cmulf(D, dsx), cmulf(nb, dsx), cmulf(nc, dsx), cmulf(A, dsx)};
#pragma unroll
                    for (int q4 = 0; q4 < 4; q4++) hv[q4][w] = mk(sat16(cvt_x86(__fdiv_rn(rr[q4].re, nn))), sat16(cvt_x86(__fdiv_rn(rr[q4].im, nn))));
                }
                __syncwarp();
                if (taps.hinv)
#pragma unroll
                    for (int q4 = 0; q4 < 4; q4++) { taps.hinv[((size_t)f * 4 + q4) * 64 + b0] = pack(hv[q4][0]); taps.hinv[((size_t)f * 4 + q4) * 64 + b1] = pack(hv[q4][1]); }
            }
        }
        // ---- data symbols ----
        const int nbpsc = mcs == 8 ? 1 : mcs <= 10 ? 2 : mcs <= 12 ? 4 : 6;
        const int q = mcs == 8 ? 0 : 1, nss = 52 * nbpsc;           // q: BPSK / QPSK position map (the 16-/64-QAM branches look theirs up per symbol)
        const int dh0 = ht_data_index(b0), dh1 = ht_data_index(b1);
        uint8_t pz[2][2][2];                            // [b0 | b1][stream][re | im] position in the stream-parsed symbol
#pragma unroll
        for (int w = 0; w < 2; w++)
#pragma unroll
            for (int s = 0; s < 2; s++)
#pragma unroll
                for (int c = 0; c < 2; c++) {
                    const int d = w ? dh1 : dh0;
                    pz[w][s][c] = (d >= 0 && c <= q) ? __ldg(N.pos + (q * 2 + s) * 104 + d * (q + 1) + c) : (uint8_t)0;
                }
        uint8_t* sout = soft_out + (size_t)f * soft_stride;
        const uint32_t ndata = total_symbols - 4u;
        for (uint32_t n = 0; n < ndata && status == E_SUCCESS; n++) {
            const uint32_t sym = 6u + n;
            if (!sym_ready(sym)) { status = E_NO_FRAME; break; }
            fft_symbol(sym);
            cs16 X[2][2];                               // [stream][b0 | b1]   TMimoChannelComp (channel_11n.hpp:446-521)
#pragma unroll
            for (int w = 0; w < 2; w++) {
                const cs16 ya = unpack(s_fft[wib][0][w ? r1 : r0]), yb = unpack(s_fft[wib][1][w ? r1 : r0]);
#pragma unroll
                for (int s = 0; s < 2; s++) {
                    int pr, pi, qr, qi; cmul32(pr, pi, hv[2 * s][w], ya); cmul32(qr, qi, hv[2 * s + 1][w], yb);
                    X[s][w] = shr_sat(wadd(pr, qr), wadd(pi, qi), 9);
                }
            }
            if (taps.eq && n < taps.max_sym)
#pragma unroll
                for (int s = 0; s < 2; s++) { const size_t o = (((size_t)f * 2 + s) * taps.max_sym + n) * 64; taps.eq[o + b0] = pack(X[s][0]); taps.eq[o + b1] = pack(X[s][1]); }
            {   // TPilotTrack_11n (pilot_11n.hpp:84-141): mean of the four pilot angles per stream, no polarity (atan is pi-periodic)
                // bins 7 and 21 sit in the first bin of lanes 7 / 21, bins 43 and 57 in the second bin of lanes 11 / 25: one pair of table walks
                const bool lo = lane == 7 || lane == 21, hi = lane == 11 || lane == 25;
                const cs16 p0 = hi ? X[0][1] : X[0][0], p1 = hi ? X[1][1] : X[1][0];
                int t0 = d_atan11n<true>(N, p0.re, p0.im), t1 = d_atan11n<true>(N, p1.re, p1.im);
                if (!(lo || hi)) { t0 = 0; t1 = 0; }
                t0 = __reduce_add_sync(FULL, t0); t1 = __reduce_add_sync(FULL, t1);
                const int th0 = sx16(t0 >> 2), th1 = sx16(t1 >> 2);
                vfo_theta = sx16(vfo_theta + sx16((th0 + th1) >> 1));
                if (taps.theta && n < taps.max_sym && lane == 0) taps.theta[(size_t)f * taps.max_sym + n] = (int16_t)vfo_theta;
            }
            if (nbpsc <= 2) {
#pragma unroll
                for (int w = 0; w < 2; w++) {
                    if ((w ? dh1 : dh0) < 0) continue;
#pragma unroll
                    for (int s = 0; s < 2; s++) {
                        sb[pz[w][s][0]] = s_demap[(unsigned)min(max(X[s][w].re, -128), 127) & 0xFF];
                        if (q) sb[pz[w][s][1]] = s_demap[(unsigned)min(max(X[s][w].im, -128), 127) & 0xFF];
                    }
                }
            } else demap_qam11n(sb, N.pos16, N.demap16, N.demap64, nbpsc, dh0, dh1, pack(X[0][0]), pack(X[0][1]), pack(X[1][0]), pack(X[1][1]));
            __syncwarp();
            {   uint32_t* dst = (uint32_t*)(sout + soft_bytes); const uint32_t* src = (const uint32_t*)sb; const int nw = nss >> 1;   // 26 x N_BPSC words
                for (int i = lane; i < nw; i += 32) dst[i] = src[i]; }
            soft_bytes += 2 * nss;
            __syncwarp();
        }
    }
    if (lane == 0) { fi.status = status; fi.soft_bytes = soft_bytes; fi.ncbps = 104; info[f] = fi; }
}

} // namespace sb
