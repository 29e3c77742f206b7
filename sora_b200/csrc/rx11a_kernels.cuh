// sora_b200 — 802.11a receive kernels (sm_90a).
//
//   k_sync11a    one thread per capture slot: 2:1 decimation, DC removal/estimation and the STS carrier-sense
//                state machine, up to the vector where the reference switches to the demod branch.
//                Reference: samples.hpp:27-49 (TDownSample2), dc.hpp:48-166, cca.hpp:106-441 (TCCA11a),
//                fb11a_demod.cpp:29-81 (per-28-sample-block error polling, CS-timeout reset).
//   k_front11a   one quarter-warp per slot: LTS (fine CFO, FFT, channel estimate), then per OFDM symbol
//                CP strip -> freq comp -> FFT64 -> equalise -> phase comp -> pilot track -> soft demap ->
//                de-interleave; SIGNAL decoded in-warp (K=7 Viterbi, 24 steps) and parsed.  Samples stay packed complex
//                int16 words from the load through the FFT to the demapper (pk_* in fixed.cuh, bit-exact to the scalar forms);
//                only the pilot recurrence and the channel estimate work on scalar ints.
//                Reference: channel_11a.hpp:34-230,534-653, fft.hpp:110-135, freqoffset.hpp:16-65,
//                pilot.hpp:123-269, demapper11a.hpp:11-73, deinterleaver.hpp, viterbicore.h:36-261,
//                PHY_11a.hpp:363-430,520-604.
// Data layout: IQ is the caller's interleaved int16 (I,Q) stream, one 32-bit word per 40 Msps sample; the
// 20 Msps stream is "every other word".  Soft bits leave this stage as one byte per coded bit (0..7),
// N_CBPS per symbol, contiguous per frame, ready for viterbi_k7_re.cuh.
#pragma once
#include "tables.cuh"
#include "viterbi_k7_common.cuh"
#include "bulk_copy.cuh"
#include "ofdm_bins.cuh"

namespace sb {

__device__ __forceinline__ int d_uatan2(const DevTables& T, int y, int x) {       // intalg.h:96-108
    unsigned ay = y > 0 ? (unsigned)y : 0u - (unsigned)y, ax = x > 0 ? (unsigned)x : 0u - (unsigned)x;
    int ys = ay > 1 ? 31 - __clz(ay) : 0, xs = ax > 1 ? 31 - __clz(ax) : 0;
    int shift = max(xs, ys) - 6;
    if (shift > 0) { y >>= shift; x >>= shift; }
    return (int)__ldg(&T.atan2_lut[((unsigned)y & 0xFF) * 256 + ((unsigned)x & 0xFF)]);
}
__device__ __forceinline__ uint32_t d_rotw(const DevTables& T, int th) {          // (ucos(th), -usin(th)), packed
    return __ldg(T.rot + ((unsigned)th & 0xFFFFu));
}

// ------------------------------------------------------------------------------------------------
// carrier sense
// ------------------------------------------------------------------------------------------------
struct CcaState {
    uint32_t his[4][4];       // CMovingWindow<vcs,4> of (x - DC) >> 2, packed c16
    int acr[4], aci[4], eng[4];
    int his_idx, acc_i, acr_reg, aci_reg, eng_reg;
    unsigned auto_count, sense_count, high_count; int sync_state, peak_corr, peak_index;
    unsigned dc_cnt; int dc_sum_re, dc_sum_im;
    __device__ void reset() {
        for (int i = 0; i < 4; i++) { for (int j = 0; j < 4; j++) his[i][j] = 0; acr[i] = aci[i] = eng[i] = 0; }
        his_idx = acc_i = 0; acr_reg = aci_reg = eng_reg = 0;
        auto_count = sense_count = high_count = 0; sync_state = 0; peak_corr = 0; peak_index = 0;
        dc_cnt = 8; dc_sum_re = dc_sum_im = 0;
    }
};

__device__ __forceinline__ int cca_xcorr(const CcaState& s, const uint32_t* __restrict__ pat) {   // cca.hpp:196-213
    int sre = 0, sim = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        int slot = (s.his_idx + j) & 3;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            int re, im; cmul_conj32(re, im, unpack(__ldg(pat + 4 * j + k)), unpack(s.his[slot][k]));
            sre = wadd(sre, re); sim = wadd(sim, im);
        }
    }
    return abs(sre) + abs(sim);
}

__global__ void __launch_bounds__(128) k_sync11a(const uint32_t* __restrict__ iq, const uint64_t* __restrict__ off,
                                                  const uint32_t* __restrict__ len, uint32_t nframes, uint32_t cca_thr,
                                                  DevTables T, FrameInfo* __restrict__ info, const int2* __restrict__ dc_init, uint32_t sh, uint32_t lsh) {
    // sh = 1: `iq` is the 40 Msps capture and TDownSample2 (samples.hpp:27-49) is the stride-2 gather below; sh = 0: the caller's samples were
    // decimated on the way in (host-side gather of the even samples, rx11a.cu), off[] then addresses that packed copy; len[] stays in 40 Msps samples
    uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nframes) return;
    const uint32_t* x = iq + off[f];
    const uint32_t nblk = (len[f] << lsh) / 28u;      // memsource.hpp:87: whole 28-sample source blocks only (lsh = 1: len[] counts 20 Msps samples)
    const uint32_t nvec = nblk * 28u / 8u;
    CcaState s; s.reset();
    int dc_re = dc_init ? dc_init[f].x : 0, dc_im = dc_init ? dc_init[f].y : 0;   // CF_VecDC: zero at Init, carried along a stream
    bool timeout = false; uint32_t cur_blk = 0; uint32_t detect = 0xFFFFFFFFu;
    for (uint32_t v = 0; v < nvec; v++) {
        uint32_t blk = (8u * v + 7u) / 28u;
        if (blk != cur_blk) {                          // driver polls error_code once per source block (fb11a_demod.cpp:35-58)
            if (timeout) { s.reset(); timeout = false; }
            cur_blk = blk;
        }
        cs16 p[4];
#pragma unroll
        for (int k = 0; k < 4; k++) p[k] = subw(unpack(__ldg(x + ((4u * v + (uint32_t)k) << sh))), mk(dc_re, dc_im));   // dc.hpp:48-85
        if (s.sync_state == 0) {                       // cca.hpp:326-398
            int sr = 0, si = 0, se = 0; uint32_t pk[4];
            const int oldest = s.his_idx;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                cs16 q = sra(p[k], 2); pk[k] = pack(q);
                int re, im; cmul_conj32(re, im, q, unpack(s.his[oldest][k]));
                sr = wadd(sr, re >> 4); si = wadd(si, im >> 4);
                se = wadd(se, wadd(q.re * q.re, q.im * q.im) >> 4);
            }
            int a = s.acc_i;
            s.acr_reg = s.acr_reg + sr - s.acr[a]; s.acr[a] = sr;
            s.aci_reg = s.aci_reg + si - s.aci[a]; s.aci[a] = si;
            s.eng_reg = s.eng_reg + se - s.eng[a]; s.eng[a] = se;
            s.acc_i = (a + 1) & 3;
            int iAuto = abs(s.acr_reg) + abs(s.aci_reg), iEnergy = s.eng_reg;
#pragma unroll
            for (int k = 0; k < 4; k++) s.his[oldest][k] = pk[k];
            s.his_idx = (oldest + 1) & 3;
            s.sense_count += 4;
            if (iEnergy > (int)cca_thr && iAuto >= iEnergy - (iEnergy >> 3)) {
                s.auto_count++; s.sense_count = 0;
                if (s.auto_count >= 4) {               // establish_sync, cca.hpp:220-243
                    int sum = 0; s.peak_corr = 0;
                    for (int i = 0; i < 16; i++) {
                        int c = cca_xcorr(s, T.sts + 16 * i);
                        if (c > s.peak_corr) { s.peak_corr = c; s.peak_index = i; }
                        sum += c;
                    }
                    if (s.peak_corr > (sum >> 3)) {
                        s.sync_state = 1; s.high_count = 0;
                        if (s.peak_index > 3) { s.high_count = (unsigned)(s.peak_index / 4); s.peak_index &= 3; }
                    }
                }
            } else s.auto_count = 0;
        } else {                                       // cca.hpp:399-418
            const int oldest = s.his_idx;
#pragma unroll
            for (int k = 0; k < 4; k++) s.his[oldest][k] = pack(sra(p[k], 2));
            s.his_idx = (oldest + 1) & 3;
            s.high_count++;
            if ((s.high_count & 3) == 0) {
                int c = cca_xcorr(s, T.sts + 16 * s.peak_index);     // check_sync, cca.hpp:245-263
                if (c < (s.peak_corr >> 1)) {
                    if (s.high_count > 8) { detect = v + 1; break; }
                    s.sync_state = 0; s.sense_count = 0;
                } else if (c > s.peak_corr) s.peak_corr = c;
            }
        }
        if (s.sync_state == 0) {                       // TDCEstimator behind the energy gate (dc.hpp:101-166)
            int hr = 0, hi = 0;
#pragma unroll
            for (int k = 0; k < 4; k++) { hr += p[k].re >> 5; hi += p[k].im >> 5; }
            s.dc_sum_re = sx16(s.dc_sum_re + sx16(hr)); s.dc_sum_im = sx16(s.dc_sum_im + sx16(hi));
            if (s.dc_cnt == 0) {
                dc_re = sx16(dc_re + (s.dc_sum_re >> 2)); dc_im = sx16(dc_im + (s.dc_sum_im >> 2));
                s.dc_cnt = 8; s.dc_sum_re = s.dc_sum_im = 0;
            }
            s.dc_cnt--;
            if (s.sense_count >= 84) timeout = true;   // cca.hpp:431-437
        }
    }
    FrameInfo fi;
    fi.status = detect == 0xFFFFFFFFu ? (uint32_t)E_NO_FRAME : (uint32_t)E_SUCCESS;
    fi.detect_vec = detect; fi.rate_kbps = 6000; fi.length = 0; fi.nsym_total = 0; fi.code_rate = CR_12; fi.ncbps = 48;
    fi.soft_bytes = 0; fi.cfo_est = 0; fi.peak_index = (uint32_t)s.peak_index; fi.dc_re = dc_re; fi.dc_im = dc_im;
    info[f] = fi;
}

// ------------------------------------------------------------------------------------------------
// warp-wide helpers for the per-symbol front end
// ------------------------------------------------------------------------------------------------
// 64-point fixed-point FFT on a warp-private 64-word shared buffer (packed c16), in place, natural-order
// input -> bit-reversed storage (fft_r4dif.h:134-141; the caller reads bin i from slot bitrev6(i)).
__device__ __forceinline__ void warp_fft64(uint32_t* x, const DevTables& T, int lane) {
    __syncwarp();
    if (lane < 16) {                                   // FFTSSE<64>: 16 radix-4 butterflies at stride 16
        cs16 a = unpack(x[lane]), b = unpack(x[lane + 16]), c = unpack(x[lane + 32]), d = unpack(x[lane + 48]);
        r4_butterfly(a, b, c, d, unpack(__ldg(T.tw64 + lane)), unpack(__ldg(T.tw64 + 16 + lane)), unpack(__ldg(T.tw64 + 32 + lane)));
        x[lane] = pack(a); x[lane + 16] = pack(b); x[lane + 32] = pack(c); x[lane + 48] = pack(d);
    }
    __syncwarp();
    if (lane < 16) {                                   // 4 x FFTSSE<16>: stride 4 inside each quarter
        int base = (lane >> 2) * 16, fidx = lane & 3;
        cs16 a = unpack(x[base + fidx]), b = unpack(x[base + fidx + 4]), c = unpack(x[base + fidx + 8]), d = unpack(x[base + fidx + 12]);
        r4_butterfly(a, b, c, d, unpack(__ldg(T.tw16 + fidx)), unpack(__ldg(T.tw16 + 4 + fidx)), unpack(__ldg(T.tw16 + 8 + fidx)));
        x[base + fidx] = pack(a); x[base + fidx + 4] = pack(b); x[base + fidx + 8] = pack(c); x[base + fidx + 12] = pack(d);
    }
    __syncwarp();
    if (lane < 16) {                                   // 16 x FFTSSEEx<4>
        cs16 a = unpack(x[4 * lane]), b = unpack(x[4 * lane + 1]), c = unpack(x[4 * lane + 2]), d = unpack(x[4 * lane + 3]);
        dft4(a, b, c, d);
        x[4 * lane] = pack(a); x[4 * lane + 1] = pack(b); x[4 * lane + 2] = pack(c); x[4 * lane + 3] = pack(d);
    }
    __syncwarp();
}

// SIGNAL-field Viterbi, one warp: lane l owns the butterfly (l, l+32) -> (2l, 2l+1).  uint8 metrics with the
// reference's wrap/mark/min/normalise rules (viterbicore.h:36-261).  `soft` = 48 deinterleaved values in shared; `dec` = 48 words of
// the warp's shared memory for the decision ballots (even states 0..23, odd states 24..47), kept out of the registers of the caller.
__device__ __forceinline__ uint32_t warp_viterbi_signal(const uint8_t* soft, uint32_t* dec, int lane) {
    const unsigned FULL = 0xFFFFFFFFu;
    const int cA = ((lane >> 1) ^ (lane >> 2) ^ (lane >> 4)) & 1;          // 133o taps on the predecessor bits
    const int cB = (lane ^ (lane >> 1) ^ (lane >> 2)) & 1;                 // 171o
    int m0 = lane == 0 ? 0x00 : 0x30, m1 = 0x30;                           // viterbilut.h:22-32
#pragma unroll
    for (int t = 0; t < 24; t++) {
        int tA = 2 * soft[2 * t], tB = 2 * soft[2 * t + 1];
        int alpha = (cA ? 14 - tA : tA) + (cB ? 14 - tB : tB), beta = 28 - alpha;
        int n0 = min((m0 + alpha) & 0xFE, ((m1 + beta) & 0xFF) | 1);
        int n1 = min((m0 + beta) & 0xFE, ((m1 + alpha) & 0xFF) | 1);
        const uint32_t dE = __ballot_sync(FULL, n0 & 1), dO = __ballot_sync(FULL, n1 & 1);
        if (lane == 0) { dec[t] = dE; dec[24 + t] = dO; }
        int w = n0 | (n1 << 8);
        int wa = __shfl_sync(FULL, w, lane >> 1), wb = __shfl_sync(FULL, w, 16 + (lane >> 1));
        int sh = 8 * (lane & 1);
        m0 = (wa >> sh) & 0xFF; m1 = (wb >> sh) & 0xFF;
        if (((t + 1) & 7) == 0) {
            int mn = __reduce_min_sync(FULL, min(m0, m1)) & 0xFE;
            m0 = (m0 - mn) & 0xFF; m1 = (m1 - mn) & 0xFF;
        }
    }
    // the extra normalise before the traceback (viterbicore.h:176-188) only subtracts a constant: order unchanged
    unsigned key = min(((unsigned)m0 << 8) | ((unsigned)lane << 2), ((unsigned)m1 << 8) | ((unsigned)(lane + 32) << 2));
    key = __reduce_min_sync(FULL, key);
    __syncwarp();                                      // lane 0's ballot words are visible to every lane
    int pos = (int)(key >> 2) & 0x7F;
    uint32_t word = 0;
#pragma unroll
    for (int i = 0; i < 24; i++) {                     // viterbicore.h:244-260; bit i of the result is time 23-i
        word |= (uint32_t)((pos >> 6) & 1) << (23 - i);
        pos = (pos >> 1) & 0x3F;
        int col = 23 - i;                              // decisions of column `col` (1-based col = t+1 -> index t), column 0 = init (all even)
        int bit = 0;
        if (col >= 1) { uint32_t wsel = dec[(pos & 1) * 24 + col - 1]; bit = (wsel >> (pos >> 1)) & 1; }
        pos |= bit << 6;
    }
    return word >> 6;                                  // viterbi.hpp:39
}

// ------------------------------------------------------------------------------------------------
// front end: one quarter-warp per slot
// ------------------------------------------------------------------------------------------------
struct FrontTaps {            // optional stage taps (device pointers, nullptr = off); per slot, per symbol, 64 packed c16
    uint32_t* freq_coeffs; uint32_t* chan_coeffs; uint32_t* fft_out; uint32_t* equalized; uint32_t* tracked; uint32_t max_sym;
    uint32_t hdr_only;        // stop after SIGNAL: status = E_SUCCESS (all symbols of the frame lie in the slot) / E_NO_FRAME (they do not) / E_PLCP_HEADER_FAIL
};

// Post-FFT role of lane ql of a quarter-warp: eight bins.  Bins 0-5 are three data-subcarrier pairs (d, d + 3), d = 6 (q / 3) + q % 3
// for q = ql + 8 p, p = 0..2 (bins 2 p, 2 p + 1), in demapper order: at 64-QAM the 802.11a de-interleaver puts coded bit i of d at an
// even position and bit (2 0 1 5 3 4)[i] of d + 3 right after it, so a pair's soft bits leave as six 16-bit stores.  Bin 6 is a pilot in
// lanes 0-3 (43, 57, 7, 21) and a zero bin in lanes 4-7, bin 7 a zero bin in every lane: of the twelve zero bins z(m) (0, 27..37),
// lane ql holds z(ql) in bin 7 and, from lane 4 on, z(ql + 4) in bin 6.  Every lane so demaps three pairs and walks one pilot angle
// (bin 6; lanes 4-7 walk a zero bin's and nobody reads it), and bin 7 needs no work behind the FFT but the stage taps.
__device__ __forceinline__ int front_pair(int ql, int p) { const int q = ql + 8 * p; return 6 * (q / 3) + q % 3; }
__device__ __forceinline__ int front_zero(int m) { return m ? 26 + m : 0; }
__device__ __forceinline__ int front_bin(int ql, int i) {
    if (i < 6) return data_bin(front_pair(ql, i >> 1) + 3 * (i & 1));
    if (i == 7) return front_zero(ql);
    return ql < 4 ? (0x1507392B >> (8 * ql)) & 0xFF : front_zero(ql + 4);
}

#define SB_FRONT_WARPS 4
#define SB_FRONT_SLOTS (4 * SB_FRONT_WARPS)   // capture slots per CTA, one per quarter-warp
#ifndef SB_FRONT_MINB
#define SB_FRONT_MINB 4           // resident CTAs per SM the register allocation aims at (tools/front_sweep.sh, DESIGN.md §8)
#endif
#define SB_FRONT_FFT_ROW 68       // words per quarter's FFT buffer: the radix-16 stage's loads of the four quarters fall on distinct banks
#define SB_FRONT_LANE_ROW 52      // words per lane of per-lane constants: 16-byte loads of the eight lanes of a quarter on distinct banks
#define SB_FRONT_STAGE_WORDS 168  // STAGE 2: words per staging buffer (160 words of a symbol at 40 Msps + alignment slack)
#define SB_FRONT_STAGE_SMEM (SB_FRONT_WARPS * 4 * 2 * SB_FRONT_STAGE_WORDS * 4)   // STAGE 2's dynamic shared memory per CTA, bytes
// Each quarter-warp decodes its own slot, and all four run the same instruction stream: lanes 8 s .. 8 s + 7 slot 4 w + s of warp w.
// Per OFDM symbol a quarter runs the three radix stages of its slot's 64-point FFT (16 butterflies per stage, two per lane), the first
// stage straight from the freq-compensated time samples in registers; behind the FFT each lane owns eight bins (front_bin), and the work
// that does not grow with the bins a lane owns (pilot angle walk, tracker, control) serves four slots at once.  A quarter whose slot ended,
// failed its header or held no frame idles in the loop with the others, so every full-mask shuffle and __syncwarp still sees all 32 lanes.
// STAGE: how the time samples of the symbols reach the FFT (A/B of the staging experiment, DESIGN.md §4):
//   0  loaded straight into registers right before the transform;
//   1  the next symbol's samples are loaded into registers while the current one is processed (register double buffer; the default);
//   2  one lane of each quarter starts a 1-D bulk asynchronous copy (cp.async.bulk, the TMA unit; SASS UBLKCP) of its slot's next symbol
//      into a shared-memory double buffer (dynamic shared memory, SB_FRONT_STAGE_SMEM), completion on an mbarrier; the lanes then read
//      their samples from shared memory.
template <int STAGE>
__global__ void __launch_bounds__(32 * SB_FRONT_WARPS, SB_FRONT_MINB) k_front11a(const uint32_t* __restrict__ iq, const uint64_t* __restrict__ off,
        const uint32_t* __restrict__ len, uint32_t nframes, DevTables T, FrameInfo* __restrict__ info,
        uint8_t* __restrict__ soft_out, uint64_t soft_stride, const uint16_t* __restrict__ inv_deint, FrontTaps taps, uint32_t sh, uint32_t lsh) {
    __shared__ __align__(16) uint32_t s_fft[SB_FRONT_WARPS][4][SB_FRONT_FFT_ROW];
    __shared__ __align__(16) uint8_t s_soft[SB_FRONT_WARPS][4][288];
    __shared__ uint32_t s_demap[256];                  // per input value: [bpsk/qpsk/first bit | 16-QAM second | 64-QAM second | 64-QAM third] soft bits
    __shared__ uint8_t s_pilot[128];
    __shared__ uint32_t s_dec[SB_FRONT_WARPS][48];     // SIGNAL decoder's decision ballots, one SIGNAL at a time
    // Per-lane constants of the symbol loop, kept out of the registers: words 0-23 the equaliser factors of the eight bins (cfac re, im,
    // nim), 24-31 the signed subcarrier numbers, 32-49 the soft-bit positions of the three pairs (see load_positions).
    __shared__ __align__(16) int s_lane[SB_FRONT_WARPS][32][SB_FRONT_LANE_ROW];
    extern __shared__ __align__(16) uint32_t s_stage[];   // STAGE 2: [SB_FRONT_WARPS][4 quarters][2 buffers][SB_FRONT_STAGE_WORDS]
    __shared__ __align__(8) unsigned long long s_mbar[STAGE == 2 ? SB_FRONT_WARPS : 1][4][2];
    const unsigned FULL = 0xFFFFFFFFu;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int qt = lane >> 3, ql = lane & 7;
    if (STAGE == 2 && ql == 0) mbar_init(smem_addr(&s_mbar[wib][qt][0]), 2);
    for (int i = threadIdx.x; i < 256; i += blockDim.x)
        s_demap[i] = (uint32_t)__ldg(T.demap + i) | ((uint32_t)__ldg(T.demap + 256 + i) << 8) | ((uint32_t)__ldg(T.demap + 512 + i) << 16) | ((uint32_t)__ldg(T.demap + 768 + i) << 24);
    for (int i = threadIdx.x; i < 128; i += blockDim.x) s_pilot[i] = __ldg(T.pilot_neg + i);
    __syncthreads();
    const uint32_t f = 4u * (blockIdx.x * SB_FRONT_WARPS + (uint32_t)wib) + (uint32_t)qt;
    FrameInfo fi;
    bool act = f < nframes;                            // this quarter's slot is still being decoded
    if (act) { fi = info[f]; act = fi.status == E_SUCCESS; }
    const uint32_t* x = iq + (act ? off[f] : 0);
    const uint32_t nvec = act ? ((len[f] << lsh) / 28u) * 28u / 8u : 0u;
    const uint32_t s0 = fi.detect_vec * 4u;            // first 20 Msps sample of the 144-sample LTS block
    if (act && fi.detect_vec + 36u > nvec) { if (ql == 0) info[f].status = E_NO_FRAME; act = false; }
    const bool own = act;                              // this quarter writes its slot's FrameInfo back at the end
    if (!__any_sync(FULL, act)) return;
    // FFTSSE<64> butterflies e = ql (twiddles wa) and e = ql + 8 (wb); FFTSSE<16> butterflies b = ql and b = ql + 8 share twiddle ql & 3
    const cfac wa1 = fac_tw(unpack(__ldg(T.tw64 + ql))), wa2 = fac_tw(unpack(__ldg(T.tw64 + 16 + ql))), wa3 = fac_tw(unpack(__ldg(T.tw64 + 32 + ql)));
    const cfac wb1 = fac_tw(unpack(__ldg(T.tw64 + 8 + ql))), wb2 = fac_tw(unpack(__ldg(T.tw64 + 24 + ql))), wb3 = fac_tw(unpack(__ldg(T.tw64 + 40 + ql)));
    const cfac w16_1 = fac_tw(unpack(__ldg(T.tw16 + (ql & 3)))), w16_2 = fac_tw(unpack(__ldg(T.tw16 + 4 + (ql & 3)))), w16_3 = fac_tw(unpack(__ldg(T.tw16 + 8 + (ql & 3))));
    uint32_t* const xb = s_fft[wib][qt];
    // 64-point FFT of eight freq-compensated time samples per lane (v[k] = sample ql + 8 k), this quarter's buffer; packed words throughout
    auto fft_from_regs = [&](uint32_t (&v)[8]) {
        pk_r4_butterfly(v[0], v[2], v[4], v[6], wa1, wa2, wa3);            // FFTSSE<64>, butterfly e = ql: samples e, e + 16, e + 32, e + 48
        pk_r4_butterfly(v[1], v[3], v[5], v[7], wb1, wb2, wb3);            // butterfly e = ql + 8
#pragma unroll
        for (int k = 0; k < 8; k++) xb[ql + 8 * k] = v[k];
        __syncwarp();
        {   const int base = (ql >> 2) * 16 + (ql & 3);                    // 4 x FFTSSE<16>: butterflies b = ql (base) and b = ql + 8 (base + 32)
            uint32_t p = xb[base], q = xb[base + 4], r = xb[base + 8], t = xb[base + 12];
            uint32_t p2 = xb[base + 32], q2 = xb[base + 36], r2 = xb[base + 40], t2 = xb[base + 44];
            pk_r4_butterfly(p, q, r, t, w16_1, w16_2, w16_3);
            pk_r4_butterfly(p2, q2, r2, t2, w16_1, w16_2, w16_3);
            xb[base] = p; xb[base + 4] = q; xb[base + 8] = r; xb[base + 12] = t;
            xb[base + 32] = p2; xb[base + 36] = q2; xb[base + 40] = r2; xb[base + 44] = t2; }
        __syncwarp();
        {   uint4* const x4 = (uint4*)xb;                                  // 16 x FFTSSEEx<4>: vectors ql and ql + 8, one 16-byte word each
            uint4 a = x4[ql], b = x4[ql + 8];
            pk_dft4(a.x, a.y, a.z, a.w);
            pk_dft4(b.x, b.y, b.z, b.w);
            x4[ql] = a; x4[ql + 8] = b; }
        __syncwarp();
    };
    // ---- T11aLTS (channel_11a.hpp:34-230) -----------------------------------------------------------
    {   // FreqOffsetEstimate<16> (dspalg.hpp:227-243): sum over the 64 samples of (LTS2 * conj(LTS1 >> 1)) >> 5, wrapping adds in any order
        int sr = 0, si = 0;
        if (act) {
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const uint32_t n = (uint32_t)ql + 8u * j;
                const cs16 l = sra(unpack(__ldg(x + ((s0 + 8u + n) << sh))), 1), h = unpack(__ldg(x + ((s0 + 72u + n) << sh)));
                int re, im; cmul_conj32(re, im, h, l);
                sr = wadd(sr, re >> 5); si = wadd(si, im >> 5);
            }
        }
        for (int o = 4; o; o >>= 1) { sr = wadd(sr, __shfl_xor_sync(FULL, sr, o)); si = wadd(si, __shfl_xor_sync(FULL, si, o)); }
        fi.cfo_est = (int)(short)(((uint32_t)d_uatan2(T, si, sr)) / 64u);  // short / size_t (dspalg.hpp:242)
    }
    rfac fcv[8];                                       // FreqCoeffs of this lane's eight time samples (dspalg.hpp:201-208)
#pragma unroll
    for (int j = 0; j < 8; j++) fcv[j] = fac_rotw(d_rotw(T, fi.cfo_est * (ql + 8 * j)));
    auto fcomp = [&](uint32_t w, int j) { return pk_cmul((int)(short)w >> 1, (int)w >> 17, fcv[j]); };   // cmul_q15(sra(w, 1), FreqCoeffs)
    auto load8 = [&](uint32_t first, uint32_t (&v)[8]) {  // (x >> 1) * FreqCoeffs for samples first + ql + 8 j; zeros in a quarter that idles
#pragma unroll
        for (int j = 0; j < 8; j++) v[j] = 0u;
        if (act) {
#pragma unroll
            for (int j = 0; j < 8; j++) v[j] = fcomp(__ldg(x + ((first + ql + 8u * j) << sh)), j);
        }
    };
    {   uint32_t v[8]; load8(s0 + 8u, v); fft_from_regs(v); }      // LTS1
    int* const tab = s_lane[wib][lane];
    const int4* const tab4 = (const int4*)tab;
    int rb[8];                                         // where bin i of this lane sits in the bit-reversed FFT output
    {   // channel_11a.hpp:124-171: H^-1 = (+-1600 conj(Y)) / (|Y|^2 >> 8), C integer division
        auto inv = [&](cs16 y, int bin) -> cs16 {
            if (bin >= 28 && bin <= 35) return mk(0, 0);
            int e = wadd(y.re * y.re, y.im * y.im) >> 8;
            int L = __ldg(T.lts_pos + bin) ? 1600 : -1600;
            int re, im; cmul_conj32(re, im, mk(L, 0), y);
            return e ? mk(sx16(re / e), sx16(im / e)) : mk(0, 0);
        };
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int b = front_bin(ql, i);
            rb[i] = bitrev6(b);
            const cs16 ch = inv(unpack(xb[rb[i]]), b);
            // bins 28..35 (SSE vectors 7,8) are forced to zero: their channel coefficient is zero, so is everything multiplied by it
            const cfac eq = fac_mul8(ch);
            tab[3 * i] = eq.re; tab[3 * i + 1] = eq.im; tab[3 * i + 2] = eq.nim;
            tab[24 + i] = b < 32 ? b : b - 64;
            if (taps.freq_coeffs && own) { taps.freq_coeffs[(size_t)f * 64 + b] = d_rotw(T, fi.cfo_est * b); taps.chan_coeffs[(size_t)f * 64 + b] = pack(ch); }
        }
    }
    __syncwarp();
    // ---- symbols -----------------------------------------------------------------------------------
    rfac comp[7];                                      // bins 0-6; bin 7 is never rotated
#pragma unroll
    for (int i = 0; i < 7; i++) comp[i] = fac_rotw(0x7fffu);
    // The tracker's accumulators only ever index the rotation table (mod 2^16) and feed each other by addition, so they wrap mod 2^32
    // instead of being truncated with sx16 at every step: the low 16 bits are the same.
    uint32_t CFO_comp = 0, SFO_comp = 0, CFO_tr = 0, SFO_tr = 0; unsigned symbol_count = 127;
    uint32_t remain = 0; uint32_t soft_bytes = 0; int nbpsc = 1;
    uint8_t* sout = soft_out + (size_t)f * soft_stride;
    uint32_t status = E_SUCCESS;
    // Where this lane's soft bits go after de-interleaving, as byte offsets into s_soft, words 32 + 6 p + i of the lane's row for pair p: at
    // 64-QAM bit i of d is at the even position (the 16-bit store of the pair); at the other rates the low half is bit i of d, the high half
    // bit i of d + 3.
    auto load_positions = [&](int nb) {
        const uint16_t* inv = inv_deint + (nb == 1 ? 0 : nb == 2 ? 48 : nb == 4 ? 144 : 336);
        const uint32_t base = (uint32_t)(4 * wib + qt) * 288u;
#pragma unroll
        for (int p = 0; p < 3; p++) {
            const int d = front_pair(ql, p);
#pragma unroll
            for (int i = 0; i < 6; i++) {
                uint32_t w = 0;
                if (i < nb) w = nb == 6 ? base + __ldg(inv + d * 6 + i) : (base + __ldg(inv + d * nb + i)) | ((base + __ldg(inv + (d + 3) * nb + i)) << 16);
                tab[32 + 6 * p + i] = (int)w;
            }
        }
    };
    load_positions(1);
    uint8_t* const s8 = &s_soft[0][0][0];
    const bool pil = ql < 4;                           // bin 6 is a pilot (rotated) here, a zero bin in lanes 4-7
    // everything behind the FFT for symbol `sym` of this quarter's slot, whose spectrum sits in xb
    auto post_fft = [&](uint32_t sym) {
        const int4 q0 = tab4[0], q1 = tab4[1], q2 = tab4[2], q3 = tab4[3], q4 = tab4[4], q5 = tab4[5], k0 = tab4[6], k1 = tab4[7];
        const cfac eq[7] = {{q0.x, q0.y, q0.z}, {q0.w, q1.x, q1.y}, {q1.z, q1.w, q2.x}, {q2.y, q2.z, q2.w},
                            {q3.x, q3.y, q3.z}, {q3.w, q4.x, q4.y}, {q4.z, q4.w, q5.x}};
        const int k[7] = {k0.x, k0.y, k0.z, k0.w, k1.x, k1.y, k1.z};
        uint32_t F[7]; int ex[7], ey[7], C[7][2];
#pragma unroll
        for (int i = 0; i < 7; i++) {
            F[i] = xb[rb[i]];
            int cx, cy;                                                                  // products as 32-bit sums, value = sum >> 16
            pk_cmul_xy((int)(short)F[i], (int)F[i] >> 16, eq[i], ex[i], ey[i]);          // channel_11a.hpp:551-579
            pk_cmul_xy(ex[i] >> 16, ey[i] >> 16, comp[i], cx, cy);                       // freqoffset.hpp:28-30
            C[i][0] = cx >> 16; C[i][1] = cy >> 16;
        }
        // pilot.hpp:168-232: one table walk for four slots, the pilots sit in bin 6 of lanes 0-3 of each quarter (43, 57, 7, 21; 21's is sent negated)
        const bool neg = ql == 3;
        const int th = turn_pi(d_uatan2(T, neg ? -C[6][1] : C[6][1], neg ? -C[6][0] : C[6][0]), s_pilot[symbol_count]);
        const int th1 = __shfl_sync(FULL, th, 0, 8), th2 = __shfl_sync(FULL, th, 1, 8), th3 = __shfl_sync(FULL, th, 2, 8), th4 = __shfl_sync(FULL, th, 3, 8);
        symbol_count++; if (symbol_count >= 127) symbol_count = 0;
        // the angles are int16, so the sum / 4 lies in [-32768, 32767] and each difference / 28 in [-2340, 2340]: the sx16 of both is the identity
        const int avg = (th1 + th2 + th3 + th4) / 4;
        const int del = ((th3 - th1) / 28 + (th4 - th2) / 28) >> 1;
        CFO_tr += (uint32_t)(avg >> 2); SFO_tr += (uint32_t)(del >> 2);
        CFO_comp += (uint32_t)avg + CFO_tr; SFO_comp += (uint32_t)del + SFO_tr;
        // subcarriers -26..-1, 1..26 are rotated, every other bin (bin 6 of lanes 4-7, bin 7) becomes zero
        uint32_t R[7];
#pragma unroll
        for (int i = 0; i < 7; i++) {
            // next symbol's phase compensation; only the rotated bins use it, every other bin's R is zero whatever its C
            comp[i] = fac_rotw(d_rotw(T, (int)(CFO_comp + (uint32_t)k[i] * SFO_comp)));
            R[i] = pk_cmul(C[i][0], C[i][1], fac_rotw(i < 6 || pil ? d_rotw(T, avg + k[i] * del) : 0u));
        }
        if (taps.fft_out && act && sym < taps.max_sym) {
            const size_t o = ((size_t)f * taps.max_sym + sym) * 64;
            const int4 q5 = tab4[5];
            const cfac eq7 = {q5.y, q5.z, q5.w};
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const int b = front_bin(ql, i);
                const uint32_t Fi = i < 7 ? F[i] : xb[rb[7]];
                int exi = i < 7 ? ex[i] : 0, eyi = i < 7 ? ey[i] : 0;
                if (i == 7) pk_cmul_xy((int)(short)Fi, (int)Fi >> 16, eq7, exi, eyi);
                taps.fft_out[o + b] = Fi; taps.equalized[o + b] = __byte_perm((uint32_t)exi, (uint32_t)eyi, 0x7632); taps.tracked[o + b] = i < 7 ? R[i] : 0u;
            }
        }
        // soft demap (demapper.h:141-151 limit + LUTs) scattered through the inverse de-interleaver map
        {
            const int4 p0 = tab4[8], p1 = tab4[9], p2 = tab4[10], p3 = tab4[11]; const int2 p4 = *(const int2*)(tab + 48);
            const uint32_t pos[18] = {(uint32_t)p0.x, (uint32_t)p0.y, (uint32_t)p0.z, (uint32_t)p0.w, (uint32_t)p1.x, (uint32_t)p1.y,
                                      (uint32_t)p1.z, (uint32_t)p1.w, (uint32_t)p2.x, (uint32_t)p2.y, (uint32_t)p2.z, (uint32_t)p2.w,
                                      (uint32_t)p3.x, (uint32_t)p3.y, (uint32_t)p3.z, (uint32_t)p3.w, (uint32_t)p4.x, (uint32_t)p4.y};
#pragma unroll
            for (int p = 0; p < 3; p++) {
                const uint32_t c0 = pk_demap_clamp(R[2 * p]), c1 = pk_demap_clamp(R[2 * p + 1]);
                const uint32_t wr0 = s_demap[(c0 >> 4) & 0xFF], wi0 = s_demap[(c0 >> 20) & 0xFF], wr1 = s_demap[(c1 >> 4) & 0xFF], wi1 = s_demap[(c1 >> 20) & 0xFF];
                const uint32_t* ps = pos + 6 * p;
                if (nbpsc == 6) {                      // bits 0-2 are bytes 0, 2, 3 of wr, bits 3-5 those of wi; d's byte low, d + 3's high
                    auto st16 = [&](uint32_t q, uint32_t v) { *(uint16_t*)(s8 + q) = (uint16_t)v; };
                    st16(ps[0], __byte_perm(wr0, wr1, 0x70)); st16(ps[1], __byte_perm(wr0, wr1, 0x42)); st16(ps[2], __byte_perm(wr0, wr1, 0x63));
                    st16(ps[3], __byte_perm(wi0, wi1, 0x70)); st16(ps[4], __byte_perm(wi0, wi1, 0x42)); st16(ps[5], __byte_perm(wi0, wi1, 0x63));
                } else {
                    auto st8 = [&](uint32_t q, uint32_t v0w, uint32_t v1w) { s8[q & 0xFFFFu] = (uint8_t)v0w; s8[q >> 16] = (uint8_t)v1w; };
                    if (nbpsc == 1) { st8(ps[0], wr0, wr1); }
                    else if (nbpsc == 2) { st8(ps[0], wr0, wr1); st8(ps[1], wi0, wi1); }
                    else { st8(ps[0], wr0, wr1); st8(ps[1], wr0 >> 8, wr1 >> 8); st8(ps[2], wi0, wi1); st8(ps[3], wi0 >> 8, wi1 >> 8); }
                }
            }
        }
        __syncwarp();
        if (sym == 0) {                                // PHY_11a.hpp:520-604; the four quarters' SIGNALs, one after the other on the whole warp
            uint32_t sig = 0;
#pragma unroll 1
            for (int h = 0; h < 4; h++) {
                const uint32_t s = warp_viterbi_signal(s_soft[wib][h], s_dec[wib], lane); if (h == qt) sig = s;
                __syncwarp();                          // every lane's traceback has read s_dec before the next SIGNAL's ballots overwrite it
            }
            sig &= 0xFFFFFFu;
            if (act) {
                bool ok = !(sig & 0xFC0010u);
                uint32_t par = (sig >> 16) ^ sig; par ^= par >> 8; par ^= par >> 4; par ^= par >> 2; par ^= par >> 1;
                ok = ok && !(par & 1);
                uint32_t rate = 0; int nd = 0, nb = 1, cr = CR_12;
                switch (sig & 0xF) {                   // ieee80211a_cmn.h:97-157
                    case 0xB: rate = 6000; nd = 24; nb = 1; cr = CR_12; break;   case 0xF: rate = 9000; nd = 36; nb = 1; cr = CR_34; break;
                    case 0xA: rate = 12000; nd = 48; nb = 2; cr = CR_12; break;  case 0xE: rate = 18000; nd = 72; nb = 2; cr = CR_34; break;
                    case 0x9: rate = 24000; nd = 96; nb = 4; cr = CR_12; break;  case 0xD: rate = 36000; nd = 144; nb = 4; cr = CR_34; break;
                    case 0x8: rate = 48000; nd = 192; nb = 6; cr = CR_23; break; case 0xC: rate = 54000; nd = 216; nb = 6; cr = CR_34; break;
                    default: if (ok) fi.rate_kbps = 0; ok = false;    // BB11aParseDataRate() == 0 is stored before the parser gives up
                }
                const uint32_t L = (sig >> 5) & 0xFFF;
                if (ok && rate) { fi.rate_kbps = rate; fi.code_rate = cr; }
                if (ok) { fi.length = L; ok = L <= 2500; }
                if (!ok) { status = E_PLCP_HEADER_FAIL; act = false; }
                else {
                    fi.nsym_total = (L * 8 + 16 + 6 + nd - 1) / nd + 1;
                    remain = fi.nsym_total; nbpsc = nb; fi.ncbps = 48 * nb;
                    load_positions(nb);
                }
            }
        } else if (act) {                              // N_CBPS = 48 N_BPSC bytes: 3 N_BPSC 16-byte lines (soft_out and soft_stride are 16-byte aligned)
            uint4* const dst = (uint4*)(sout + soft_bytes); const uint4* const src = (const uint4*)s_soft[wib][qt];
            const int lines = 3 * nbpsc;
            if (ql < lines) dst[ql] = src[ql];
            if (ql + 8 < lines) dst[ql + 8] = src[ql + 8];
            if (ql + 16 < lines) dst[ql + 16] = src[ql + 16];
            soft_bytes += 48u * nbpsc;
        }
        __syncwarp();
        if (act) { remain--; act = remain != 0; }
    };
    auto sym_first = [&](uint32_t sym) { return s0 + 144u + 80u * sym; };                        // first sample of symbol sym (its CP)
    auto sym_ready = [&](uint32_t sym) { return (sym_first(sym) + 80u) / 4u <= nvec; };         // all 80 samples arrived
    // ---- staging (see STAGE above) ----
    const uint32_t nsamp20 = nvec * 4u;                                   // 20 Msps samples of the slot that may be read
    uint32_t raw[8] = {0, 0, 0, 0, 0, 0, 0, 0}; uint32_t raw_first = 0xFFFFFFFFu;   // STAGE 1: samples first + ql + 8 j of the prefetched symbol
    auto prefetch_regs = [&](uint32_t first) {                            // whole symbol inside the slot, else nothing
        raw_first = 0xFFFFFFFFu;
        if (act && first + 72u <= nsamp20) {
#pragma unroll
            for (int j = 0; j < 8; j++) raw[j] = __ldg(x + ((first + ql + 8u * j) << sh));
            raw_first = first;
        }
    };
    // STAGE 2: parity / first 20 Msps sample / samples per buffer, and which buffers have a copy in flight (bit b)
    uint32_t st_par[2] = {0, 0}, st_base[2] = {0, 0}, st_cnt[2] = {0, 0}, st_busy = 0;
    uint32_t* const st_buf = s_stage + (4 * wib + qt) * 2 * SB_FRONT_STAGE_WORDS;   // this quarter's two buffers
    auto stage_issue = [&](int b, uint32_t first20, uint32_t n20) {       // samples [first20, first20 + n20) of the slot -> buffer b (word index << sh)
        st_base[b] = first20; st_cnt[b] = 0;
        if (!act || first20 >= nsamp20) return;
        if (first20 + n20 > nsamp20) n20 = nsamp20 - first20;
        st_cnt[b] = n20; st_busy |= 1u << b;
        if (ql == 0) {
            const uint32_t* src = x + (first20 << sh);
            const uintptr_t a0 = (uintptr_t)src & ~(uintptr_t)15, a1 = ((uintptr_t)(src + (n20 << sh)) + 15) & ~(uintptr_t)15;
            const uint32_t bytes = (uint32_t)(a1 - a0);
            const uint32_t mb = smem_addr(&s_mbar[wib][qt][b]);
            mbar_expect_tx(mb, bytes);
            bulk_copy_g2s(smem_addr(st_buf + b * SB_FRONT_STAGE_WORDS), (const void*)a0, bytes, mb);
        }
    };
    auto stage_wait = [&](int b) {
        if (!((st_busy >> b) & 1u)) return;
        mbar_wait(smem_addr(&s_mbar[wib][qt][b]), st_par[b]);
        st_par[b] ^= 1u; st_busy &= ~(1u << b);
    };
    auto stage_load8 = [&](int b, uint32_t first, uint32_t (&v)[8]) {    // (x >> 1) * FreqCoeffs from buffer b; the buffer starts at the 16-byte line of its first sample
        const uint32_t skew = (uint32_t)(((uintptr_t)(x + (st_base[b] << sh)) & 15u) >> 2);
        const uint32_t* const buf = st_buf + b * SB_FRONT_STAGE_WORDS;
#pragma unroll
        for (int j = 0; j < 8; j++) v[j] = fcomp(buf[skew + ((first - st_base[b] + ql + 8u * j) << sh)], j);
    };
    if (STAGE == 2) stage_issue(0, sym_first(0), 80u);
    if (STAGE == 1) prefetch_regs(sym_first(0) + 8u);
    // SIGNAL, then the data symbols, one per iteration in each quarter
    for (uint32_t sym = 0; ; sym++) {
        if (act && !sym_ready(sym)) { status = E_NO_FRAME; act = false; }
        if (!__any_sync(FULL, act)) break;
        {   uint32_t v[8];
            const uint32_t first = sym_first(sym) + 8u;
            if (STAGE == 2) {
                const int b = (int)(sym & 1u);
                const bool staged = st_base[b] == sym_first(sym) && st_cnt[b] >= 80u;
                stage_wait(b);
                if (act && staged) stage_load8(b, first, v); else load8(first, v);
                __syncwarp();                                               // every lane has its samples: the other buffer's previous contents are no longer needed either
                stage_issue(b ^ 1, sym_first(sym + 1u), 80u);
            } else if (STAGE == 1) {
                if (raw_first == first) {
#pragma unroll
                    for (int j = 0; j < 8; j++) v[j] = fcomp(raw[j], j);
                } else load8(first, v);
                prefetch_regs(first + 80u);
            } else load8(first, v);
            fft_from_regs(v); }
        post_fft(sym);
        if (sym == 0 && taps.hdr_only && act) {                           // continuous-capture scout pass: where the frame ends is all the caller wants
            if (!sym_ready(fi.nsym_total - 1u)) status = E_NO_FRAME;
            act = false;
        }
    }
    if (STAGE == 2) { stage_wait(0); stage_wait(1); __syncwarp(); }       // no copy may be in flight when the CTA's shared memory is released
    if (own && ql == 0) { fi.status = status; fi.soft_bytes = soft_bytes; info[f] = fi; }
}

// ------------------------------------------------------------------------------------------------
// 44 -> 40 Msps front end (Brick11/src/44MTo40M.hpp:63-123 Down44to40, sampling.hpp:37-65 TDownSample44_40)
// ------------------------------------------------------------------------------------------------
// The reference's running interpolator is a pure function of the sample index inside the slot:
//   out[10k]     = in[11k]
//   out[10k + r] = (in[11k + r] * R[r] + in[11k + r + 1] * L[r + 1]) >> 7,  r = 1..9
// so it is a gather: one thread per output sample, coalesced reads (each input word is read by at most two threads).
__host__ __device__ inline uint32_t resampled_len_40(uint32_t len44) {      // whole 28-blocks in, whole 28-blocks out
    const uint32_t n = len44 / 28u * 28u, q = n / 11u, rem = n % 11u;
    const uint32_t m = 10u * q + (rem >= 1u ? 1u : 0u) + (rem > 2u ? rem - 2u : 0u);
    return m / 28u * 28u;
}
__global__ void __launch_bounds__(256) k_resample_44_40(const uint32_t* __restrict__ iq, const uint64_t* __restrict__ off, const uint32_t* __restrict__ len,
                                                        uint32_t nframes, uint32_t* __restrict__ out, uint64_t out_stride /*samples per slot*/,
                                                        uint64_t* __restrict__ off40, uint32_t* __restrict__ len40) {
    const uint32_t f = blockIdx.x;                      // slots on x (2^31 - 1 blocks), sample tiles on y
    if (f >= nframes) return;
    const uint32_t n40 = resampled_len_40(len[f]);
    if (blockIdx.y == 0 && threadIdx.x == 0) { off40[f] = (uint64_t)f * out_stride; len40[f] = n40; }
    const uint32_t* x = iq + off[f];
    uint32_t* y = out + (size_t)f * out_stride;
    for (uint32_t m = blockIdx.y * blockDim.x + threadIdx.x; m < n40; m += gridDim.y * blockDim.x) {
        const uint32_t k = m / 10u, r = m - 10u * k;
        if (r == 0) { y[m] = __ldg(x + 11u * k); continue; }
        const int R = r == 1 ? 115 : r == 2 ? 102 : r == 3 ? 90 : r == 4 ? 77 : r == 5 ? 64 : r == 6 ? 51 : r == 7 ? 38 : r == 8 ? 26 : 13;
        const int L = r == 1 ? 13 : r == 2 ? 26 : r == 3 ? 38 : r == 4 ? 51 : r == 5 ? 64 : r == 6 ? 77 : r == 7 ? 90 : r == 8 ? 102 : 115;
        const cs16 a = unpack(__ldg(x + 11u * k + r)), b = unpack(__ldg(x + 11u * k + r + 1u));
        y[m] = pack(mk(sx16((a.re * R + b.re * L) >> 7), sx16((a.im * R + b.im * L) >> 7)));
    }
}

} // namespace sb
