// sora_b200 — 802.11a receive kernels (sm_90a).
//
//   k_sync11a    one thread per capture slot: 2:1 decimation, DC removal/estimation and the STS carrier-sense
//                state machine, up to the vector where the reference switches to the demod branch.
//                Reference: samples.hpp:27-49 (TDownSample2), dc.hpp:48-166, cca.hpp:106-441 (TCCA11a),
//                fb11a_demod.cpp:29-81 (per-28-sample-block error polling, CS-timeout reset).
//   k_front11a   one warp per slot: LTS (fine CFO, FFT, channel estimate), then per OFDM symbol
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
    // decimated on the way in (host-side gather of the even samples, sb200.cu), off[] then addresses that packed copy; len[] stays in 40 Msps samples
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
__device__ __forceinline__ int bitrev6(int i) { return (int)(__brev((unsigned)i) >> 26); }

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
// front end: one warp per slot
// ------------------------------------------------------------------------------------------------
struct FrontTaps {            // optional stage taps (device pointers, nullptr = off); per slot, per symbol, 64 packed c16
    uint32_t* freq_coeffs; uint32_t* chan_coeffs; uint32_t* fft_out; uint32_t* equalized; uint32_t* tracked; uint32_t max_sym;
    uint32_t hdr_only;        // stop after SIGNAL: status = E_SUCCESS (all symbols of the frame lie in the slot) / E_NO_FRAME (they do not) / E_PLCP_HEADER_FAIL
};

__device__ __forceinline__ int data_index(int bin) {   // demapper11a.hpp:22-36 subcarrier order; -1 for non-data bins
    if (bin >= 38) { if (bin == 43 || bin == 57) return -1; return bin - 38 - (bin > 43) - (bin > 57); }
    if (bin >= 1 && bin <= 26) { if (bin == 7 || bin == 21) return -1; return 24 + bin - 1 - (bin > 7) - (bin > 21); }
    return -1;
}
__device__ __forceinline__ int data_bin(int d) {       // inverse of data_index, d = 0..47
    return d < 24 ? 38 + d + (d >= 5) + (d >= 18) : d - 23 + (d >= 30) + (d >= 43);
}

#define SB_FRONT_WARPS 4
#ifndef SB_FRONT_MINB
#define SB_FRONT_MINB 5           // resident CTAs per SM the register allocation aims at; front end on the H100 (tools/front_sweep.sh, DESIGN.md §8):
                                  // 4 -> 2.50 ms (123 registers), 5 -> 2.32 ms (96), 6 -> 2.83 ms (80 registers, 184 B of spill stores)
#endif
// Two OFDM symbols are transformed at once: lanes 0-15 run the three radix stages of symbol A, lanes 16-31 those of
// symbol B (16 butterflies per stage = 16 lanes, so every lane is busy); the first stage consumes the freq-compensated
// time samples straight from registers.  Only the part behind the FFT (phase compensation from the pilot recurrence)
// is serial across symbols, and there every lane owns two subcarriers.
// STAGE: how the time samples of the DATA symbols reach the FFT (A/B of the staging experiment, DESIGN.md §4):
//   0  loaded straight into registers right before the transform (round 1);
//   1  the next symbol pair's samples are loaded into registers while the current pair is processed (register double buffer);
//   2  one lane starts a 1-D bulk asynchronous copy (cp.async.bulk, the TMA unit; SASS UBLKCP) of the next pair's span into a shared-memory
//      double buffer, completion on an mbarrier; the lanes then read their samples from shared memory.
template <int STAGE>
__global__ void __launch_bounds__(32 * SB_FRONT_WARPS, SB_FRONT_MINB) k_front11a(const uint32_t* __restrict__ iq, const uint64_t* __restrict__ off,
        const uint32_t* __restrict__ len, uint32_t nframes, DevTables T, FrameInfo* __restrict__ info,
        uint8_t* __restrict__ soft_out, uint64_t soft_stride, const uint16_t* __restrict__ inv_deint, FrontTaps taps, uint32_t sh, uint32_t lsh) {
    __shared__ uint32_t s_fft[SB_FRONT_WARPS][2][64];
    __shared__ __align__(16) uint8_t s_soft[SB_FRONT_WARPS][288];
    __shared__ uint32_t s_demap[256];                  // per input value: [bpsk/qpsk/first bit | 16-QAM second | 64-QAM second | 64-QAM third] soft bits
    __shared__ uint8_t s_pilot[128];
    __shared__ uint32_t s_dec[SB_FRONT_WARPS][48];     // SIGNAL decoder's decision ballots
    __shared__ __align__(16) uint32_t s_stage[STAGE == 2 ? SB_FRONT_WARPS : 1][2][STAGE == 2 ? 328 : 4];   // 2 x (320 words of a symbol pair + alignment slack)
    __shared__ __align__(8) unsigned long long s_mbar[STAGE == 2 ? SB_FRONT_WARPS : 1][2];
    const unsigned FULL = 0xFFFFFFFFu;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    if (STAGE == 2 && lane == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"((uint32_t)__cvta_generic_to_shared(&s_mbar[wib][0])));
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"((uint32_t)__cvta_generic_to_shared(&s_mbar[wib][1])));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = threadIdx.x; i < 256; i += blockDim.x)
        s_demap[i] = (uint32_t)__ldg(T.demap + i) | ((uint32_t)__ldg(T.demap + 256 + i) << 8) | ((uint32_t)__ldg(T.demap + 512 + i) << 16) | ((uint32_t)__ldg(T.demap + 768 + i) << 24);
    for (int i = threadIdx.x; i < 128; i += blockDim.x) s_pilot[i] = __ldg(T.pilot_neg + i);
    __syncthreads();
    const uint32_t f = blockIdx.x * SB_FRONT_WARPS + wib;
    if (f >= nframes) return;
    FrameInfo fi = info[f];
    if (fi.status != E_SUCCESS) return;
    uint8_t* sb = s_soft[wib];
    const uint32_t* x = iq + off[f];
    const uint32_t nvec = ((len[f] << lsh) / 28u) * 28u / 8u;
    const uint32_t s0 = fi.detect_vec * 4u;            // first 20 Msps sample of the 144-sample LTS block
    if (fi.detect_vec + 36u > nvec) { if (lane == 0) info[f].status = E_NO_FRAME; return; }
    const int half = lane >> 4, hl = lane & 15;        // FFT role: which of the two symbols, which butterfly
    // Post-FFT role: this lane's two bins.  Lanes 0-23 own the data subcarriers d0 = 6 (lane / 3) + lane % 3 and d1 = d0 + 3 (demapper
    // order): at 64-QAM the 802.11a de-interleaver puts coded bit i of d0 at an even position and bit (2 0 1 5 3 4)[i] of d1 right after
    // it, so the pair's soft bits leave as six 16-bit stores.  Lanes 24-27 own the pilots (bins 43, 57, 7, 21) in b0, the twelve zero
    // bins (0, 27..37) fill the rest.
    const int d0 = lane < 24 ? 6 * (lane / 3) + lane % 3 : -1, d1 = lane < 24 ? d0 + 3 : -1;
    const int j24 = lane - 24;
    const int b0 = lane < 24 ? data_bin(d0) : j24 < 4 ? (0x1507392B >> (8 * j24)) & 0xFF : j24 == 4 ? 0 : 22 + j24;
    const int b1 = lane < 24 ? data_bin(d1) : 30 + j24;
    const int r0 = bitrev6(b0), r1 = bitrev6(b1);
    const cfac w64_1 = fac_tw(unpack(__ldg(T.tw64 + hl))), w64_2 = fac_tw(unpack(__ldg(T.tw64 + 16 + hl))), w64_3 = fac_tw(unpack(__ldg(T.tw64 + 32 + hl)));
    const cfac w16_1 = fac_tw(unpack(__ldg(T.tw16 + (hl & 3)))), w16_2 = fac_tw(unpack(__ldg(T.tw16 + 4 + (hl & 3)))), w16_3 = fac_tw(unpack(__ldg(T.tw16 + 8 + (hl & 3))));
    // 64-point FFT of four freq-compensated time samples per lane (n = hl + 16 j), this half-warp's buffer; packed words throughout
    auto fft_from_regs = [&](uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
        uint32_t* xb = s_fft[wib][half];
        pk_r4_butterfly(a, b, c, d, w64_1, w64_2, w64_3);                   // FFTSSE<64>, butterfly e = hl
        xb[hl] = a; xb[hl + 16] = b; xb[hl + 32] = c; xb[hl + 48] = d;
        __syncwarp();
        {   const int base = (hl >> 2) * 16 + (hl & 3);                    // 4 x FFTSSE<16>
            uint32_t p = xb[base], q = xb[base + 4], r = xb[base + 8], t = xb[base + 12];
            pk_r4_butterfly(p, q, r, t, w16_1, w16_2, w16_3);
            xb[base] = p; xb[base + 4] = q; xb[base + 8] = r; xb[base + 12] = t; }
        __syncwarp();
        {   uint32_t p = xb[4 * hl], q = xb[4 * hl + 1], r = xb[4 * hl + 2], t = xb[4 * hl + 3];
            pk_dft4(p, q, r, t);                                            // 16 x FFTSSEEx<4>
            xb[4 * hl] = p; xb[4 * hl + 1] = q; xb[4 * hl + 2] = r; xb[4 * hl + 3] = t; }
        __syncwarp();
    };
    // ---- T11aLTS (channel_11a.hpp:34-230) -----------------------------------------------------------
    {   // FreqOffsetEstimate<16> (dspalg.hpp:227-243): sum over the 64 samples of (LTS2 * conj(LTS1 >> 1)) >> 5
        const uint32_t n0 = (uint32_t)lane, n1 = n0 + 32u;
        cs16 l0 = sra(unpack(__ldg(x + ((s0 + 8u + n0) << sh))), 1), l1 = sra(unpack(__ldg(x + ((s0 + 8u + n1) << sh))), 1);
        cs16 h0 = unpack(__ldg(x + ((s0 + 72u + n0) << sh))), h1 = unpack(__ldg(x + ((s0 + 72u + n1) << sh)));
        int re0, im0, re1, im1; cmul_conj32(re0, im0, h0, l0); cmul_conj32(re1, im1, h1, l1);
        int sr = wadd(re0 >> 5, re1 >> 5), si = wadd(im0 >> 5, im1 >> 5);
        for (int o = 16; o; o >>= 1) { sr = wadd(sr, __shfl_xor_sync(FULL, sr, o)); si = wadd(si, __shfl_xor_sync(FULL, si, o)); }
        fi.cfo_est = (int)(short)(((uint32_t)d_uatan2(T, si, sr)) / 64u);  // short / size_t (dspalg.hpp:242)
    }
    rfac fcv[4];                                       // FreqCoeffs of this lane's four time samples (dspalg.hpp:201-208)
#pragma unroll
    for (int j = 0; j < 4; j++) fcv[j] = fac_rotw(d_rotw(T, fi.cfo_est * (hl + 16 * j)));
    auto fcomp = [&](uint32_t w, int j) { return pk_cmul((int)(short)w >> 1, (int)w >> 17, fcv[j]); };   // cmul_q15(sra(w, 1), FreqCoeffs)
    auto load4 = [&](uint32_t first, uint32_t (&v)[4]) {  // (x >> 1) * FreqCoeffs for samples first + hl + 16 j
#pragma unroll
        for (int j = 0; j < 4; j++) v[j] = fcomp(__ldg(x + ((first + hl + 16u * j) << sh)), j);
    };
    {   uint32_t v[4]; load4(s0 + 8u, v); fft_from_regs(v[0], v[1], v[2], v[3]); }     // both halves transform LTS1 (same data)
    cs16 ch0, ch1;
    {   // channel_11a.hpp:124-171: H^-1 = (+-1600 conj(Y)) / (|Y|^2 >> 8), C integer division
        const uint32_t* xb = s_fft[wib][0];
        auto inv = [&](cs16 y, int bin) -> cs16 {
            if (bin >= 28 && bin <= 35) return mk(0, 0);
            int e = wadd(y.re * y.re, y.im * y.im) >> 8;
            int L = __ldg(T.lts_pos + bin) ? 1600 : -1600;
            int re, im; cmul_conj32(re, im, mk(L, 0), y);
            return e ? mk(sx16(re / e), sx16(im / e)) : mk(0, 0);
        };
        ch0 = inv(unpack(xb[r0]), b0); ch1 = inv(unpack(xb[r1]), b1);
    }
    __syncwarp();
    if (taps.freq_coeffs) { taps.freq_coeffs[(size_t)f * 64 + b0] = d_rotw(T, fi.cfo_est * b0); taps.freq_coeffs[(size_t)f * 64 + b1] = d_rotw(T, fi.cfo_est * b1);
                            taps.chan_coeffs[(size_t)f * 64 + b0] = pack(ch0); taps.chan_coeffs[(size_t)f * 64 + b1] = pack(ch1); }
    // ---- symbols -----------------------------------------------------------------------------------
    const int k0 = b0 < 32 ? b0 : b0 - 64, k1 = b1 < 32 ? b1 : b1 - 64;   // signed subcarrier numbers of this lane's bins
    const bool v0 = k0 != 0 && k0 >= -26 && k0 <= 26, v1 = k1 != 0 && k1 >= -26 && k1 <= 26;
    // bins 28..35 (SSE vectors 7,8) are forced to zero: their channel coefficient is zero, so is everything multiplied by it
    const cfac eq0 = fac_mul8(ch0), eq1 = fac_mul8(ch1);
    rfac comp0 = fac_rotw(0x7fffu), comp1 = comp0;
    // The tracker's accumulators only ever index the rotation table (mod 2^16) and feed each other by addition, so they wrap mod 2^32
    // instead of being truncated with sx16 at every step: the low 16 bits are the same.
    uint32_t CFO_comp = 0, SFO_comp = 0, CFO_tr = 0, SFO_tr = 0; unsigned symbol_count = 127;
    int plcp_data = 0; uint32_t remain = 0; uint32_t soft_bytes = 0; int nbpsc = 1;
    uint8_t* sout = soft_out + (size_t)f * soft_stride;
    uint32_t status = E_SUCCESS;
    // Where this lane's soft bits go after de-interleaving, as byte offsets into s_soft: at 64-QAM pos[i] is the even position of bit i of
    // d0 (the 16-bit store of the pair); at the other rates the low half of pos[i] is bit i of d0, the high half bit i of d1.
    uint32_t pos[6];
    auto load_positions = [&](int nb) {
        const uint16_t* inv = inv_deint + (nb == 1 ? 0 : nb == 2 ? 48 : nb == 4 ? 144 : 336);
        const uint32_t base = (uint32_t)wib * 288u;
#pragma unroll
        for (int i = 0; i < 6; i++) {
            if (d0 < 0 || i >= nb) pos[i] = 0;
            else if (nb == 6) pos[i] = base + __ldg(inv + d0 * 6 + i);
            else pos[i] = (base + __ldg(inv + d0 * nb + i)) | ((base + __ldg(inv + d1 * nb + i)) << 16);
        }
    };
    load_positions(1);
    uint8_t* const s8 = &s_soft[0][0];
    // everything behind the FFT for one symbol whose spectrum sits in s_fft[wib][h]; returns false when the frame ended
    auto post_fft = [&](int h, uint32_t sym) -> bool {
        const uint32_t* xb = s_fft[wib][h];
        const uint32_t F0 = xb[r0], F1 = xb[r1];
        int e0x, e0y, e1x, e1y, c0x, c0y, c1x, c1y;                                    // products as 32-bit sums, value = sum >> 16
        pk_cmul_xy((int)(short)F0, (int)F0 >> 16, eq0, e0x, e0y);                       // channel_11a.hpp:551-579
        pk_cmul_xy((int)(short)F1, (int)F1 >> 16, eq1, e1x, e1y);
        pk_cmul_xy(e0x >> 16, e0y >> 16, comp0, c0x, c0y);                              // freqoffset.hpp:28-30
        pk_cmul_xy(e1x >> 16, e1y >> 16, comp1, c1x, c1y);
        const int C0re = c0x >> 16, C0im = c0y >> 16, C1re = c1x >> 16, C1im = c1y >> 16;
        // pilot.hpp:168-232: one table walk for the whole warp, the pilots sit in C0 of lanes 24-27 (bins 43, 57, 7, 21; bin 21's is sent negated)
        const bool neg = lane == 27;
        const int th = turn_pi(d_uatan2(T, neg ? -C0im : C0im, neg ? -C0re : C0re), s_pilot[symbol_count]);
        const int th1 = __shfl_sync(FULL, th, 24), th2 = __shfl_sync(FULL, th, 25), th3 = __shfl_sync(FULL, th, 26), th4 = __shfl_sync(FULL, th, 27);
        symbol_count++; if (symbol_count >= 127) symbol_count = 0;
        // the angles are int16, so the sum / 4 lies in [-32768, 32767] and each difference / 28 in [-2340, 2340]: the sx16 of both is the identity
        const int avg = (th1 + th2 + th3 + th4) / 4;
        const int del = ((th3 - th1) / 28 + (th4 - th2) / 28) >> 1;
        CFO_tr += (uint32_t)(avg >> 2); SFO_tr += (uint32_t)(del >> 2);
        CFO_comp += (uint32_t)avg + CFO_tr; SFO_comp += (uint32_t)del + SFO_tr;
        // next symbol's phase compensation; only the rotated bins below use it, every other bin's R is zero whatever its C
        comp0 = fac_rotw(d_rotw(T, (int)(CFO_comp + (uint32_t)k0 * SFO_comp)));
        comp1 = fac_rotw(d_rotw(T, (int)(CFO_comp + (uint32_t)k1 * SFO_comp)));
        // subcarriers -26..-1, 1..26 are rotated, every other bin becomes zero
        const uint32_t R0 = pk_cmul(C0re, C0im, fac_rotw(v0 ? d_rotw(T, avg + k0 * del) : 0u));
        const uint32_t R1 = pk_cmul(C1re, C1im, fac_rotw(v1 ? d_rotw(T, avg + k1 * del) : 0u));
        if (taps.fft_out && sym < taps.max_sym) {
            size_t o = ((size_t)f * taps.max_sym + sym) * 64;
            taps.fft_out[o + b0] = F0; taps.fft_out[o + b1] = F1;
            taps.equalized[o + b0] = __byte_perm((uint32_t)e0x, (uint32_t)e0y, 0x7632); taps.equalized[o + b1] = __byte_perm((uint32_t)e1x, (uint32_t)e1y, 0x7632);
            taps.tracked[o + b0] = R0; taps.tracked[o + b1] = R1;
        }
        // soft demap (demapper.h:141-151 limit + LUTs) scattered through the inverse de-interleaver map
        const int ncbps = 48 * nbpsc;
        if (d0 >= 0) {
            const uint32_t c0 = pk_demap_clamp(R0), c1 = pk_demap_clamp(R1);
            const uint32_t wr0 = s_demap[(c0 >> 4) & 0xFF], wi0 = s_demap[(c0 >> 20) & 0xFF], wr1 = s_demap[(c1 >> 4) & 0xFF], wi1 = s_demap[(c1 >> 20) & 0xFF];
            if (nbpsc == 6) {                          // bits 0-2 are bytes 0, 2, 3 of wr, bits 3-5 those of wi; d0's byte low, d1's high
                auto st16 = [&](uint32_t p, uint32_t v) { *(uint16_t*)(s8 + p) = (uint16_t)v; };
                st16(pos[0], __byte_perm(wr0, wr1, 0x70)); st16(pos[1], __byte_perm(wr0, wr1, 0x42)); st16(pos[2], __byte_perm(wr0, wr1, 0x63));
                st16(pos[3], __byte_perm(wi0, wi1, 0x70)); st16(pos[4], __byte_perm(wi0, wi1, 0x42)); st16(pos[5], __byte_perm(wi0, wi1, 0x63));
            } else {
                auto st8 = [&](uint32_t p, uint32_t v0w, uint32_t v1w) { s8[p & 0xFFFFu] = (uint8_t)v0w; s8[p >> 16] = (uint8_t)v1w; };
                if (nbpsc == 1) { st8(pos[0], wr0, wr1); }
                else if (nbpsc == 2) { st8(pos[0], wr0, wr1); st8(pos[1], wi0, wi1); }
                else { st8(pos[0], wr0, wr1); st8(pos[1], wr0 >> 8, wr1 >> 8); st8(pos[2], wi0, wi1); st8(pos[3], wi0 >> 8, wi1 >> 8); }
            }
        }
        __syncwarp();
        if (!plcp_data) {                              // PHY_11a.hpp:520-604
            uint32_t sig = warp_viterbi_signal(sb, s_dec[wib], lane) & 0xFFFFFFu;
            bool ok = !(sig & 0xFC0010u);
            uint32_t par = (sig >> 16) ^ sig; par ^= par >> 8; par ^= par >> 4; par ^= par >> 2; par ^= par >> 1;
            ok = ok && !(par & 1);
            uint32_t rate = 0; int nd = 0, nb = 1, cr = CR_12;
            switch (sig & 0xF) {                       // ieee80211a_cmn.h:97-157
                case 0xB: rate = 6000; nd = 24; nb = 1; cr = CR_12; break;   case 0xF: rate = 9000; nd = 36; nb = 1; cr = CR_34; break;
                case 0xA: rate = 12000; nd = 48; nb = 2; cr = CR_12; break;  case 0xE: rate = 18000; nd = 72; nb = 2; cr = CR_34; break;
                case 0x9: rate = 24000; nd = 96; nb = 4; cr = CR_12; break;  case 0xD: rate = 36000; nd = 144; nb = 4; cr = CR_34; break;
                case 0x8: rate = 48000; nd = 192; nb = 6; cr = CR_23; break; case 0xC: rate = 54000; nd = 216; nb = 6; cr = CR_34; break;
                default: if (ok) fi.rate_kbps = 0; ok = false;    // BB11aParseDataRate() == 0 is stored before the parser gives up
            }
            uint32_t L = (sig >> 5) & 0xFFF;
            if (ok && rate) { fi.rate_kbps = rate; fi.code_rate = cr; }
            if (ok) { fi.length = L; ok = L <= 2500; }
            if (!ok) { status = E_PLCP_HEADER_FAIL; return false; }
            fi.nsym_total = (L * 8 + 16 + 6 + nd - 1) / nd + 1;
            remain = fi.nsym_total; plcp_data = 1; nbpsc = nb; fi.ncbps = 48 * nb;
            load_positions(nb);
        } else {                                       // N_CBPS = 48 N_BPSC bytes: 3 N_BPSC 16-byte lines (soft_out and soft_stride are 16-byte aligned)
            if (lane < 3 * nbpsc) ((uint4*)(sout + soft_bytes))[lane] = ((const uint4*)sb)[lane];
            soft_bytes += ncbps;
        }
        __syncwarp();
        remain--;
        return remain != 0;
    };
    auto sym_ready = [&](uint32_t sym) { return (s0 + 144u + 80u * sym + 80u) / 4u <= nvec; };   // all 80 samples arrived
    // SIGNAL symbol alone, then the data symbols two at a time
    bool more = true;
    if (!sym_ready(0)) { status = E_NO_FRAME; more = false; }
    if (more) {
        uint32_t v[4]; load4(s0 + 144u + 8u, v); fft_from_regs(v[0], v[1], v[2], v[3]);
        more = post_fft(0, 0);
    }
    if (taps.hdr_only && more) {                                          // continuous-capture scout pass: where the frame ends is all the caller wants
        if (!sym_ready(fi.nsym_total - 1u)) status = E_NO_FRAME;
        more = false;
    }
    // ---- staging of the DATA symbols (see STAGE above) ----
    const uint32_t nsamp20 = nvec * 4u;                                   // 20 Msps samples of the slot that may be read
    uint32_t raw[4] = {0, 0, 0, 0}; uint32_t raw_first = 0xFFFFFFFFu;     // STAGE 1: samples first + hl + 16 j of the prefetched symbol
    auto prefetch_regs = [&](uint32_t first) {                            // whole symbol inside the slot, else nothing
        raw_first = 0xFFFFFFFFu;
        if (first + 72u <= nsamp20) {
#pragma unroll
            for (int j = 0; j < 4; j++) raw[j] = __ldg(x + ((first + hl + 16u * j) << sh));
            raw_first = first;
        }
    };
    uint32_t st_par[2] = {0, 0}; uint32_t st_base[2] = {0, 0}, st_cnt[2] = {0, 0}; uint32_t st_i = 0;   // STAGE 2: parity / first 20 Msps sample / samples per buffer
    auto stage_issue = [&](int b, uint32_t first20, uint32_t n20) {       // samples [first20, first20 + n20) of the slot -> buffer b (word index << sh)
        st_base[b] = first20; st_cnt[b] = 0;
        if (first20 >= nsamp20) return;
        if (first20 + n20 > nsamp20) n20 = nsamp20 - first20;
        st_cnt[b] = n20;
        if (lane == 0) {
            const uint32_t* src = x + (first20 << sh);
            const uintptr_t a0 = (uintptr_t)src & ~(uintptr_t)15, a1 = ((uintptr_t)(src + (n20 << sh)) + 15) & ~(uintptr_t)15;
            const uint32_t bytes = (uint32_t)(a1 - a0);
            const uint32_t mb = (uint32_t)__cvta_generic_to_shared(&s_mbar[wib][b]), dst = (uint32_t)__cvta_generic_to_shared(&s_stage[wib][b][0]);
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(mb), "r"(bytes) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" :: "r"(dst), "l"(a0), "r"(bytes), "r"(mb) : "memory");
        }
    };
    auto stage_wait = [&](int b) {
        if (st_cnt[b] == 0) return;
        const uint32_t mb = (uint32_t)__cvta_generic_to_shared(&s_mbar[wib][b]); uint32_t ok = 0;
        while (!ok) asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(ok) : "r"(mb), "r"(st_par[b]) : "memory");
        st_par[b] ^= 1u;
    };
    auto stage_load4 = [&](int b, uint32_t first, uint32_t (&v)[4]) {    // (x >> 1) * FreqCoeffs from buffer b; the buffer starts at the 16-byte line of its first sample
        const uint32_t skew = (uint32_t)(((uintptr_t)(x + (st_base[b] << sh)) & 15u) >> 2);
#pragma unroll
        for (int j = 0; j < 4; j++) v[j] = fcomp(s_stage[wib][b][skew + ((first - st_base[b] + hl + 16u * j) << sh)], j);
    };
    if (STAGE == 2 && more) stage_issue(0, s0 + 144u + 80u, 160u);        // symbols 1 and 2
    if (STAGE == 1 && more) prefetch_regs(s0 + 144u + 80u * (1u + (uint32_t)half) + 8u);
    for (uint32_t sym = 1; more; sym += 2) {
        const bool haveA = sym_ready(sym), haveB = remain >= 2 && sym_ready(sym + 1);
        if (!haveA) { status = E_NO_FRAME; break; }
        {   uint32_t v[4];
            const uint32_t mine = (half && haveB) ? sym + 1 : sym;          // without a second symbol both halves transform A
            const uint32_t first = s0 + 144u + 80u * mine + 8u;
            if (STAGE == 2) {
                const int b = (int)(st_i & 1u);
                const bool staged = st_base[b] == s0 + 144u + 80u * sym && st_cnt[b] >= (mine - sym + 1u) * 80u;
                stage_wait(b);
                if (staged) stage_load4(b, first, v); else load4(first, v);
                __syncwarp();                                               // every lane has its samples: the other buffer's previous contents are no longer needed either
                st_i++; stage_issue((int)(st_i & 1u), s0 + 144u + 80u * (sym + 2u), 160u);
            } else if (STAGE == 1) {
                if (raw_first == first) {
#pragma unroll
                    for (int j = 0; j < 4; j++) v[j] = fcomp(raw[j], j);
                } else load4(first, v);
                prefetch_regs(s0 + 144u + 80u * (sym + 2u + (uint32_t)half) + 8u);
            } else load4(first, v);
            fft_from_regs(v[0], v[1], v[2], v[3]); }
        more = post_fft(0, sym);
        if (!more) break;
        if (!haveB) {
            if (remain >= 1 && !sym_ready(sym + 1)) { status = E_NO_FRAME; break; }
            sym -= 1;                                                       // the next pair starts one symbol later than staged: restage
            if (STAGE == 2) { stage_wait((int)(st_i & 1u)); __syncwarp(); stage_issue((int)(st_i & 1u), s0 + 144u + 80u * (sym + 2u), 160u); }
            continue;
        }
        more = post_fft(1, sym + 1);
    }
    if (STAGE == 2) { stage_wait((int)(st_i & 1u)); __syncwarp(); }        // no copy may be in flight when the CTA's shared memory is released
    if (lane == 0) { fi.status = status; fi.soft_bytes = soft_bytes; info[f] = fi; }
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
