// sora_b200 — arbitrary-rate channelizer (sb200_channelize_arbitrary, sm_90a): per channel the NCO shift of sb200_channelize, then a
// 256-phase polyphase interpolator at any rate between x16 interpolation and /4 decimation; and its transmit counterpart, the arbitrary-rate
// combiner (sb200_combine_arbitrary, k_combine_arbitrary below).  EXTENSIONS with no reference counterpart:
// its oracle is the arithmetic stated in include/sora_b200.h, restated in numpy by tests/arbitrary_model.py:
//     t_m = tau0 + m * step (Q32.32 input samples),  t' = t_m + 2^23,  i = t' >> 32,  p = (t' >> 24) & 255,
//     y[m] = sat16((sum_{k < ntaps} H[p][k] * v(i - c + k) + 2^13) >> 14),   c = (ntaps - 1) / 2, v the rotated input (0 outside it).
//
// Mapping of k_channelize_arbitrary: one CTA per (tile of TM = 256 J outputs, group of channels).  The tile's outputs read the input
// words i(m0) - c .. i(m0 + TM - 1) - c + ntaps, at most (TM - 1) step / 2^32 + ntaps + 2 of them; stage_window brings them in (from a
// multiple of 4 below the first) together with the call's table (the NCO, only when a channel of the group rotates, then H) on one
// mbarrier.  Per channel the CTA rotates the window into a second buffer (skipped for the identity channel), then every thread makes the
// outputs m0 + tid + 256 j.  Each output has its own row p of H, so the filter is a per-lane gather: one shared word holds two taps
// (2k in the low half, 2k + 1 in the high half) and meets two input words.  Rows are RS = arb_row_words(ntaps) words apart, RS odd: the
// lanes of a warp sit on different rows, and an odd stride puts rows p and p' on the same bank only when p = p' (mod 32), so a warp whose
// rows differ mod 32 reads every tap pair in one wavefront (with ntaps / 2 = 32 words per row and no padding, every row would start on
// bank 0).  The J outputs of a thread are independent sums, interleaved tap pair by tap pair.
// Work per output: 2 ntaps multiply-adds per component pair (ntaps / 2 shared loads of H, ntaps of input), plus per input sample and
// rotating channel the 4 multiply-adds of the rotation.
#pragma once
#include "fir_kernels.cuh"

namespace sb {

#define SB_ARB_MAXTAPS 64
#define SB_ARB_ROWS 256                    // phases of H: p / 256 of an input sample
#define SB_ARB_J 4                         // outputs per thread and tile: TM = 1024
#define SB_ARB_TM (SB_FIR_THREADS * SB_ARB_J)
#define SB_ARB_MINSTEP (1ull << 28)        // x16 interpolation
#define SB_ARB_MAXSTEP (1ull << 34)        // /4 decimation

// Words per row of H: ceil(ntaps / 2) tap pairs, made odd.
__host__ __device__ constexpr uint32_t arb_row_words(uint32_t ntaps) { return ((ntaps + 1) / 2) | 1u; }
// Window words of a tile of tm outputs: i(m0 + tm - 1) - i(m0) <= floor((tm - 1) step / 2^32) + 1, plus ntaps + 1 words from i - c (the
// last tap pair's high half of an odd ntaps reads one word past the taps), plus up to 3 below for the 16-byte aligned start; rounded up to 4.
__host__ __device__ constexpr uint32_t arb_win(uint64_t step, uint32_t ntaps, uint32_t tm = SB_ARB_TM) {
    return (uint32_t)((((uint64_t)(tm - 1) * step) >> 32) + 1 + ntaps + 1 + 3 + 3) & ~3u;
}
// Dynamic shared memory: the NCO (when a channel rotates), H, the window, the rotated window (when a channel rotates), the mbarrier.
__host__ __device__ constexpr uint32_t arb_smem(uint64_t step, uint32_t ntaps, bool rot) {
    return ((rot ? SB_CH_NCO : 0u) + SB_ARB_ROWS * arb_row_words(ntaps) + (rot ? 2u : 1u) * arb_win(step, ntaps)) * 4u + 16u;
}
#define SB_ARB_SMEM_MAX (arb_smem(SB_ARB_MAXSTEP, SB_ARB_MAXTAPS, true))
static_assert(SB_ARB_SMEM_MAX <= 227 * 1024, "the largest tile must fit one multiprocessor's shared memory");

struct ArbArgs {
    const uint32_t* x; uint64_t n_in;
    const uint32_t* tab;                   // SB_CH_NCO words of NCO, then SB_ARB_ROWS rows of H, rs words apart
    ChChannels ch; uint32_t chan_per_group;
    uint64_t tau0, step; uint32_t ntaps, rs, win, nco_words;   // nco_words: SB_CH_NCO when a channel of the call rotates, else 0
    uint32_t* y; uint64_t stride, n_out;
};

// grid (tiles, channel groups), SB_FIR_THREADS threads, arb_smem(step, ntaps, nco_words != 0) bytes of dynamic shared memory.
__global__ void __launch_bounds__(SB_FIR_THREADS) k_channelize_arbitrary(ArbArgs a) {
    constexpr int J = SB_ARB_J; constexpr uint32_t TM = SB_ARB_TM;
    extern __shared__ __align__(16) uint32_t smem[];
    const uint32_t tid = threadIdx.x, rs = a.rs, win = a.win, c = (a.ntaps - 1) / 2, npair = (a.ntaps + 1) / 2;
    const uint32_t* s_nco = smem; const uint32_t* s_h = smem + a.nco_words;
    uint32_t* s_x = smem + a.nco_words + SB_ARB_ROWS * rs; uint32_t* s_v = s_x + win;
    unsigned long long* s_bar = (unsigned long long*)(s_x + (a.nco_words ? 2u : 1u) * win);
    const uint64_t m0 = (uint64_t)blockIdx.x * TM;
    const uint64_t tb = a.tau0 + m0 * a.step + (1ull << 23);           // t' of the tile's first output (the host keeps t_m below 2^63)
    const int64_t lo = ((int64_t)(tb >> 32) - (int64_t)c) & ~3ll;       // first window word: input i(m0) - c rounded down to 4
    const uint32_t ch0 = blockIdx.y * a.chan_per_group, ch1 = min(ch0 + a.chan_per_group, a.ch.n);
    bool rotate = false;                                                // the NCO is only brought in when a channel of the group needs it
    for (uint32_t k = ch0; k < ch1; k++) rotate |= a.ch.inc[k] != 0u || (a.ch.phase0[k] >> 20) != 0u;
    stage_window(a.x, 0, 1, a.n_in, lo, win, s_x, 0, rotate ? a.tab : a.tab + SB_CH_NCO, SB_ARB_ROWS * rs + (rotate ? SB_CH_NCO : 0u),
                 rotate ? smem : smem + a.nco_words, s_bar);

    // output m0 + tid + 256 j: window word of tap 0 and word of its row of H
    uint32_t off[J], hrow[J];
#pragma unroll
    for (int j = 0; j < J; j++) {
        const uint64_t t = tb + (uint64_t)(tid + SB_FIR_THREADS * j) * a.step;
        off[j] = (uint32_t)((int64_t)(t >> 32) - (int64_t)c - lo);
        hrow[j] = (uint32_t)((t >> 24) & 255u) * rs;
    }
    for (uint32_t k = ch0; k < ch1; k++) {
        const uint32_t inc = a.ch.inc[k];
        const bool ident = inc == 0u && (a.ch.phase0[k] >> 20) == 0u;     // NCO[0] = (2^14, 0): the rotation is the identity
        const uint32_t* src = s_x;
        if (!ident) {                                                   // window word i is input lo + i
            uint32_t phi = a.ch.phase0[k] + ((uint32_t)lo + tid) * inc;
            for (uint32_t i = tid; i < win; i += SB_FIR_THREADS, phi += SB_FIR_THREADS * inc) s_v[i] = nco_rotate(s_x[i], s_nco[phi >> 20]);
            __syncthreads();
            src = s_v;
        }
        int accr[J], acci[J];
#pragma unroll
        for (int j = 0; j < J; j++) accr[j] = acci[j] = 1 << 13;
        for (uint32_t q = 0; q < npair; q++) {                          // taps 2q and 2q + 1 of every output's own row
#pragma unroll
            for (int j = 0; j < J; j++) {
                const cs16 h2 = unpack(s_h[hrow[j] + q]), v0 = unpack(src[off[j] + 2 * q]), v1 = unpack(src[off[j] + 2 * q + 1]);
                accr[j] += h2.re * v0.re + h2.im * v1.re; acci[j] += h2.re * v0.im + h2.im * v1.im;   // the row-sum limit keeps this from wrapping
            }
        }
        uint32_t* yr = a.y + (uint64_t)k * a.stride;
#pragma unroll
        for (int j = 0; j < J; j++) {
            const uint64_t m = m0 + tid + SB_FIR_THREADS * j;
            if (m < a.n_out) yr[m] = pack(mk(sat16(accr[j] >> 14), sat16(acci[j] >> 14)));
        }
        if (!ident) __syncthreads();                                    // s_v is rewritten by the next channel
    }
}

// ---- k_combine_arbitrary: the transmit counterpart (sb200_combine_arbitrary) ----------------------------------------------------------
// K rows x_k at their own rate, each resampled at row times t_n = tau0 + n step (Q32.32) by the same 256-phase interpolator, then moved to
// +f_k by sb200_combine's rotation (the absolute output index's phase), scaled by a Q12 gain and summed into one capture y (include/sora_b200.h
// states the arithmetic):
//     u_k(n) = sat16((sum_{j < ntaps} H[p][j] * x_k(i - c + j) + 2^13) >> 14),  t' = t_n + 2^23, i = t' >> 32, p = (t' >> 24) & 255,
//     y(n)   = sat16(a(n) + sum_k ((rotate_up(u_k(n), NCO[(phase0_k + n inc_k) >> 20]) * gain_k + 2^11) >> 12)),  a = out or 0.
//
// Mapping: one CTA per tile of TM = 256 J consecutive outputs, all K rows summed in the CTA (no channel groups: every output needs every
// row).  The tile's outputs read row words i(n0) - c .. i(n0 + TM - 1) - c + ntaps of every row; stage_window brings in each row's span
// (from a multiple of 4 below the first) and the call's table (the NCO, only when a channel rotates, then H) on one mbarrier, and with
// accumulate the lanes load their own outputs meanwhile (coalesced 4-byte loads).  Every thread makes outputs n0 + tid + 256 j, so the
// stores coalesce without an output tile.  Each output gathers its own row p of H as in k_channelize_arbitrary (rows arb_row_words(ntaps)
// words apart, an odd stride); per channel the FIR, the rotation (skipped for the identity channel) and the Q12 gain, summed in int32 and
// saturated once.  The rotation acts on outputs, not on the window, so there is no second window buffer.
// Work per output: K (2 ntaps multiply-adds per component pair + 4 of the rotation + 2 of the gain).  The host picks the largest J whose
// shared memory fits SB_CBR_SMEM (four CTAs per multiprocessor, k_combine<J, true>'s budget; the NCO and a 64-tap H alone take 50 176 B),
// else J = 1, which fits SB_ARB_CB_SMEM_MAX at every limit.
// Dynamic shared memory of k_combine_arbitrary for K rows and a tile of tm outputs: the NCO (when a channel rotates), H, K windows, the mbarrier.
__host__ __device__ constexpr uint32_t arb_combine_smem(uint32_t K, uint64_t step, uint32_t ntaps, bool rot, uint32_t tm) {
    return ((rot ? SB_CH_NCO : 0u) + SB_ARB_ROWS * arb_row_words(ntaps) + K * arb_win(step, ntaps, tm)) * 4u + 16u;
}
#define SB_ARB_CB_SMEM_MAX (arb_combine_smem(SB_CH_MAXCH, SB_ARB_MAXSTEP, SB_ARB_MAXTAPS, true, SB_FIR_THREADS))   // 120 080 B
static_assert(SB_ARB_CB_SMEM_MAX <= 227 * 1024, "a tile of 256 outputs must fit one multiprocessor's shared memory at every K, step and ntaps");

struct ArbCbArgs {
    const uint32_t* x; uint64_t stride, n_in;   // row k at x + k * stride
    const uint32_t* tab;                   // SB_CH_NCO words of NCO, then SB_ARB_ROWS rows of H, rs words apart
    CbChannels ch;
    uint64_t tau0, step; uint32_t ntaps, rs, win, nco_words;   // nco_words: SB_CH_NCO when a channel of the call rotates, else 0
    uint32_t* y; uint64_t n_out; uint32_t accumulate;
};

// grid tile_grid(ceil(n_out / 256 J)) with tile = x + gx y, SB_FIR_THREADS threads, arb_combine_smem(K, step, ntaps, nco_words != 0, 256 J)
// bytes of dynamic shared memory.
template <int J>
__global__ void __launch_bounds__(SB_FIR_THREADS) k_combine_arbitrary(ArbCbArgs a) {
    constexpr uint32_t TM = SB_FIR_THREADS * J;
    extern __shared__ __align__(16) uint32_t smem[];
    const uint32_t tid = threadIdx.x, K = a.ch.n, rs = a.rs, win = a.win, c = (a.ntaps - 1) / 2, npair = (a.ntaps + 1) / 2;
    const uint64_t n0 = ((uint64_t)blockIdx.y * gridDim.x + blockIdx.x) * TM;   // first output of this tile
    if (n0 >= a.n_out) return;                                          // the rounded-up grid's last CTAs
    const uint32_t* s_nco = smem; const uint32_t* s_h = smem + a.nco_words; uint32_t* s_x = smem + a.nco_words + SB_ARB_ROWS * rs;
    unsigned long long* s_bar = (unsigned long long*)(s_x + K * win);
    const uint64_t tb = a.tau0 + n0 * a.step + (1ull << 23);           // t' of the tile's first output (the host keeps t_n below 2^63)
    const int64_t lo = ((int64_t)(tb >> 32) - (int64_t)c) & ~3ll;       // first window word: row sample i(n0) - c rounded down to 4
    const uint32_t bytes = stage_window_issue(a.x, a.stride, K, a.n_in, lo, win, s_x, win, a.tab + (SB_CH_NCO - a.nco_words),
                                              SB_ARB_ROWS * rs + a.nco_words, smem, s_bar);
    uint32_t acc[J];                                                    // with accumulate, out[n] as it was before the call
#pragma unroll
    for (int j = 0; j < J; j++) {
        const uint64_t n = n0 + tid + SB_FIR_THREADS * j;
        acc[j] = a.accumulate && n < a.n_out ? a.y[n] : 0u;
    }
    stage_window_wait(bytes, smem_addr(s_bar));

    // output n0 + tid + 256 j: window word of tap 0 and word of its row of H
    uint32_t off[J], hrow[J];
#pragma unroll
    for (int j = 0; j < J; j++) {
        const uint64_t t = tb + (uint64_t)(tid + SB_FIR_THREADS * j) * a.step;
        off[j] = (uint32_t)((int64_t)(t >> 32) - (int64_t)c - lo);
        hrow[j] = (uint32_t)((t >> 24) & 255u) * rs;
    }
    int sre[J], sim[J];
#pragma unroll
    for (int j = 0; j < J; j++) { const cs16 v = unpack(acc[j]); sre[j] = v.re; sim[j] = v.im; }
    for (uint32_t k = 0; k < K; k++) {
        const uint32_t* src = s_x + k * win;
        int accr[J], acci[J];
#pragma unroll
        for (int j = 0; j < J; j++) accr[j] = acci[j] = 1 << 13;
        for (uint32_t q = 0; q < npair; q++) {                          // taps 2q and 2q + 1 of every output's own row
#pragma unroll
            for (int j = 0; j < J; j++) {
                const cs16 h2 = unpack(s_h[hrow[j] + q]), v0 = unpack(src[off[j] + 2 * q]), v1 = unpack(src[off[j] + 2 * q + 1]);
                accr[j] += h2.re * v0.re + h2.im * v1.re; acci[j] += h2.re * v0.im + h2.im * v1.im;   // the row-sum limit keeps this from wrapping
            }
        }
        const uint32_t inc = a.ch.inc[k], ph0 = a.ch.phase0[k], g = a.ch.gain[k];
        const bool ident = inc == 0u && (ph0 >> 20) == 0u;             // NCO[0] = (2^14, 0): the rotation is the identity
#pragma unroll
        for (int j = 0; j < J; j++) {
            cs16 v = mk(sat16(accr[j] >> 14), sat16(acci[j] >> 14));
            if (!ident) v = nco_rotate_up(v, s_nco[(ph0 + (uint32_t)(n0 + tid + SB_FIR_THREADS * j) * inc) >> 20]);   // absolute output index mod 2^32
            sre[j] += (v.re * (int)g + (1 << 11)) >> 12; sim[j] += (v.im * (int)g + (1 << 11)) >> 12;
        }
    }
#pragma unroll
    for (int j = 0; j < J; j++) {
        const uint64_t n = n0 + tid + SB_FIR_THREADS * j;
        if (n < a.n_out) a.y[n] = pack(mk(sat16(sre[j]), sat16(sim[j])));
    }
}

} // namespace sb
