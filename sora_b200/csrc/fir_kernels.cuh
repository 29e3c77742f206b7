// sora_b200 — wideband channelizer for COMPLEX16 captures (sm_90a): per channel a stateless NCO shift, a real FIR and a decimation by D.
//
// BASELINE.json's north_star lists "FIR decimation / channel-select" as the first stage of the chain.  The reference's 802.11a graph has no
// filter there: TDownSample2 (Brick11/src/samples.hpp:27-49) just keeps every other sample, which aliases whatever sits between 10 and
// 20 MHz off the carrier into the channel.  This kernel is the filtering alternative and moves channels that do not sit at 0 Hz there first,
// an EXTENSION with no reference counterpart (its oracle is the arithmetic stated in include/sora_b200.h, restated in numpy by
// tests/wideband_inputs.py):
//     phi(n) = phase0 + (uint32)n * phase_inc (mod 2^32),  (C, S) = NCO[phi >> 20]  (Q14),
//     v(n)   = sat16((x(n) * e^{-j theta} + 2^13) >> 14),
//     y[m]   = sat16((sum_k taps[k] * v(D m + k - (ntaps-1)/2) + 2^14) >> 15),   x = 0 outside the buffer, int32 accumulator,
// taps in Q15 (int16), ntaps odd <= 255.  sb200_fir_decimate2 is one channel (0, 0) of it with D = 2: the Q14 rotation by NCO[0] = (2^14, 0)
// is the identity bit for bit, and such a channel skips it; it keeps its own kernel, k_fir_decimate2 below, which is faster for that case.
//
// Mapping of k_channelize: one CTA per tile of 4096 input samples and group of channels.  One elected thread starts a 1-D bulk asynchronous copy
// (cp.async.bulk, the TMA unit: SASS UBLKCP) of the tile plus a halo of (ntaps-1)/2 samples (rounded up to 4) on each side, and one of the
// 16 KB NCO table, into shared memory; all threads wait on the mbarrier.  The input is read from HBM once per channel group, whatever K is.
// Per channel the CTA then rotates the window into a second buffer in polyphase order (sample i of the window at phase i mod D, index
// i / D), so that for one tap the lanes of a warp read consecutive words: no bank conflicts whatever D is.  Every thread then produces J
// outputs of the tile (tid + 256 j), one tap at a time (the tap is a uniform constant; zero taps of a half-band filter are skipped).
// Work per input sample and channel: 4 multiply-adds of the rotation and 2 ntaps / D of the filter; integer issue bounds it, not HBM
// (4 B read + 4 K / D B written per input sample).
//
// sb200_channelize_rational runs the same kernel at a rational rate U / D: the rotated input is zero-stuffed by U before the filter,
//     y[m]   = sat16((sum_k taps[k] * z(D m + k - c) + 2^14) >> 15),   z(i) = v(i / U) if U divides i, else 0.
// Output m = U q + s (phase s) meets only the branch of taps k = r_s + U l, r_s = (c - D s) mod U, on the inputs n = D q + e_s + l,
// e_s = (D s + r_s - c) / U exactly.  Within one phase consecutive q step the input by D, as at U = 1, so the same polyphase buffer serves
// every phase without bank conflicts and the tap stays uniform across the warp; the tile's phases run one after another (or side by side
// on groups of warps when one phase needs fewer warps than the CTA has).  The sb200_channelize case, U = 1, is a compile-time
// specialisation of the same source (RAT = false): one phase, the taps in ChTaps, and the rotation pass by polyphase column.
#pragma once
#include <type_traits>
#include "fixed.cuh"
#include "bulk_copy.cuh"

namespace sb {

#define SB_FIR_TILE 4096                   // input samples per CTA
#define SB_FIR_THREADS 256
#define SB_FIR_MAXTAPS 63                  // sb200_fir_decimate2's limit
#define SB_CH_MAXTAPS 255                  // sb200_channelize's limit
#define SB_CH_MAXHALO 128                  // (SB_CH_MAXTAPS - 1) / 2 rounded up to a 16-byte multiple of samples
#define SB_CH_MAXCH 16
#define SB_CH_MAXDECIM 16                  // sb200_channelize's and sb200_combine's limit
#define SB_CH_MAXINTERP 16                 // sb200_channelize_rational's limits: U <= 16, D <= 64
#define SB_CH_MAXRDECIM 64
#define SB_CBR_MAXTAPS 4095                // sb200_combine_rational's limits: U <= 64, D <= 16, ntaps <= 4095
#define SB_CBR_MAXINTERP 64
// Words of one window buffer.  The staged window has win = SB_FIR_TILE + 2 halo words; its polyphase copy spans D phases of
// P = ceil(win / D) words, D P <= win + D - 1, so a buffer holds the largest window plus SB_CH_MAXRDECIM words.
#define SB_CH_WIN (SB_FIR_TILE + 2 * SB_CH_MAXHALO + SB_CH_MAXRDECIM)
#define SB_CH_NCO 4096                     // NCO table entries (phi >> 20)
#define SB_CH_SMEM ((2 * SB_CH_WIN + SB_CH_NCO) * 4 + 16)                  // dynamic shared memory of k_channelize: window, rotated window, table, mbarrier
static_assert(SB_CH_WIN % 4 == 0, "the NCO table behind the two window buffers must stay 16-byte aligned for the bulk copy");
static_assert(SB_CH_WIN >= SB_FIR_TILE + 2 * SB_CH_MAXHALO + SB_CH_MAXRDECIM - 1, "the polyphase buffer must hold D * ceil(win / D) words");

struct ChTaps { int16_t t[SB_CH_MAXTAPS + 1]; uint32_t n; };
// The taps of the rational-rate kernels (k_channelize<J, true>, k_combine<J, true>) by branch: taps[r + U l] at t[r L + l],
// L = ceil(ntaps / U), U L <= ntaps + U - 1.  8.3 KB of kernel parameters (allowed up to 32 KB since CUDA 12.1 on sm_70 and later), read
// like ChTaps: one uniform constant-bank load per tap.
struct BrTaps { int16_t t[SB_CBR_MAXTAPS + SB_CBR_MAXINTERP + 1]; uint32_t n, u, L; };
static_assert(SB_CH_MAXINTERP * SB_CH_MAXTAPS <= SB_CBR_MAXTAPS + SB_CBR_MAXINTERP, "BrTaps must hold the channelizer's U L taps as well");
struct ChChannels { uint32_t inc[SB_CH_MAXCH], phase0[SB_CH_MAXCH]; uint32_t n; };

// Staging of k_channelize, k_combine and k_channel_sim (sim_kernels.cuh).  Stages input samples [lo, lo + win) of each of `rows` rows
// x + k * xstride (each x[0 .. n_in)) into s + k * sstride, zero outside [0, n_in), with one bulk copy per row (plus the 0..3 trailing
// samples by hand); when `tab` is not null one more bulk copy brings its tab_words words to s_tab on the same barrier.  lo (which may be
// negative), xstride and sstride are multiples of 4 and x and s are 16-byte aligned, so every copy's source and destination are 16-byte
// aligned.  Every thread of the CTA calls both halves: stage_window_issue starts the copies and returns the bytes in flight, which
// stage_window_wait takes with the barrier's address (smem_addr(bar)); it returns after a __syncthreads with the windows in place.
// Between the two a kernel may do other work that does not touch the windows (k_combine loads its output tile there).
__device__ __forceinline__ uint32_t stage_window_issue(const uint32_t* __restrict__ x, uint64_t xstride, uint32_t rows, uint64_t n_in, int64_t lo,
                                                       uint32_t win, uint32_t* s, uint32_t sstride, const uint32_t* __restrict__ tab,
                                                       uint32_t tab_words, uint32_t* s_tab, unsigned long long* bar) {
    const uint32_t tid = threadIdx.x, nthr = blockDim.x;
    // samples [w0, w1) of the buffer land in s[w0 - lo ...]; everything else of the window is zero
    const int64_t hi = lo + (int64_t)win;
    const uint64_t w0 = lo > 0 ? (uint64_t)lo : 0ull;
    const uint64_t w1e = hi > 0 ? ((uint64_t)hi < n_in ? (uint64_t)hi : n_in) : 0ull, w1 = w1e > w0 ? w1e : w0;
    const uint32_t dst0 = (uint32_t)((int64_t)w0 - lo);                // -lo while the window starts before the buffer, else 0
    const uint32_t nw = (uint32_t)(w1 - w0);
    const uint32_t bulk = nw & ~3u;                                     // whole 16-byte units by the copy engine, the last 0..3 samples by hand
    // zero the parts of the windows the copies will not write (buffer edges); done before the copies are started, different words
    for (uint32_t k = 0; k < rows; k++)
        for (uint32_t i = tid; i < win; i += nthr) if (i < dst0 || i >= dst0 + bulk) s[k * sstride + i] = 0;
    if (tid == 0) mbar_init(smem_addr(bar));
    __syncthreads();
    const uint32_t bytes = rows * bulk * 4u + (tab ? tab_words * 4u : 0u);
    if (tid == 0 && bytes) {
        const uint32_t mb = smem_addr(bar);
        mbar_expect_tx(mb, bytes);
        if (bulk) for (uint32_t k = 0; k < rows; k++) bulk_copy_g2s(smem_addr(s + k * sstride + dst0), x + k * xstride + w0, bulk * 4u, mb);
        if (tab) bulk_copy_g2s(smem_addr(s_tab), tab, tab_words * 4u, mb);
    }
    const uint32_t tail = nw & 3u;
    if (tid < rows * tail) { const uint32_t k = tid / tail, q = tid % tail; s[k * sstride + dst0 + bulk + q] = __ldg(x + k * xstride + w0 + bulk + q); }
    return bytes;
}
__device__ __forceinline__ void stage_window_wait(uint32_t bytes, uint32_t mb) {
    if (bytes) mbar_wait(mb, 0);
    __syncthreads();
}
__device__ __forceinline__ void stage_window(const uint32_t* __restrict__ x, uint64_t xstride, uint32_t rows, uint64_t n_in, int64_t lo, uint32_t win,
                                             uint32_t* s, uint32_t sstride, const uint32_t* __restrict__ tab, uint32_t tab_words, uint32_t* s_tab,
                                             unsigned long long* bar) {
    const uint32_t bytes = stage_window_issue(x, xstride, rows, n_in, lo, win, s, sstride, tab, tab_words, s_tab, bar);
    stage_window_wait(bytes, smem_addr(bar));
}

// sb200_fir_decimate2: channel (0, 0), D = 2 of the arithmetic above, ntaps <= 63, on its own kernel.  k_channelize computes the same bits
// but at half the speed here (DESIGN.md §8).  This kernel reaches 37 % of the HBM peak and is limited by how many tile loads are in flight:
// its 17 KB of static shared memory keep many more tiles resident than k_channelize's 51 KB, and it has no polyphase pass.  One CTA per
// tile, every thread 8 outputs of it, one tap at a time.
struct FirTaps { int16_t t[SB_FIR_MAXTAPS + 1]; uint32_t n; };
#define SB_FIR_HALO 32                     // (SB_FIR_MAXTAPS - 1) / 2 rounded up to a 16-byte multiple of samples

__global__ void __launch_bounds__(SB_FIR_THREADS) k_fir_decimate2(const uint32_t* __restrict__ x, uint64_t n_in, FirTaps taps, uint32_t* __restrict__ y, uint64_t n_out) {
    __shared__ __align__(16) uint32_t s_x[SB_FIR_HALO + SB_FIR_TILE + SB_FIR_HALO + 4];
    __shared__ __align__(8) unsigned long long s_bar;
    const uint64_t t0 = (uint64_t)blockIdx.x * SB_FIR_TILE;             // first input sample of this tile
    const uint32_t tid = threadIdx.x;
    // stage_window's steps for one row with its sizes as constants and no NCO table: called through the helper, with a runtime halo and
    // block size, this kernel ran 5 % slower (DESIGN.md §8).
    const uint64_t w0 = t0 >= SB_FIR_HALO ? t0 - SB_FIR_HALO : 0ull;
    const uint64_t w1 = t0 + SB_FIR_TILE + SB_FIR_HALO < n_in ? t0 + SB_FIR_TILE + SB_FIR_HALO : n_in;
    const uint32_t dst0 = (uint32_t)(w0 - (t0 - SB_FIR_HALO));
    const uint32_t nw = (uint32_t)(w1 - w0);
    for (uint32_t i = tid; i < SB_FIR_HALO + SB_FIR_TILE + SB_FIR_HALO + 4; i += SB_FIR_THREADS) if (i < dst0 || i >= dst0 + (nw & ~3u)) s_x[i] = 0;
    if (tid == 0) mbar_init(smem_addr(&s_bar));
    __syncthreads();
    const uint32_t bulk = nw & ~3u;
    if (tid == 0 && bulk) {
        const uint32_t mb = smem_addr(&s_bar);
        mbar_expect_tx(mb, bulk * 4u);
        bulk_copy_g2s(smem_addr(&s_x[dst0]), x + w0, bulk * 4u, mb);
    }
    if (tid < (nw & 3u)) s_x[dst0 + bulk + tid] = __ldg(x + w0 + bulk + tid);
    if (bulk) mbar_wait(smem_addr(&s_bar), 0);
    __syncthreads();
    // thread -> outputs tid + 256 j, j = 0..7 of the tile (lanes two words apart in shared memory: at most a 2-way bank conflict; stores coalesce)
    const int c = (int)(taps.n >> 1);
    int accr[8], acci[8];
#pragma unroll
    for (int j = 0; j < 8; j++) accr[j] = acci[j] = 1 << 14;
    for (int k = -c; k <= c; k++) {                                     // one tap at a time over the eight outputs: the tap is a uniform constant
        const int t = taps.t[k + c];
        if (t == 0) continue;                                           // half-band filters: every other tap
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const cs16 v = unpack(s_x[SB_FIR_HALO + 2 * (int)(tid + SB_FIR_THREADS * j) + k]);
            accr[j] += t * v.re; acci[j] += t * v.im;
        }
    }
    const uint64_t m0 = t0 / 2;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const uint64_t m = m0 + tid + (uint64_t)SB_FIR_THREADS * j;
        if (m < n_out) y[m] = pack(mk(sat16(accr[j] >> 15), sat16(acci[j] >> 15)));
    }
}

// x * e^{-j theta} in Q14 with (C, S) = (cos theta, sin theta) packed as cs16
__device__ __forceinline__ uint32_t nco_rotate(uint32_t w, uint32_t cs) {
    const cs16 v = unpack(w), r = unpack(cs);
    const int re = v.re * r.re + v.im * r.im + (1 << 13), im = v.im * r.re - v.re * r.im + (1 << 13);
    return pack(mk(sat16(re >> 14), sat16(im >> 14)));
}

// Halo (samples each side) of a tile for ntaps taps at interpolation U: ceil(c / U) rounded up to a 16-byte multiple of samples, at most
// SB_CH_MAXHALO while ceil(ntaps / U) <= 255.  k_channelize's tile reads input D m / U - c / U .. D m / U + c / U for its outputs; k_combine
// (below) reads input i + e_r .. for output U i + r.
__host__ __device__ constexpr uint32_t combine_halo(uint32_t ntaps, uint32_t U) { return ((ntaps / 2 + U - 1) / U + 3u) & ~3u; }

// grid (tiles, channel groups), SB_FIR_THREADS threads, SB_CH_SMEM bytes of dynamic shared memory.  J = outputs per thread per tile,
// channel and phase, at least ceil(ceil(SB_FIR_TILE / D) / SB_FIR_THREADS).  Channel c's row starts at y + c * stride.  RAT = false:
// U = 1 with ChTaps (sb200_channelize); RAT = true: U = taps.u with the branches of BrTaps.
template <int J, bool RAT>
__global__ void __launch_bounds__(SB_FIR_THREADS) k_channelize(const uint32_t* __restrict__ x, uint64_t n_in, const uint32_t* __restrict__ nco, ChChannels ch,
                                                              uint32_t chan_per_group, uint32_t D, typename std::conditional<RAT, BrTaps, ChTaps>::type taps,
                                                              uint32_t* __restrict__ y, uint64_t stride, uint64_t n_out) {
    extern __shared__ __align__(16) uint32_t smem[];
    uint32_t* s_x = smem; uint32_t* s_v = smem + SB_CH_WIN; uint32_t* s_nco = smem + 2 * SB_CH_WIN;
    unsigned long long* s_bar = (unsigned long long*)(smem + 2 * SB_CH_WIN + SB_CH_NCO);
    const uint32_t tid = threadIdx.x;
    uint32_t U = 1u;
    if constexpr (RAT) U = taps.u;
    const uint64_t t0 = (uint64_t)blockIdx.x * SB_FIR_TILE;             // first input sample of this tile
    const uint32_t c = taps.n >> 1, halo = combine_halo(taps.n, U), win = SB_FIR_TILE + 2 * halo;
    const uint32_t ch0 = blockIdx.y * chan_per_group, ch1 = min(ch0 + chan_per_group, ch.n);
    bool rotate = false;                                                // the table is only brought in when a channel of the group needs it
    for (uint32_t k = ch0; k < ch1; k++) rotate |= ch.inc[k] != 0u || (ch.phase0[k] >> 20) != 0u;
    stage_window(x, 0, 1, n_in, (int64_t)t0 - (int64_t)halo, win, s_x, 0, rotate ? nco : nullptr, SB_CH_NCO, s_nco, s_bar);
    // outputs m0 .. m1 of the tile: D m in [U t0, U (t0 + tile)); output m = U q + s reads window words D q + e_s + l - (t0 - halo)
    const uint64_t m0 = (U * t0 + D - 1) / D, m1e = (U * (t0 + SB_FIR_TILE) + D - 1) / D, m1 = m1e < n_out ? m1e : n_out;
    const uint32_t P = (win + D - 1) / D;                               // words per phase of the polyphase buffer
    // Phases side by side: at J = 1 one phase's outputs (at most ceil(tile / D)) need W warps, and G = 8 / W groups of W warps take the
    // phases g, g + G, ...; warps past the last group idle in the filter.  At U = 1 (and J > 1) one group of all warps.
    const uint32_t W = (RAT && J == 1) ? (((SB_FIR_TILE + D - 1) / D + 31u) >> 5) : SB_FIR_THREADS / 32u;
    const uint32_t G = (SB_FIR_THREADS / 32u) / W, grp = (tid >> 5) / W, lt = tid - grp * W * 32u;
    for (uint32_t k = ch0; k < ch1; k++) {
        const uint32_t inc = ch.inc[k];
        // window word i = D p + r -> s_v[r P + p]; sample index t0 - halo + i
        uint32_t ph = ch.phase0[k] + (uint32_t)(t0 - halo) * inc;
        const bool ident = inc == 0u && (ch.phase0[k] >> 20) == 0u;     // NCO[0] = (2^14, 0): the rotation is the identity
        if constexpr (RAT) {                                            // by window word: P < 256 threads for D > 17
            const uint32_t sa = SB_FIR_THREADS / D, sb = SB_FIR_THREADS % D;
            uint32_t p = tid / D, r = tid % D, phi = ph + tid * inc;
            for (uint32_t i = tid; i < win; i += SB_FIR_THREADS) {
                const uint32_t w = s_x[i];
                s_v[r * P + p] = ident ? w : nco_rotate(w, s_nco[phi >> 20]);
                phi += SB_FIR_THREADS * inc; p += sa; r += sb; if (r >= D) { r -= D; p++; }
            }
        } else {
            for (uint32_t p = tid; p < P; p += SB_FIR_THREADS) {
                uint32_t phi = ph + (uint32_t)(D * p) * inc;
                for (uint32_t r = 0, i = D * p; r < D && i < win; r++, i++, phi += inc) {
                    const uint32_t w = s_x[i];
                    s_v[r * P + p] = ident ? w : nco_rotate(w, s_nco[phi >> 20]);
                }
            }
        }
        __syncthreads();
        uint32_t* yr = y + (uint64_t)k * stride;
        for (uint32_t s = grp; s < U; s += G) {
            // phase s: outputs m = U q + s, q = qa .. qb; branch r_s of the taps (length L), first input e_s past D q
            const uint64_t qa = (m0 + U - 1 - s) / U, qb = (m1 + U - 1 - s) / U;
            const uint32_t nq = qb > qa ? (uint32_t)(qb - qa) : 0u;
            const uint32_t rs = (c % U + U - (D * s) % U) % U, L = rs < taps.n ? (taps.n - 1 - rs) / U + 1 : 0u;
            const int es = ((int)(D * s + rs) - (int)c) / (int)U;      // exact: D s + r_s - c is a multiple of U
            int tb = 0;                                                 // branch r_s in taps.t (int: the unrolled tap loads take immediate offsets)
            if constexpr (RAT) tb = (int)(rs * taps.L);
            const uint32_t i0 = (uint32_t)((int64_t)(D * qa) - (int64_t)t0 + (int64_t)halo + es);   // window word of output qa, tap 0
            uint32_t off[J];                                            // word of output j within its phase (0 for outputs past the tile: read, never stored)
#pragma unroll
            for (int j = 0; j < J; j++) { const uint32_t q = lt + SB_FIR_THREADS * j; off[j] = q < nq ? q : 0u; }
            uint32_t accr[J], acci[J];
#pragma unroll
            for (int j = 0; j < J; j++) accr[j] = acci[j] = 1u << 14;
            uint32_t r = i0 % D, base = r * P + i0 / D;                 // phase and word of tap 0 for output qa
            for (uint32_t l = 0; l < L; l++) {                          // one tap at a time over the J outputs: the tap is a uniform constant
                const int t = taps.t[tb + (int)l];
                if (t != 0) {                                           // half-band filters: every other tap
#pragma unroll
                    for (int j = 0; j < J; j++) {
                        const cs16 v = unpack(s_v[base + off[j]]);
                        accr[j] += (uint32_t)(t * v.re); acci[j] += (uint32_t)(t * v.im);   // int32 accumulator, two's-complement wrap
                    }
                }
                if (++r == D) { r = 0; base += 1u - (D - 1u) * P; } else base += P;
            }
#pragma unroll
            for (int j = 0; j < J; j++) {
                const uint32_t q = lt + SB_FIR_THREADS * j;
                if (q < nq) yr[U * (qa + q) + s] = pack(mk(sat16((int)accr[j] >> 15), sat16((int)acci[j] >> 15)));
            }
        }
        __syncthreads();                                                // s_v is rewritten by the next channel
    }
}

// ---- k_combine: the transmit counterpart (sb200_combine) ------------------------------------------------------------------------------
// K rows x_k at the channel rate, each zero-stuffed by U, filtered by the taps, moved to +f_k by the NCO (the channelizer's table, the
// opposite sign), scaled by a Q12 gain and summed into one capture y at U times the rate (include/sora_b200.h states the arithmetic).
// Output n = U i + r sees only the taps j = j0 + U l, j0 = (c - r) mod U, on the inputs x(i + e_r + l), e_r = (r + j0 - c) / U; so the
// filter runs on the rows as they are, one branch of taps per phase r, with no zero-stuffed buffer.
//
// Mapping: one CTA per tile of TI = 256 J input samples of every row (U TI outputs).  One elected thread starts one bulk copy per row of
// the tile plus a halo of ceil(c / U) samples (rounded up to 4) on each side, and one of the NCO table when a channel rotates, all on one
// mbarrier.  For each phase r a thread takes the J input indices tid + 256 j: for one tap the lanes of a warp read consecutive words (no
// bank conflicts) and the tap is a uniform constant (zero taps skipped).  The K channels of one output are summed in registers; the sums
// go to a shared output tile that is written to HBM with 16-byte stores.  Each input sample is read from HBM once, each output written once.
#define SB_CB_SMEM 51200                   // dynamic shared memory budget of k_combine: four CTAs per multiprocessor

struct CbChannels { uint32_t inc[SB_CH_MAXCH], phase0[SB_CH_MAXCH], gain[SB_CH_MAXCH]; uint32_t n; };

// Dynamic shared memory of k_combine for a tile of ti input samples: K windows (halo combine_halo above), the U ti output tile, the NCO
// table and the mbarrier.
__host__ __device__ constexpr uint32_t combine_smem(uint32_t K, uint32_t U, uint32_t ntaps, uint32_t ti) {
    return (K * (ti + 2 * combine_halo(ntaps, U)) + U * ti + SB_CH_NCO) * 4u + 16u;
}
static_assert(combine_smem(SB_CH_MAXCH, 1, SB_CH_MAXTAPS, SB_FIR_THREADS) <= SB_CB_SMEM && combine_smem(SB_CH_MAXCH, SB_CH_MAXDECIM, SB_CH_MAXTAPS, SB_FIR_THREADS) <= SB_CB_SMEM,
              "a tile of 256 input samples must fit the budget at every K, U and ntaps (the largest need is at U = 1 and at U = 16)");

// u * e^{+j theta} in Q14 with (C, S) = (cos theta, sin theta) packed as cs16: nco_rotate with the opposite sign
__device__ __forceinline__ cs16 nco_rotate_up(cs16 u, uint32_t cs) {
    const cs16 r = unpack(cs);
    return mk(sat16((u.re * r.re - u.im * r.im + (1 << 13)) >> 14), sat16((u.im * r.re + u.re * r.im + (1 << 13)) >> 14));
}

// sb200_combine_rational runs the same kernel at a rational rate U / D (RAT = true): output n = U q + s (phase s) meets only the branch of
// taps j = r_s + U l, r_s = (c - D s) mod U, on the inputs x(D q + e_s + l), e_s = (D s + r_s - c) / U exactly; at D = 1 this is the
// mapping above with q = i.  A tile is TQ = 32 W J consecutive q of every phase (U TQ outputs) and reads the inputs D q0 - halo ..
// D (q0 + TQ) + halo of every row.  The lanes of a warp take consecutive q of one phase, so the tap stays a uniform constant and the lanes
// read words D apart: free of bank conflicts for odd D (even D is accepted with its gcd(D, 32)-way conflicts, DESIGN.md §8).  Groups of W
// warps take the phases g, g + G, ... (G = 8 / W) side by side.  The host picks the largest TQ whose shared memory fits SB_CBR_SMEM
// (four CTAs per multiprocessor), else TQ = 32, which fits SB_CBR_SMEM_MAX (three) at every limit.  With accumulate the output tile is
// first loaded from HBM with 16-byte loads and each sum adds onto it before its single saturation.
#define SB_CBR_SMEM 57344                  // preferred budget: four CTAs per multiprocessor (4 x (56 + 1) KB of 228 KB)
#define SB_CBR_SMEM_MAX 75776              // the budget of TQ = 32: three CTAs per multiprocessor (3 x (74 + 1) KB)
// Dynamic shared memory of k_combine<J, true> for tq outputs per phase: K windows of D tq + 2 halo words, the U tq output tile, the NCO
// table and the mbarrier.
__host__ __device__ constexpr uint32_t combine_smem_r(uint32_t K, uint32_t U, uint32_t D, uint32_t ntaps, uint32_t tq) {
    return (K * (D * tq + 2 * combine_halo(ntaps, U)) + U * tq + SB_CH_NCO) * 4u + 16u;
}
static_assert(combine_smem_r(SB_CH_MAXCH, SB_CBR_MAXINTERP, SB_CH_MAXDECIM, 255 * SB_CBR_MAXINTERP, 32) <= SB_CBR_SMEM_MAX && combine_halo(255 * SB_CBR_MAXINTERP, SB_CBR_MAXINTERP) == SB_CH_MAXHALO,
              "a tile of 32 outputs per phase must fit SB_CBR_SMEM_MAX at every K, U, D and ntaps (halo <= 128 while ceil(ntaps / U) <= 255)");

// grid (tiles, 1) or, RAT, (gx, gy) with tile = x + gx y; SB_FIR_THREADS threads; combine_smem(K, U, ntaps, 256 J) or, RAT,
// combine_smem_r(K, U, D, ntaps, 32 W J) bytes of dynamic shared memory.  Row k starts at x + k * stride; outputs y[0 .. n_out).
// RAT = false: D = W / 8 = 1, ChTaps, n_out = U n_in, no accumulate (sb200_combine); RAT = true: BrTaps (sb200_combine_rational).
template <int J, bool RAT>
__global__ void __launch_bounds__(SB_FIR_THREADS) k_combine(const uint32_t* __restrict__ x, uint64_t stride, uint64_t n_in, const uint32_t* __restrict__ nco,
                                                           CbChannels ch, uint32_t U, uint32_t Dr, uint32_t Wr, typename std::conditional<RAT, BrTaps, ChTaps>::type taps,
                                                           uint32_t* __restrict__ y, uint64_t n_out, uint32_t accumulate) {
    const uint32_t D = RAT ? Dr : 1u, W = RAT ? Wr : SB_FIR_THREADS / 32u;
    const uint32_t TQ = 32u * W * J, G = (SB_FIR_THREADS / 32u) / W;    // outputs per phase of a tile; groups of W warps
    extern __shared__ __align__(16) uint32_t smem[];
    const uint32_t tid = threadIdx.x, K = ch.n, c = taps.n >> 1, halo = combine_halo(taps.n, U), win = D * TQ + 2 * halo;
    uint32_t* s_y = smem + K * win; uint32_t* s_nco = s_y + U * TQ;
    unsigned long long* s_bar = (unsigned long long*)(s_nco + SB_CH_NCO);
    const uint64_t q0 = (RAT ? (uint64_t)blockIdx.y * gridDim.x + blockIdx.x : (uint64_t)blockIdx.x) * TQ;   // first output of every phase of this tile
    const uint64_t n0 = U * q0;                                         // first output of this tile
    if (RAT && n0 >= n_out) return;                                     // the rounded-up grid's last CTAs
    const uint64_t t0 = D * q0;                                         // input D q0 lines up with output U q0
    bool rotate = false;                                                // the table is only brought in when a channel needs it
    for (uint32_t k = 0; k < K; k++) rotate |= ch.inc[k] != 0u || (ch.phase0[k] >> 20) != 0u;

    // window k holds samples [t0 - halo, t0 + D TQ + halo) of row k; halo, D TQ and stride are multiples of 4
    const uint32_t bytes = stage_window_issue(x, stride, K, n_in, (int64_t)t0 - (int64_t)halo, win, smem, win, rotate ? nco : nullptr, SB_CH_NCO, s_nco, s_bar);
    // outputs n0 .. n0 + nt of y[0 .. n_out); with accumulate they are loaded into the output tile first (16-byte loads: n0 is a multiple of 4)
    if (RAT && accumulate) {
        const uint64_t nt = n_out - n0 < (uint64_t)U * TQ ? n_out - n0 : (uint64_t)U * TQ;
        const uint32_t n4 = (uint32_t)nt >> 2;
        const uint4* y4 = (const uint4*)(y + n0); uint4* s4 = (uint4*)s_y;
        for (uint32_t q = tid; q < n4; q += SB_FIR_THREADS) s4[q] = y4[q];
        if (tid < ((uint32_t)nt & 3u)) s_y[4 * n4 + tid] = y[n0 + 4 * n4 + tid];
    }
    stage_window_wait(bytes, smem_addr(s_bar));

    // RAT = false: one group, grp = 0 and lt = tid at compile time, so the phase and its taps stay uniform to the compiler (DESIGN.md §8)
    const uint32_t grp = RAT ? (tid >> 5) / W : 0u, lt = RAT ? tid - grp * W * 32u : tid;
    for (uint32_t s = grp; s < U; s += G) {                             // warps past the last group (8 % W of them) idle
        const uint32_t rs = (c % U + U - (D * s) % U) % U;              // first tap of phase s's branch
        const int e = ((int)(D * s + rs) - (int)c) / (int)U;            // exact: D s + r_s - c is a multiple of U
        const uint32_t* s_r = smem + (int)halo + e + D * lt;            // window word of input D (q0 + lt) + e_s, tap r_s
        int sre[J], sim[J];
#pragma unroll
        for (int j = 0; j < J; j++) sre[j] = sim[j] = 0;
        for (uint32_t k = 0; k < K; k++, s_r += win) {
            uint32_t accr[J], acci[J];
#pragma unroll
            for (int j = 0; j < J; j++) accr[j] = acci[j] = 1u << 14;
            if constexpr (RAT) {
                const uint32_t L = rs < taps.n ? (taps.n - 1 - rs) / U + 1 : 0u;
                const int tb = (int)(rs * taps.L);                      // branch r_s in taps.t (int: the unrolled tap loads take immediate offsets)
                for (uint32_t l = 0; l < L; l++) {                      // one tap at a time over the J outputs: the tap is a uniform constant
                    const int t = taps.t[tb + (int)l];
                    if (t != 0) {
#pragma unroll
                        for (int j = 0; j < J; j++) {
                            const cs16 v = unpack(s_r[l + D * 32u * W * j]);
                            accr[j] += (uint32_t)(t * v.re); acci[j] += (uint32_t)(t * v.im);   // the per-branch tap limit keeps this from wrapping
                        }
                    }
                }
            } else {
                for (uint32_t jj = rs, l = 0; jj < taps.n; jj += U, l++) {  // one tap at a time over the J inputs: the tap is a uniform constant
                    const int t = taps.t[jj];
                    if (t != 0) {
#pragma unroll
                        for (int j = 0; j < J; j++) {
                            const cs16 v = unpack(s_r[l + SB_FIR_THREADS * j]);
                            accr[j] += (uint32_t)(t * v.re); acci[j] += (uint32_t)(t * v.im);   // the per-branch tap limit keeps this from wrapping
                        }
                    }
                }
            }
            const uint32_t inc = ch.inc[k], g = ch.gain[k];
            const bool ident = inc == 0u && (ch.phase0[k] >> 20) == 0u;     // NCO[0] = (2^14, 0): the rotation is the identity
#pragma unroll
            for (int j = 0; j < J; j++) {
                cs16 v = mk(sat16((int)accr[j] >> 15), sat16((int)acci[j] >> 15));
                if (!ident) {
                    const uint32_t n = U * (uint32_t)(q0 + lt + 32u * W * j) + s;   // absolute output index mod 2^32
                    v = nco_rotate_up(v, s_nco[(ch.phase0[k] + n * inc) >> 20]);
                }
                sre[j] += (v.re * (int)g + (1 << 11)) >> 12; sim[j] += (v.im * (int)g + (1 << 11)) >> 12;
            }
        }
#pragma unroll
        for (int j = 0; j < J; j++) {
            uint32_t* o = s_y + (lt + 32u * W * j) * U + s;
            if (RAT && accumulate) { const cs16 a = unpack(*o); sre[j] += a.re; sim[j] += a.im; }
            *o = pack(mk(sat16(sre[j]), sat16(sim[j])));
        }
    }
    __syncthreads();

    // the tile's outputs to HBM: 16-byte stores, the last 0..3 of the capture by hand
    const uint64_t nt = n_out - n0 < (uint64_t)U * TQ ? n_out - n0 : (uint64_t)U * TQ;
    const uint32_t n4 = (uint32_t)nt >> 2;
    uint4* y4 = (uint4*)(y + n0); const uint4* s4 = (const uint4*)s_y;
    for (uint32_t q = tid; q < n4; q += SB_FIR_THREADS) y4[q] = s4[q];
    if (tid < ((uint32_t)nt & 3u)) y[n0 + 4 * n4 + tid] = s_y[4 * n4 + tid];
}

} // namespace sb
