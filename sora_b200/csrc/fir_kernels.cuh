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
#pragma once
#include "fixed.cuh"

namespace sb {

#define SB_FIR_TILE 4096                   // input samples per CTA
#define SB_FIR_THREADS 256
#define SB_FIR_MAXTAPS 63                  // sb200_fir_decimate2's limit
#define SB_CH_MAXTAPS 255                  // sb200_channelize's limit
#define SB_CH_MAXHALO 128                  // (SB_CH_MAXTAPS - 1) / 2 rounded up to a 16-byte multiple of samples
#define SB_CH_MAXCH 16
#define SB_CH_MAXDECIM 16
// Words of one window buffer.  The staged window has win = SB_FIR_TILE + 2 halo words; its polyphase copy spans D phases of
// P = ceil(win / D) words, D P <= win + D - 1, so a buffer holds the largest window plus SB_CH_MAXDECIM words.
#define SB_CH_WIN (SB_FIR_TILE + 2 * SB_CH_MAXHALO + SB_CH_MAXDECIM)
#define SB_CH_NCO 4096                     // NCO table entries (phi >> 20)
#define SB_CH_SMEM ((2 * SB_CH_WIN + SB_CH_NCO) * 4 + 16)                  // dynamic shared memory of k_channelize: window, rotated window, table, mbarrier
static_assert(SB_CH_WIN % 4 == 0, "the NCO table behind the two window buffers must stay 16-byte aligned for the bulk copy");
static_assert(SB_CH_WIN >= SB_FIR_TILE + 2 * SB_CH_MAXHALO + SB_CH_MAXDECIM - 1, "the polyphase buffer must hold D * ceil(win / D) words");

struct ChTaps { int16_t t[SB_CH_MAXTAPS + 1]; uint32_t n; };
struct ChChannels { uint32_t inc[SB_CH_MAXCH], phase0[SB_CH_MAXCH]; uint32_t n; };

// k_channelize's staging.  k_fir_decimate2 below keeps a copy of these steps inline with its sizes as constants: keep the two in step.
// Stages input samples [t0 - halo, t0 + tile + halo) of x[0 .. n_in) into s[0 .. tile + 2 halo), zero outside the buffer, with one bulk
// copy (plus the 0..3 trailing samples by hand); when `nco` is not null one more bulk copy brings the SB_CH_NCO-word table to s_nco on the
// same barrier.  halo is a multiple of 4 and t0 of SB_FIR_TILE, so the copy's source and destination are 16-byte aligned.  Every thread
// of the CTA calls it; it returns after a __syncthreads with the window in place.
__device__ __forceinline__ void stage_window(const uint32_t* __restrict__ x, uint64_t n_in, uint64_t t0, uint32_t tile, uint32_t halo,
                                             uint32_t* s, const uint32_t* __restrict__ nco, uint32_t* s_nco, unsigned long long* bar) {
    const uint32_t tid = threadIdx.x, nthr = blockDim.x, win = tile + 2 * halo;
    // samples [lo, hi) of the buffer land in s[lo - (t0 - halo) ...]; everything else of the window is zero
    const uint64_t w0 = t0 >= halo ? t0 - halo : 0ull;
    const uint64_t w1 = t0 + tile + halo < n_in ? t0 + tile + halo : n_in;
    const uint32_t dst0 = (uint32_t)(w0 - (t0 - halo));                // halo at the first tile, else 0 (t0 - halo wraps to w0 there)
    const uint32_t nw = (uint32_t)(w1 - w0);
    const uint32_t bulk = nw & ~3u;                                     // whole 16-byte units by the copy engine, the last 0..3 samples by hand
    // zero the parts of the window the copy will not write (buffer edges); done before the copy is started, different words
    for (uint32_t i = tid; i < win; i += nthr) if (i < dst0 || i >= dst0 + bulk) s[i] = 0;
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"((uint32_t)__cvta_generic_to_shared(bar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t bytes = bulk * 4u + (nco ? SB_CH_NCO * 4u : 0u);
    if (tid == 0 && bytes) {
        const uint32_t mb = (uint32_t)__cvta_generic_to_shared(bar);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(mb), "r"(bytes) : "memory");
        if (bulk) asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                               :: "r"((uint32_t)__cvta_generic_to_shared(s + dst0)), "l"(x + w0), "r"(bulk * 4u), "r"(mb) : "memory");
        if (nco) asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                              :: "r"((uint32_t)__cvta_generic_to_shared(s_nco)), "l"(nco), "r"(SB_CH_NCO * 4u), "r"(mb) : "memory");
    }
    if (tid < (nw & 3u)) s[dst0 + bulk + tid] = __ldg(x + w0 + bulk + tid);
    if (bytes) {
        const uint32_t mb = (uint32_t)__cvta_generic_to_shared(bar); uint32_t ok = 0;
        while (!ok) asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }" : "=r"(ok) : "r"(mb) : "memory");
    }
    __syncthreads();
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
    // A copy of stage_window above (keep the two in step) with its sizes as constants and no NCO table: called through the helper, with
    // a runtime halo and block size, this kernel ran 5 % slower (DESIGN.md §8).
    const uint64_t w0 = t0 >= SB_FIR_HALO ? t0 - SB_FIR_HALO : 0ull;
    const uint64_t w1 = t0 + SB_FIR_TILE + SB_FIR_HALO < n_in ? t0 + SB_FIR_TILE + SB_FIR_HALO : n_in;
    const uint32_t dst0 = (uint32_t)(w0 - (t0 - SB_FIR_HALO));
    const uint32_t nw = (uint32_t)(w1 - w0);
    for (uint32_t i = tid; i < SB_FIR_HALO + SB_FIR_TILE + SB_FIR_HALO + 4; i += SB_FIR_THREADS) if (i < dst0 || i >= dst0 + (nw & ~3u)) s_x[i] = 0;
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"((uint32_t)__cvta_generic_to_shared(&s_bar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t bulk = nw & ~3u;
    if (tid == 0 && bulk) {
        const uint32_t mb = (uint32_t)__cvta_generic_to_shared(&s_bar), dst = (uint32_t)__cvta_generic_to_shared(&s_x[dst0]);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(mb), "r"(bulk * 4u) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" :: "r"(dst), "l"(x + w0), "r"(bulk * 4u), "r"(mb) : "memory");
    }
    if (tid < (nw & 3u)) s_x[dst0 + bulk + tid] = __ldg(x + w0 + bulk + tid);
    if (bulk) {
        const uint32_t mb = (uint32_t)__cvta_generic_to_shared(&s_bar); uint32_t ok = 0;
        while (!ok) asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }" : "=r"(ok) : "r"(mb) : "memory");
    }
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

// grid (tiles, channel groups), SB_FIR_THREADS threads, SB_CH_SMEM bytes of dynamic shared memory.  J = outputs per thread per tile and
// channel, at least ceil(ceil(SB_FIR_TILE / D) / SB_FIR_THREADS).  Channel c's row starts at y + c * stride.
template <int J>
__global__ void __launch_bounds__(SB_FIR_THREADS) k_channelize(const uint32_t* __restrict__ x, uint64_t n_in, const uint32_t* __restrict__ nco, ChChannels ch,
                                                              uint32_t chan_per_group, uint32_t D, ChTaps taps, uint32_t* __restrict__ y, uint64_t stride, uint64_t n_out) {
    extern __shared__ __align__(16) uint32_t smem[];
    uint32_t* s_x = smem; uint32_t* s_v = smem + SB_CH_WIN; uint32_t* s_nco = smem + 2 * SB_CH_WIN;
    unsigned long long* s_bar = (unsigned long long*)(smem + 2 * SB_CH_WIN + SB_CH_NCO);
    const uint32_t tid = threadIdx.x;
    const uint64_t t0 = (uint64_t)blockIdx.x * SB_FIR_TILE;             // first input sample of this tile
    const uint32_t c = taps.n >> 1, halo = (c + 3u) & ~3u, win = SB_FIR_TILE + 2 * halo;
    const uint32_t ch0 = blockIdx.y * chan_per_group, ch1 = min(ch0 + chan_per_group, ch.n);
    bool rotate = false;                                                // the table is only brought in when a channel of the group needs it
    for (uint32_t k = ch0; k < ch1; k++) rotate |= ch.inc[k] != 0u || (ch.phase0[k] >> 20) != 0u;
    stage_window(x, n_in, t0, SB_FIR_TILE, halo, s_x, rotate ? nco : nullptr, s_nco, s_bar);
    // outputs m0 .. m1 of the tile: D m in [t0, t0 + tile); output m reads window words D m - (t0 - halo) - c + k, k = 0 .. ntaps-1
    const uint64_t m0 = (t0 + D - 1) / D, m1e = (t0 + SB_FIR_TILE + D - 1) / D, m1 = m1e < n_out ? m1e : n_out;
    const uint32_t nm = m1 > m0 ? (uint32_t)(m1 - m0) : 0u;
    const uint32_t i0 = (uint32_t)(D * m0 - t0) + halo - c;             // window word of output m0, tap 0
    const uint32_t P = (win + D - 1) / D;                               // words per phase of the polyphase buffer
    uint32_t off[J];                                                    // word of output j within its phase (0 for outputs past the tile: read, never stored)
#pragma unroll
    for (int j = 0; j < J; j++) { const uint32_t q = tid + SB_FIR_THREADS * j; off[j] = q < nm ? q : 0u; }
    for (uint32_t k = ch0; k < ch1; k++) {
        const uint32_t inc = ch.inc[k];
        // window word i = D p + r -> s_v[r P + p]; sample index t0 - halo + i
        uint32_t ph = ch.phase0[k] + (uint32_t)(t0 - halo) * inc;
        const bool ident = inc == 0u && (ch.phase0[k] >> 20) == 0u;     // NCO[0] = (2^14, 0): the rotation is the identity
        for (uint32_t p = tid; p < P; p += SB_FIR_THREADS) {
            uint32_t phi = ph + (uint32_t)(D * p) * inc;
            for (uint32_t r = 0, i = D * p; r < D && i < win; r++, i++, phi += inc) {
                const uint32_t w = s_x[i];
                s_v[r * P + p] = ident ? w : nco_rotate(w, s_nco[phi >> 20]);
            }
        }
        __syncthreads();
        uint32_t accr[J], acci[J];
#pragma unroll
        for (int j = 0; j < J; j++) accr[j] = acci[j] = 1u << 14;
        uint32_t r = i0 % D, base = r * P + i0 / D;                     // phase and word of tap 0 for output m0
        for (uint32_t kk = 0; kk < taps.n; kk++) {                      // one tap at a time over the J outputs: the tap is a uniform constant
            const int t = taps.t[kk];
            if (t != 0) {                                               // half-band filters: every other tap
#pragma unroll
                for (int j = 0; j < J; j++) {
                    const cs16 v = unpack(s_v[base + off[j]]);
                    accr[j] += (uint32_t)(t * v.re); acci[j] += (uint32_t)(t * v.im);   // int32 accumulator, two's-complement wrap
                }
            }
            if (++r == D) { r = 0; base += 1u - (D - 1u) * P; } else base += P;
        }
        uint32_t* yr = y + (uint64_t)k * stride;
#pragma unroll
        for (int j = 0; j < J; j++) {
            const uint32_t q = tid + SB_FIR_THREADS * j;
            if (q < nm) yr[m0 + q] = pack(mk(sat16((int)accr[j] >> 15), sat16((int)acci[j] >> 15)));
        }
        __syncthreads();                                                // s_v is rewritten by the next channel
    }
}

} // namespace sb
