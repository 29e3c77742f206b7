// sora_b200 — anti-alias FIR decimator 2:1 for COMPLEX16 captures (sm_90a).
//
// BASELINE.json's north_star lists "FIR decimation / channel-select" as the first stage of the chain.  The reference's 802.11a graph has no
// filter there: TDownSample2 (Brick11/src/samples.hpp:27-49) just keeps every other sample, which aliases whatever sits between 10 and
// 20 MHz off the carrier into the channel.  This kernel is the filtering alternative, an EXTENSION with no reference counterpart (its oracle
// is the arithmetic stated here, tests/test_gpu_fir.py restates it in numpy):
//     y[m] = sat16( ( sum_k taps[k] * x[2 m + k - (ntaps-1)/2] + 2^14 ) >> 15 ),   x = 0 outside the buffer, re and im independently,
// taps in Q15 (int16), ntaps odd <= 63.  Its output is a 20 Msps stream that sb200_rx11a_batch_ex(sample_rate_mhz = 20) decodes.
//
// It is the one stage of the path that streams: 4 B read per input sample, 4 B written per two.  Mapping: one CTA per tile of 4096 input
// samples; one elected thread starts a 1-D bulk asynchronous copy (cp.async.bulk, the TMA unit: SASS UBLKCP) of the tile plus halo into shared
// memory and all threads wait on its mbarrier; every thread then produces 8 outputs of the tile, one tap at a time (zero taps of a half-band
// filter are skipped).  HBM roofline: 6 B per input sample.
#pragma once
#include "fixed.cuh"

namespace sb {

#define SB_FIR_TILE 4096                   // input samples per CTA
#define SB_FIR_THREADS 256                 // 8 outputs per thread
#define SB_FIR_MAXTAPS 63
#define SB_FIR_HALO 32                     // (MAXTAPS - 1) / 2 rounded up to a 16-byte multiple of samples

struct FirTaps { int16_t t[SB_FIR_MAXTAPS + 1]; uint32_t n; };

__global__ void __launch_bounds__(SB_FIR_THREADS) k_fir_decimate2(const uint32_t* __restrict__ x, uint64_t n_in, FirTaps taps, uint32_t* __restrict__ y, uint64_t n_out) {
    __shared__ __align__(16) uint32_t s_x[SB_FIR_HALO + SB_FIR_TILE + SB_FIR_HALO + 4];
    __shared__ __align__(8) unsigned long long s_bar;
    const uint64_t t0 = (uint64_t)blockIdx.x * SB_FIR_TILE;             // first input sample of this tile
    const uint32_t tid = threadIdx.x;
    // samples [lo, hi) of the buffer land in s_x[lo - (t0 - HALO) ...]; everything else of the window is zero
    const uint64_t w0 = t0 >= SB_FIR_HALO ? t0 - SB_FIR_HALO : 0ull;
    const uint64_t w1 = t0 + SB_FIR_TILE + SB_FIR_HALO < n_in ? t0 + SB_FIR_TILE + SB_FIR_HALO : n_in;
    const uint32_t dst0 = (uint32_t)(w0 - (t0 - SB_FIR_HALO));         // SB_FIR_HALO at the first tile, else 0 (t0 - HALO wraps to w0 there)
    const uint32_t nw = (uint32_t)(w1 - w0);
    // zero the parts of the window the copy will not write (buffer edges); done before the copy is started, different words
    for (uint32_t i = tid; i < SB_FIR_HALO + SB_FIR_TILE + SB_FIR_HALO + 4; i += SB_FIR_THREADS) if (i < dst0 || i >= dst0 + (nw & ~3u)) s_x[i] = 0;
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"((uint32_t)__cvta_generic_to_shared(&s_bar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t bulk = nw & ~3u;                                     // whole 16-byte units by the copy engine, the last 0..3 samples by hand
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

} // namespace sb
