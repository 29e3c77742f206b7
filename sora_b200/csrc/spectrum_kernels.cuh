// sora_b200 — the spectrum and power meters of the reference spectrum analyser (kernel/sdl/inc/sdlmeasure.hpp:9-121), over captures and
// channel rows: k_spectrum<N> (TSpecMeter<N>: FFT<N>, SquaredNorm per bin, bin 0 cleared; with overlap, a Q15 window and group sums) and
// k_power_meter (TPowerMeter<N>).  Arithmetic and limits: include/sora_b200.h, sb200_spectrum and sb200_power_meter.
#pragma once
#include "fixed.cuh"

namespace sb {

#define SB_SP_MINN 4
#define SB_SP_MAXN 32768
#define SB_SP_MAXROWS 64
#define SB_SP_TW (3 * (2 * SB_SP_MAXN - 16) / 4)       // twiddle words of every radix-4 stage size 16 .. 32768 (sp_tw_off(2 SB_SP_MAXN))
#define SB_PM_MAXN 65536

// Twiddles of the radix-4 stage of size L (16 .. 32768) in the table: rows M = 1, 2, 3 of L / 4 words each, packed like cs16, at
// 3 (L - 16) / 4 (the sizes 16, 32, .. L / 2 before it sum to L - 16).  Word j of row M is FFT_GetTwiddleConst<L, M>()[j / 4] lane j % 4,
// (trunc(32767 cos(2 pi j M / L)), trunc(-32767 sin(2 pi j M / L))), built on the host (spectrum.cu).
__host__ __device__ constexpr uint32_t sp_tw_off(uint32_t L) { return 3u * (L - 16u) / 4u; }

// Launch shape of k_spectrum<N>.  A CTA of TB threads holds S = TB / TS frames in shared memory, one per slot of TS threads; a thread does
// K / 4 butterflies of its frame per stage and owns the K = N / TS bins k = t + TS i of its slot's group sums.  K is 16 (N / 4 at N <= 8)
// up to N = 16384, whose slots are whole CTAs of 1024 threads; at N = 32768 (K = 32) the sums would not fit the registers of 1024 threads,
// so they are kept in `out` itself, each word read and written by its one owner (GACC).
template <int N> struct SpShape {
    static constexpr int TS = N / 16 < 1 ? 1 : (N / 16 > 1024 ? 1024 : N / 16);
    static constexpr int TB = TS > 256 ? TS : 256;
    static constexpr int S = TB / TS;
    static constexpr int K = N / TS;
    static constexpr bool GACC = K > 16;
    static constexpr uint32_t SMEM = (uint32_t)S * N * 4u;
    static_assert(K % 4 == 0 && S * TS == TB, "k_spectrum shape");
};

struct SpArgs {
    const uint32_t* x; uint64_t stride;                // rows of packed COMPLEX16, `stride` words apart
    const int16_t* win;                                // Q15 window of N taps, or null
    const uint32_t* tw;                                // twiddle table (sp_tw_off)
    uint64_t hop; uint32_t avg;
    uint64_t ngroups, total;                           // groups per row, nrows * ngroups
    int64_t* out;                                      // [nrows * ngroups, N]
};

// FFTSSEEx<8> (core/inc/fft_r4dif.h:86-130) on the 8 samples of one sub-transform, restated from its lane permutations.  v[0..3] is
// pInput[0], v[4..7] pInput[1]; both are >> 3 first.  d = a - b and s = a + b (saturating).  The odd half: permutate_high<0xb1> and the XOR
// of the high imaginary halves turn lanes 2, 3 of d into t = d * -j (im, ~re); o = (d0 + t2, d1 + t3, ~t2 + d0, ~t3 + d1) (the XOR with
// the high-half mask is a one's-complement negation); each lane times wFFTLUT8 = (W^0, W^1, W^0, W^3) of N = 8 by mul_shift; then the
// pairs (m0 + m1, ~m1 + m0, m2 + m3, ~m3 + m2) into pInput[1].  The even half is FFTSSEEx<4>'s arithmetic (dft4) without its input shift,
// into pInput[0].  Outputs in lane order [X0 X4 X2 X6 | X1 X5 X3 X7], which the bit-reversed read-out puts in order.
__device__ __forceinline__ void dft8(cs16 (&v)[8]) {
    const cs16 W0 = mk(32767, 0), W1 = mk(23169, -23169), W3 = mk(-23169, -23169);
    cs16 d[4], s[4];
#pragma unroll
    for (int i = 0; i < 4; i++) { const cs16 a = sra(v[i], 3), b = sra(v[4 + i], 3); d[i] = subs(a, b); s[i] = adds(a, b); }
    const cs16 t2 = mk(d[2].im, ~d[2].re), t3 = mk(d[3].im, ~d[3].re);
    const cs16 m0 = cmul_tw(adds(d[0], t2), W0), m1 = cmul_tw(adds(d[1], t3), W1);
    const cs16 m2 = cmul_tw(adds(cnot(t2), d[0]), W0), m3 = cmul_tw(adds(cnot(t3), d[1]), W3);
    v[4] = adds(m0, m1); v[5] = adds(cnot(m1), m0); v[6] = adds(m2, m3); v[7] = adds(cnot(m3), m2);
    const cs16 e0 = adds(s[0], s[2]), e1 = adds(s[1], s[3]), e2 = adds(cnot(s[2]), s[0]), e3 = adds(cnot(s[3]), s[1]);
    const cs16 t = mk(e3.im, ~e3.re);
    v[0] = adds(e0, e1); v[1] = adds(cnot(e1), e0); v[2] = adds(e2, t); v[3] = adds(cnot(t), e2);
}

// The radix-4 stages of FFTSSEEx<N> (fft_r4dif.h:49-60) from sub-transform size L down to 16, each FFTSSE<L> (:11-47) on every block of L
// samples: butterfly j of a block takes slots j, j + L/4, j + L/2, j + 3L/4 (r4_butterfly).  Then the base case of the remaining size.
template <int N, int L>
__device__ __forceinline__ void sp_stages(uint32_t* fr, const uint32_t* __restrict__ tw, int t) {
    using Sh = SpShape<N>;
    if constexpr (L >= 16) {
        constexpr int Q = L / 4;
        const uint32_t* w = tw + sp_tw_off(L);
#pragma unroll
        for (int u = 0; u < N / 4 / Sh::TS; u++) {
            const int b = t + Sh::TS * u, j = b % Q, p = (b / Q) * L + j;
            cs16 x0 = unpack(fr[p]), x1 = unpack(fr[p + Q]), x2 = unpack(fr[p + 2 * Q]), x3 = unpack(fr[p + 3 * Q]);
            r4_butterfly(x0, x1, x2, x3, unpack(__ldg(w + j)), unpack(__ldg(w + Q + j)), unpack(__ldg(w + 2 * Q + j)));
            fr[p] = pack(x0); fr[p + Q] = pack(x1); fr[p + 2 * Q] = pack(x2); fr[p + 3 * Q] = pack(x3);
        }
        __syncthreads();
        sp_stages<N, L / 4>(fr, tw, t);
    } else if constexpr (L == 8) {                     // FFTSSEEx<8>
#pragma unroll
        for (int u = 0; u < N / 8 / Sh::TS; u++) {
            uint32_t* g = fr + 8 * (t + Sh::TS * u);
            cs16 v[8];
#pragma unroll
            for (int i = 0; i < 8; i++) v[i] = unpack(g[i]);
            dft8(v);
#pragma unroll
            for (int i = 0; i < 8; i++) g[i] = pack(v[i]);
        }
    } else {                                           // FFTSSEEx<4>
#pragma unroll
        for (int u = 0; u < N / 4 / Sh::TS; u++) {
            uint32_t* g = fr + 4 * (t + Sh::TS * u);
            cs16 v0 = unpack(g[0]), v1 = unpack(g[1]), v2 = unpack(g[2]), v3 = unpack(g[3]);
            dft4(v0, v1, v2, v3);
            g[0] = pack(v0); g[1] = pack(v1); g[2] = pack(v2); g[3] = pack(v3);
        }
    }
}

// Spectrum meter: CTA work unit u holds the groups u S .. u S + S - 1 of all rows (group G = row G / ngroups, group G % ngroups), one per
// slot; units are walked grid-stride.  For each of the avg frames of its group every slot loads its frame (the CTA together, so that
// consecutive threads read consecutive samples), windows it, transforms it in shared memory and adds P[k] = re^2 + im^2 (wrapping int32,
// SquaredNorm) of bin k, read at the bit-reversed position (FFT<N>'s FFTLUTMapTable read-out), to its int64 sums; P[0] = 0.
template <int N>
__global__ void __launch_bounds__(SpShape<N>::TB) k_spectrum(const SpArgs a) {
    using Sh = SpShape<N>;
    extern __shared__ __align__(16) uint32_t sp_smem[];
    __shared__ uint64_t base[Sh::S];                   // per slot: word offset of its group's first frame, or ~0 past the last group
    const int slot = threadIdx.x / Sh::TS, t = threadIdx.x % Sh::TS;
    uint32_t* fr = sp_smem + slot * N;
    constexpr int LOGN = 31 - __builtin_clz(N);
    const uint64_t units = (a.total + Sh::S - 1) / Sh::S;
    for (uint64_t unit = blockIdx.x; unit < units; unit += gridDim.x) {
        const uint64_t G = unit * Sh::S + slot;
        const bool live = G < a.total;
        if (t == 0) base[slot] = live ? (G / a.ngroups) * a.stride + (G % a.ngroups) * a.avg * a.hop : ~0ull;
        int64_t acc[Sh::GACC ? 1 : Sh::K];
#pragma unroll
        for (int i = 0; i < (Sh::GACC ? 1 : Sh::K); i++) acc[i] = 0;
        int64_t* o = a.out + G * N;
        __syncthreads();
        for (uint32_t f = 0; f < a.avg; f++) {
#pragma unroll 4
            for (int e = threadIdx.x; e < Sh::S * N; e += Sh::TB) {
                const uint64_t b = base[e / N];
                const int n = e % N;
                uint32_t w = 0;
                if (b != ~0ull) {
                    w = __ldg(a.x + b + f * a.hop + n);
                    if (a.win) {                       // (x w + 2^14) >> 15 per component: w in [0, 32767] keeps it in int16
                        const int q = __ldg(a.win + n);
                        const cs16 c = unpack(w);
                        w = pack(mk((c.re * q + 16384) >> 15, (c.im * q + 16384) >> 15));
                    }
                }
                sp_smem[e] = w;
            }
            __syncthreads();
            sp_stages<N, N>(fr, a.tw, t);
            __syncthreads();
#pragma unroll
            for (int i = 0; i < Sh::K; i++) {
                const int k = t + Sh::TS * i;
                const cs16 c = unpack(fr[__brev((uint32_t)k) >> (32 - LOGN)]);
                const int p = k == 0 ? 0 : wadd(c.re * c.re, c.im * c.im);
                if constexpr (Sh::GACC) { if (live) o[k] = (f ? o[k] : 0) + p; }
                else acc[i] += p;
            }
            __syncthreads();                           // the next frame's load overwrites the slots
        }
        if constexpr (!Sh::GACC) {
            if (live) {
#pragma unroll
                for (int i = 0; i < Sh::K; i++) o[t + Sh::TS * i] = acc[i];
            }
        }
    }
}

// One vector's (or one tail sample's) share of TPowerMeter<N>'s average (sdlmeasure.hpp:30-63): the wrapping int32 sum converted to the
// 64-bit size_t of N (a negative sum divides as 2^64 + v), divided by N and added into the uint sum.
__device__ __forceinline__ uint32_t pm_share(int v, uint32_t N) {
    return v >= 0 ? (uint32_t)v / N : (uint32_t)((uint64_t)(int64_t)v / N);
}
// SquaredNorm of 4 consecutive samples with hadd's wrapping sum (per vector), or of one (the tail), as int
__device__ __forceinline__ int pm_norm(uint32_t w) { const cs16 c = unpack(w); return wadd(c.re * c.re, c.im * c.im); }
__device__ __forceinline__ uint32_t pm_block_part(const uint32_t* __restrict__ p, uint32_t N, uint32_t v0, uint32_t dv) {
    uint32_t s = 0;
    const uint32_t vlen = N / 4;
    for (uint32_t i = v0; i < vlen; i += dv) {
        const uint32_t* q = p + 4 * i;
        s += pm_share(wadd(wadd(pm_norm(__ldg(q)), pm_norm(__ldg(q + 1))), wadd(pm_norm(__ldg(q + 2)), pm_norm(__ldg(q + 3)))), N);
    }
    for (uint32_t i = 4 * vlen + v0; i < N; i += dv) s += pm_share(pm_norm(__ldg(p + i)), N);
    return s;
}

// Power meter: block b of row r (samples [b N, b N + N)) into out[r nblocks + b].  N < 128: one thread per block; larger N: one warp per
// block, the lanes taking every 32nd vector (and tail sample) and summing their uint shares with a shuffle reduction (the uint sum wraps,
// so its order does not matter).  Launched with 256 threads per CTA, grid-stride over the blocks.
__global__ void __launch_bounds__(256) k_power_meter(const uint32_t* __restrict__ x, uint64_t stride, uint64_t nblocks, uint64_t total, uint32_t N,
                                                     uint32_t* __restrict__ out) {
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (uint64_t)gridDim.x * blockDim.x;
    if (N < 128) {
        for (uint64_t g = tid; g < total; g += nth)
            out[g] = pm_block_part(x + (g / nblocks) * stride + (g % nblocks) * N, N, 0, 1);
        return;
    }
    const int lane = threadIdx.x & 31;
    for (uint64_t g = tid / 32; g < total; g += nth / 32) {
        uint32_t s = pm_block_part(x + (g / nblocks) * stride + (g % nblocks) * N, N, lane, 32);
#pragma unroll
        for (int m = 16; m; m >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, m);
        if (lane == 0) out[g] = s;
    }
}

} // namespace sb
