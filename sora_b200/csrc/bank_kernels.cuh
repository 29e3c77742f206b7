// sora_b200 — polyphase filter-bank channelizer for COMPLEX16 captures (sm_90a): every channel of a uniform grid of M = 2 .. 64 channels,
// centred at (k + o/2) fs / M, out of one capture in one pass (sb200_channelize_bank); and its transmit counterpart, the filter-bank
// combiner (k_combine_bank below, sb200_combine_bank).  The channelizer's stated arithmetic (include/sora_b200.h) is
// channel k of sb200_channelize with phase_inc = (2k + o) 2^31 / M, with the rotated sample kept exact and one rounding at the end:
//     n_j    = D m + j - c,   (C, S) = NCO[((2k + o) n_j (2048 / M)) mod 4096]
//     y_k[m] = sat16((sum_j taps[j] (x(n_j) e^{-j theta}) + 2^28) >> 29)        int64
// Integer arithmetic is exact, so the polyphase form below gives the same bits.  With n = M a + p, the table index is
// (2k + o) p (2048 / M) + 2048 o a (mod 4096), and NCO[i + 2048] = -NCO[i]; so
//     s_p[m] = sum_{j : n_j = p (mod M)} taps[j] sigma(n_j) x(n_j)    sigma(n) = (-1)^(o floor(n / M)), int32 (sum |taps| <= 65535)
//     y_k[m] = round(sum_p s_p[m] conj(T[(2k + o) p mod 2M])),        T[i] = NCO[i 2048 / M]
// and NCO[i + 1024] = j NCO[i] makes the pair p, p + M/2 one multiply: for k even the DFT input is A_p = s_p + s_{p+M/2} (o = 0) or
// s_p - j s_{p+M/2} (o = 1), for k odd B_p = s_p - s_{p+M/2} or s_p + j s_{p+M/2}, each still within int32 (every tap meets one branch).
// Only these exact +-1 / +-j butterflies are used: a further FFT stage would multiply table entries, which are not table entries.
//
// Mapping of k_channelize_bank<M>: one CTA per tile of 4096 input samples (4096 / D outputs of every channel).  The tile plus a halo of
// c samples (rounded up to 4) on each side is staged by stage_window (fir_kernels.cuh); the taps go to shared memory in their own order,
// negated in int32 for odd l of tap r + M l when o = 1 (sigma's part that changes along a branch).  The tile's outputs then go in chunks of
// CH = 2048 / M, three passes each:
//   - branch sums: thread (r = tid mod M, q = tid / M) sums branch r (taps r + M l) for the outputs q + (256 / M) j, j < 8.  The lanes of a
//     warp read the words D m + r + M l - c: at most 32 consecutive words, no bank conflicts for any D; the tap is one word per lane and l,
//     shared by the eight outputs.  The sum, times sigma of its first sample, is stored as s_p, p = (D m + r - c) mod M;
//   - butterflies: s_p, s_{p+M/2} -> A_p, B_p in place;
//   - DFT: warp -> channel k (uniform: the twiddle is a broadcast), lane -> output; int32 x Q14 products in int64 (IMAD.WIDE), one
//     rounding, 32 consecutive outputs of row k per store.
// Work per input sample: 2 ntaps / D multiply-adds of the branch sums and 2 M^2 / D wide ones of the DFT (4 M^2 / D without the butterflies).
#pragma once
#include "fir_kernels.cuh"

namespace sb {

#define SB_BK_MAXCH 64
#define SB_BK_MAXTAPS 1023
#define SB_BK_MAXHALO 512                  // combine_halo(SB_BK_MAXTAPS, 1)
#define SB_BK_SUMS 2048                    // branch sums per chunk: CH = 2048 / M outputs of every branch
// Window words: the tile, its halos, and M more: the last branch of an output reads up to M - D words past the halo, where its taps are zero.
#define SB_BK_WIN (SB_FIR_TILE + 2 * SB_BK_MAXHALO + SB_BK_MAXCH)
#define SB_BK_TAPS (SB_BK_MAXTAPS + 1)     // taps rounded up to a multiple of M
static_assert(combine_halo(SB_BK_MAXTAPS, 1) == SB_BK_MAXHALO, "the window must hold the largest halo");
static_assert(SB_FIR_TILE % SB_BK_MAXCH == 0 && SB_FIR_TILE % SB_BK_SUMS == 0,
              "every D | M divides the tile, and its 4096 / D outputs are a whole number of chunks of 2048 / M");

__host__ __device__ constexpr int bank_log2(int v) { return v <= 1 ? 0 : 1 + bank_log2(v >> 1); }

__device__ __forceinline__ int sat16_q29(long long acc) {
    const long long v = (acc + (1ll << 28)) >> 29;
    return v > 32767 ? 32767 : (v < -32768 ? -32768 : (int)v);
}

// grid (tiles), SB_FIR_THREADS threads, static shared memory only (at most 42.5 KB: four CTAs per multiprocessor).  taps: the taps in
// their own order (branch_taps with U = 1).  Channel k's row starts at y + k * stride.
template <int M>
__global__ void __launch_bounds__(SB_FIR_THREADS, 4) k_channelize_bank(const uint32_t* __restrict__ x, uint64_t n_in, const uint32_t* __restrict__ nco,
                                                                      uint32_t D, uint32_t odd, BrTaps taps, uint32_t* __restrict__ y, uint64_t stride,
                                                                      uint64_t n_out) {
    constexpr int LM = bank_log2(M);
    constexpr uint32_t CH = SB_BK_SUMS / M, CHP = CH + 1;              // outputs per chunk; rows of s_s CH + 1 apart (fewer conflicting stores)
    constexpr uint32_t Q = SB_FIR_THREADS / M;                          // branch pass: outputs q + Q j, j < J
    constexpr int J = CH / Q;
    constexpr uint32_t KW = M >= 8 ? M / 8 : 1, MB = 8 / KW, WPK = M >= 8 ? 1 : 8 / M;   // DFT pass: channels per warp, 32-output blocks per channel
    constexpr uint32_t MBT = MB > 4 ? 4 : MB;
    static_assert(J == 8 && MB * KW * 32 * 8 == CH * M, "the DFT pass covers every channel and output of a chunk once");
    __shared__ __align__(16) uint32_t s_x[SB_BK_WIN];
    __shared__ int s_t[SB_BK_TAPS];
    __shared__ uint32_t s_tw[2 * M];
    __shared__ int2 s_s[M * CHP];
    __shared__ __align__(8) unsigned long long s_bar;

    const uint32_t tid = threadIdx.x, c = taps.n >> 1, halo = combine_halo(taps.n, 1u);
    const uint64_t t0 = (uint64_t)blockIdx.x * SB_FIR_TILE;             // first input sample of this tile
    const uint32_t bytes = stage_window_issue(x, 0, 1, n_in, (int64_t)t0 - (int64_t)halo, SB_FIR_TILE + 2 * halo, s_x, 0, nullptr, 0, nullptr, &s_bar);
    const uint32_t L = (taps.n + M - 1) >> LM;                           // taps per branch
    for (uint32_t j = tid; j < (L << LM); j += SB_FIR_THREADS) {
        const int t = j < taps.n ? (int)taps.t[j] : 0;
        s_t[j] = (odd & (j >> LM)) ? -t : t;                            // in int32: -(-32768) is exact
    }
    for (uint32_t i = tid; i < 2 * M; i += SB_FIR_THREADS) s_tw[i] = __ldg(nco + i * (2048 / M));
    stage_window_wait(bytes, smem_addr(&s_bar));

    const uint64_t m_t = t0 / D;                                        // first output of the tile
    const uint32_t TM = SB_FIR_TILE / D, r = tid & (M - 1), q = tid >> LM, warp = tid >> 5, lane = tid & 31;
    for (uint32_t mc = 0; mc < TM && m_t + mc < n_out; mc += CH) {
        // branch sums: word D m + r + M l - c of the capture is window word D (mc + m) + r + M l + halo - c
        {
            const uint32_t* xb = s_x + D * (mc + q) + r + halo - c;
            const uint32_t dj = D * Q;
            int ar[J], ai[J];
#pragma unroll
            for (int j = 0; j < J; j++) ar[j] = ai[j] = 0;
            for (uint32_t l = 0; l < L; l++, xb += M) {
                const int t = s_t[r + (l << LM)];
#pragma unroll
                for (int j = 0; j < J; j++) {
                    const cs16 v = unpack(xb[dj * j]);
                    ar[j] += t * v.re; ai[j] += t * v.im;               // |sum| <= 65535 * 32768: no wrap
                }
            }
#pragma unroll
            for (int j = 0; j < J; j++) {
                const uint32_t m = q + Q * j;
                const int64_t n = (int64_t)(D * (m_t + mc + m) + r) - (int64_t)c;     // absolute index of the branch's first tap
                const uint32_t p = (uint32_t)n & (M - 1);
                const bool neg = odd & (uint32_t)(n >> LM);                // sigma: arithmetic shift = floor(n / M)
                s_s[p * CHP + m] = neg ? make_int2(-ar[j], -ai[j]) : make_int2(ar[j], ai[j]);
            }
        }
        __syncthreads();
        // butterflies: A_p to row p, B_p to row p + M/2
        for (uint32_t i = tid; i < (M / 2) * CH; i += SB_FIR_THREADS) {
            const uint32_t p = i / CH, m = i % CH;
            int2* pa = s_s + p * CHP + m; int2* pb = pa + (M / 2) * CHP;
            const int2 a = *pa, b = *pb;
            if (odd) { *pa = make_int2(a.x + b.y, a.y - b.x); *pb = make_int2(a.x - b.y, a.y + b.x); }
            else     { *pa = make_int2(a.x + b.x, a.y + b.y); *pb = make_int2(a.x - b.x, a.y - b.y); }
        }
        __syncthreads();
        // DFT: channel k from row (k & 1) (M / 2) + p, p < M / 2; four 32-output blocks at a time (eight int64 sums per thread)
#pragma unroll 1
        for (uint32_t kk = 0; kk < KW; kk++) {
            const uint32_t k = M >= 8 ? warp + 8 * kk : warp % M, b0 = M >= 8 ? 0u : warp / M;
#pragma unroll 1
            for (uint32_t bh = 0; bh < MB; bh += MBT) {
                const uint32_t o0 = lane + 32 * (b0 + WPK * bh);           // output of the chunk of block 0
                const int2* A = s_s + (k & 1) * (M / 2) * CHP + o0;
                long long yr[MBT], yi[MBT];
#pragma unroll
                for (int b = 0; b < (int)MBT; b++) yr[b] = yi[b] = 0;
                for (uint32_t p = 0; p < M / 2; p++, A += CHP) {
                    const cs16 T = unpack(s_tw[((2 * k + odd) * p) & (2 * M - 1)]);
#pragma unroll
                    for (int b = 0; b < (int)MBT; b++) {
                        const int2 a = A[32 * WPK * b];
                        yr[b] += (long long)a.x * T.re + (long long)a.y * T.im;
                        yi[b] += (long long)a.y * T.re - (long long)a.x * T.im;
                    }
                }
                uint32_t* yk = y + (uint64_t)k * stride + m_t + mc + o0;
#pragma unroll
                for (int b = 0; b < (int)MBT; b++)
                    if (m_t + mc + o0 + 32 * WPK * b < n_out) yk[32 * WPK * b] = pack(mk(sat16_q29(yr[b]), sat16_q29(yi[b])));
            }
        }
        __syncthreads();                                                // s_s is rewritten by the next chunk
    }
}

// ---- k_combine_bank: the transmit counterpart (sb200_combine_bank) --------------------------------------------------------------------
// M rows x_k at the channel rate into one capture y at U times the rate, row k centred at (k + o/2) fs / M.  The stated arithmetic
// (include/sora_b200.h), with T[i] = NCO[i 2048 / M] and sigma(n) = (-1)^(o floor(n / M)):
//     W_p(i) = (sum_k x_k(i) T[(2k + o) p mod 2M] + 2^13) >> 14                   the IDFT, rotating up, one rounding
//     acc(n) = sum_i taps[c + U i - n] W_{n mod M}(i)                               int64
//     y(n)   = sat16(a(n) + ((sigma(n) acc(n) + 2^14) >> 15))                       a(n) = out[n] with accumulate, else 0
// The DFT comes first, then the branch filter: the dual of k_channelize_bank.  T[i + M] = -T[i] and T[i + M/2] = j T[i] (NCO[i + 2048] =
// -NCO[i], NCO[i + 1024] = j NCO[i]) split the IDFT into the even-k and odd-k halves E_p, O_p: W_p = E_p + O_p, W_{p+M/2} = j^o (E_p - O_p),
// exact in int64 before the rounding, half the multiplies of the direct sum.
//
// Mapping of k_combine_bank<M>: one CTA per tile of TI = 1024 / M input times (U TI outputs).  The M rows' samples of the tile plus a halo
// of ceil(c / U) (rounded up to 4) on each side are staged by stage_window (fir_kernels.cuh), the taps go to shared memory in their own
// order, zero-padded to U ceil(ntaps / U).  Then two passes:
//   - IDFT: warp -> phase pair (p, p + M/2), so the twiddle is a broadcast; lane -> input time of the window.  E_p and O_p in int64, the
//     butterfly, one rounding each, W stored as int2 at s_w[i M + p] (time-major);
//   - filter: lane -> consecutive outputs n, each with J outputs 256 apart (same p and branch, so one tap load serves J of them).  Output n
//     reads W_{n mod M}(i_n + l) with tap j_n + U l, l < ceil(ntaps / U), j_n = (c - n) mod U.  The U branches of a warp are U consecutive
//     tap words (the taps' own order interleaves the branches: no bank conflicts), and for M >= 16 the W words of 16 consecutive lanes fall
//     in 16 different bank pairs.  sigma is taken on the int64 sum before its rounding; with accumulate each thread loads its outputs'
//     samples from HBM while the staging copies are in flight.  Stores are coalesced.
// Ranges: |W| <= M 2^15 (|C| + |S|) / 2^14 < 2^22, |acc| <= 2048 / M 2^15 |W| < 2^47: no tap-sum limit is needed.  ceil(ntaps / U) M <= 2048
// bounds the halo by 1024 / M, so a tile's window and its IDFT outputs fit one fixed budget at every M.
// Work per output: 2 ntaps / U multiply-adds of the filter and 2 M^2 / U of the IDFT (4 M^2 / U without the butterflies), the IDFT of the
// halo recomputed by both tiles that meet it (DESIGN.md §8).
#define SB_CBK_SPAN 1024                   // rows x input times of a tile: TI = 1024 / M
#define SB_CBK_WORDS (3 * SB_CBK_SPAN + 4 * SB_BK_MAXCH)   // M win = M (TI + 2 halo + 4) <= 1024 + 2048 + 4 M: staged words, and IDFT outputs
#define SB_CBK_TAPS (SB_BK_MAXTAPS + SB_BK_MAXCH + 1)      // taps zero-padded to U ceil(ntaps / U) <= ntaps + U - 1
#define SB_CBK_SMEM 46080                  // static shared memory budget: four CTAs per multiprocessor (4 x (45 + 1) KB of 228 KB)
static_assert(SB_CBK_WORDS * (4 + 8) + SB_CBK_TAPS * 4 + 2 * SB_BK_MAXCH * 4 + 8 <= SB_CBK_SMEM, "k_combine_bank's shared memory must fit its budget");

// The largest halo sb200_combine_bank accepts at M: the largest odd ntaps <= min(1023, 2048 U / M) for every U | M.
__host__ __device__ constexpr uint32_t combine_bank_halo_max(uint32_t M) {
    uint32_t h = 0;
    for (uint32_t U = 1; U <= M; U *= 2) {
        const uint32_t nt = 2048u * U / M > SB_BK_MAXTAPS ? SB_BK_MAXTAPS : 2048u * U / M - 1u;
        h = combine_halo(nt, U) > h ? combine_halo(nt, U) : h;
    }
    return h;
}

__device__ __forceinline__ int sat16_64(long long v) { return v > 32767 ? 32767 : (v < -32768 ? -32768 : (int)v); }

// The filter pass of k_combine_bank<M>: thread tid -> outputs n0 + tid + 256 j, j < J, of the TO in the tile (J = 1: tid < TO only).
template <int M, int J>
__device__ __forceinline__ void combine_bank_filter(const int2* __restrict__ s_w, const int* __restrict__ s_t, uint32_t U, uint32_t L, uint32_t c,
                                                    uint32_t halo, uint32_t odd, uint64_t n0, uint32_t TO, const int (&ar)[4], const int (&ai)[4],
                                                    uint32_t* __restrict__ y, uint64_t n_out) {
    constexpr int LM = bank_log2(M);
    const uint32_t tid = threadIdx.x;
    if (tid >= TO) return;
    const uint64_t n = n0 + tid;
    const uint32_t p = (uint32_t)n & (M - 1), jn = (c - (uint32_t)n) & (U - 1);          // U | M: n0 + 256 j has the same p and branch
    const int2* w = s_w + (((int)(tid + jn) - (int)c) / (int)U + (int)halo) * M + p;     // exact: n - c + j_n is a multiple of U
    const int* t = s_t + jn;
    const uint32_t dj = (SB_FIR_THREADS / U) * M;                                       // words between outputs j and j + 1
    long long accr[J], acci[J];
#pragma unroll
    for (int j = 0; j < J; j++) accr[j] = acci[j] = 0;
    for (uint32_t l = 0; l < L; l++, w += M, t += U) {
        const int tv = *t;
#pragma unroll
        for (int j = 0; j < J; j++) {
            const int2 v = w[dj * j];
            accr[j] += (long long)tv * v.x; acci[j] += (long long)tv * v.y;
        }
    }
#pragma unroll
    for (int j = 0; j < J; j++) {
        const uint64_t nj = n + SB_FIR_THREADS * j;
        if (nj < n_out) {
            const bool neg = odd & (uint32_t)(nj >> LM);                                  // sigma(n)
            const long long vr = neg ? -accr[j] : accr[j], vi = neg ? -acci[j] : acci[j];
            y[nj] = pack(mk(sat16_64(ar[j] + ((vr + (1 << 14)) >> 15)), sat16_64(ai[j] + ((vi + (1 << 14)) >> 15))));
        }
    }
}

// grid (gx, gy) with tile = x + gx y, SB_FIR_THREADS threads, static shared memory only.  Row k starts at x + k * stride; outputs y[0 .. n_out).
// taps: the taps in their own order (branch_taps with U = 1), ceil(ntaps / U) M <= 2048.
template <int M>
__global__ void __launch_bounds__(SB_FIR_THREADS, 4) k_combine_bank(const uint32_t* __restrict__ x, uint64_t stride, uint64_t n_in, const uint32_t* __restrict__ nco,
                                                                   uint32_t U, uint32_t odd, BrTaps taps, uint32_t* __restrict__ y, uint64_t n_out, uint32_t accumulate) {
    constexpr uint32_t TI = SB_CBK_SPAN / M;                            // input times of a tile
    static_assert(M * (TI + 2 * combine_bank_halo_max(M) + 4) <= SB_CBK_WORDS, "the window of the largest halo must fit SB_CBK_WORDS");
    __shared__ __align__(16) uint32_t s_x[SB_CBK_WORDS];
    __shared__ int2 s_w[SB_CBK_WORDS];
    __shared__ int s_t[SB_CBK_TAPS];
    __shared__ uint32_t s_tw[2 * M];
    __shared__ __align__(8) unsigned long long s_bar;

    const uint64_t i0 = ((uint64_t)blockIdx.y * gridDim.x + blockIdx.x) * TI, n0 = U * i0;   // first input time and output of this tile
    if (n0 >= n_out) return;                                            // the rounded-up grid's last CTAs
    const uint32_t tid = threadIdx.x, c = taps.n >> 1, halo = combine_halo(taps.n, U), win = TI + 2 * halo + 4, TO = U * TI;
    // window row k holds x_k(i0 - halo .. i0 + TI + halo + 4); the last 4 cover the zero taps that pad a branch to L
    const uint32_t bytes = stage_window_issue(x, stride, M, n_in, (int64_t)i0 - (int64_t)halo, win, s_x, win, nullptr, 0, nullptr, &s_bar);
    const uint32_t L = (taps.n + U - 1) / U;                             // taps per branch
    for (uint32_t j = tid; j < U * L; j += SB_FIR_THREADS) s_t[j] = j < taps.n ? (int)taps.t[j] : 0;
    for (uint32_t i = tid; i < 2 * M; i += SB_FIR_THREADS) s_tw[i] = __ldg(nco + i * (2048 / M));
    int ar[4] = {0, 0, 0, 0}, ai[4] = {0, 0, 0, 0};                      // a(n) of outputs n0 + tid + 256 j, loaded while the copies fly
    if (accumulate) {
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint32_t o = tid + SB_FIR_THREADS * j;
            if (o < TO && n0 + o < n_out) { const cs16 a = unpack(y[n0 + o]); ar[j] = a.re; ai[j] = a.im; }
        }
    }
    stage_window_wait(bytes, smem_addr(&s_bar));

    // IDFT: warp -> pair (p, p + M/2) and a block of 32 window times
    const uint32_t warp = tid >> 5, lane = tid & 31, nb = (win + 31) >> 5;
    for (uint32_t u = warp; u < (M / 2) * nb; u += SB_FIR_THREADS / 32) {
        const uint32_t p = u / nb, i = ((u - p * nb) << 5) + lane;
        if (i < win) {
            long long er = 0, ei = 0, orr = 0, oi = 0;
#pragma unroll
            for (int k = 0; k < M; k += 2) {
                const cs16 a = unpack(s_x[k * win + i]), b = unpack(s_x[(k + 1) * win + i]);
                const cs16 ta = unpack(s_tw[((2 * k + odd) * p) & (2 * M - 1)]), tb = unpack(s_tw[((2 * k + 2 + odd) * p) & (2 * M - 1)]);
                er += a.re * ta.re - a.im * ta.im; ei += a.im * ta.re + a.re * ta.im;      // each product exact in int32: |x| (|C| + |S|) < 2^30
                orr += b.re * tb.re - b.im * tb.im; oi += b.im * tb.re + b.re * tb.im;
            }
            const long long sr = er + orr, si = ei + oi, dr = er - orr, di = ei - oi;
            int2* w = s_w + i * M + p;
            w[0] = make_int2((int)((sr + (1 << 13)) >> 14), (int)((si + (1 << 13)) >> 14));
            w[M / 2] = odd ? make_int2((int)((-di + (1 << 13)) >> 14), (int)((dr + (1 << 13)) >> 14))        // j (E - O)
                           : make_int2((int)((dr + (1 << 13)) >> 14), (int)((di + (1 << 13)) >> 14));
        }
    }
    __syncthreads();

    // filter: U = M gives TO = 1024 outputs (four per thread), U = M / 2 512 (two), smaller U at most 256 (one)
    if (TO >= 4 * SB_FIR_THREADS) combine_bank_filter<M, 4>(s_w, s_t, U, L, c, halo, odd, n0, TO, ar, ai, y, n_out);
    else if (TO >= 2 * SB_FIR_THREADS) combine_bank_filter<M, 2>(s_w, s_t, U, L, c, halo, odd, n0, TO, ar, ai, y, n_out);
    else combine_bank_filter<M, 1>(s_w, s_t, U, L, c, halo, odd, n0, TO, ar, ai, y, n_out);
}

} // namespace sb
