// sora_b200 — radio channel simulator (sb200_channel_sim, sm_90a): per link a sampling-clock offset, multipath, a carrier offset and seeded
// Gaussian noise between T transmit rows and R receive rows of COMPLEX16.  An EXTENSION with no reference counterpart: its oracle is the
// arithmetic stated in include/sora_b200.h, restated in numpy by tests/sim_model.py.
//
// Mapping of k_channel_sim<J>: one CTA per (tile of TM = 256 J outputs, link).  Output m of the tile needs s_t(m - j) for j < L, so the CTA
// interpolates the TM + L - 1 samples s_t(m0 - L + 1 .. m0 + TM) of every input row, and those read the input samples from
// i(m0 - L + 1) - 3 to i(m0 + TM - 1) + 4: at most SIM_WIN(TM) of them whatever the clock step (|step - 2^32| <= 2^24).  stage_window brings
// the T windows and the 28 KB table (NCO | H | LNT) in with bulk copies on one mbarrier; the link's taps come in with plain loads.
//   1. interpolation: thread -> samples q = tid + 256 k of the s buffers, one 8-tap row of H (one 16-byte load) over the T windows;
//   2. per output row r: thread -> outputs m0 + tid + 256 j; the T L complex taps one at a time (a uniform shared word) over the J outputs;
//   3. the carrier rotation (skipped when it is the identity), then the noise: one Philox4x32-10 block gives two outputs, so in every pair of
//      output groups (j, j + 1) lane L computes the block of the pair L of group j (lanes 0..15) or L - 16 of group j + 1 (lanes 16..31)
//      and four shuffles hand every lane its words; every lane is active there (no exits before the last store);
//   4. coalesced 4-byte stores of row r.
#pragma once
#include "../../include/sora_b200.h"      // sb200_link
#include "fir_kernels.cuh"

namespace sb {

#define SB_SIM_MAXROWS 4
#define SB_SIM_MAXTAPS 64
#define SB_SIM_H 1024                      // words of H: 256 rows of 8 int16 taps
#define SB_SIM_LNT 2048                    // words of LNT
#define SB_SIM_TAB (SB_CH_NCO + SB_SIM_H + SB_SIM_LNT)      // the table behind the windows: NCO | H | LNT

// Input samples one tile can read: (TM + 63) outputs span at most (TM + 63)(1 + 2^-8) + 1 inputs, plus the 7 taps around them and the
// rounding of the window start down to a multiple of 4.
__host__ __device__ constexpr uint32_t sim_win(uint32_t tm) { return (tm + 64u + (tm + 64u) / 256u + 16u + 3u) & ~3u; }
__host__ __device__ constexpr uint32_t sim_sbuf(uint32_t tm) { return tm + SB_SIM_MAXTAPS; }
// dynamic shared memory of k_channel_sim<J>: table, T windows, T interpolated rows, the link's R T L taps (rounded to 4 words), mbarrier
__host__ __device__ constexpr uint32_t sim_smem(uint32_t T, uint32_t R, uint32_t L, uint32_t tm) {
    return (SB_SIM_TAB + T * sim_win(tm) + T * sim_sbuf(tm) + ((R * T * L + 3u) & ~3u)) * 4u + 16u;
}

struct SimArgs {
    const uint32_t* x; uint64_t in_link, in_row, n_in; uint32_t T;
    const sb200_link* links; const uint32_t* taps; uint32_t L; uint32_t nlinks;
    uint64_t seed;
    uint32_t* y; uint64_t out_link, out_row, n_out; uint32_t R;
    uint32_t ntiles;
    const uint32_t* tab;                   // SB_SIM_TAB words: NCO (packed cs16), H (packed int16 pairs), LNT (uint32)
};

// Random123's Philox4x32 with 10 rounds
__host__ __device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int i = 0; i < 10; i++) {
        const uint32_t lo0 = 0xD2511F53u * c.x, lo1 = 0xCD9E8D57u * c.z;
#ifdef __CUDA_ARCH__
        const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), hi1 = __umulhi(0xCD9E8D57u, c.z);
#else
        const uint32_t hi0 = (uint32_t)((0xD2511F53ull * c.x) >> 32), hi1 = (uint32_t)((0xCD9E8D57ull * c.z) >> 32);
#endif
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return c;
}

// The Gaussian pair of stage 4 from (wa, wb): (sigma Rn Cn, sigma Rn Sn) rounded >> 34
__device__ __forceinline__ void sim_noise(uint32_t wa, uint32_t wb, uint32_t sigma, const uint32_t* s_nco, const uint32_t* s_lnt, int& nre, int& nim) {
    const uint32_t a = wa | 1u; const int e = __clz(a);
    const uint32_t mant = (a << e) >> 20;                                           // 2048 .. 4095
    const uint32_t v = 2u * (11629080u * (uint32_t)e + s_lnt[mant - 2048u]);       // 2 Lq < 2^30
    uint32_t rn = (uint32_t)__fsqrt_rn(__uint2float_rn(v));                         // within one of floor(sqrt(v)): corrected to it exactly
    if (rn * rn > v) rn--; else if ((rn + 1u) * (rn + 1u) <= v) rn++;
    const cs16 cs = unpack(s_nco[wb >> 20]);
    const long long q = (long long)((unsigned long long)sigma * rn);                // < 2^39
    nre = (int)((q * cs.re + (1ll << 33)) >> 34); nim = (int)((q * cs.im + (1ll << 33)) >> 34);
}

// grid ntiles * nlinks CTAs (tile-minor), SB_FIR_THREADS threads, sim_smem(T, R, L, 256 J) bytes of dynamic shared memory.  J even.
template <int J>
__global__ void __launch_bounds__(SB_FIR_THREADS) k_channel_sim(SimArgs a) {
    constexpr uint32_t TM = SB_FIR_THREADS * J, WIN = sim_win(TM), SB = sim_sbuf(TM);
    extern __shared__ __align__(16) uint32_t smem[];
    const uint32_t T = a.T, R = a.R, L = a.L, tid = threadIdx.x, lane = tid & 31u;
    uint32_t* s_tab = smem; const uint32_t* s_nco = smem; const uint32_t* s_h = smem + SB_CH_NCO; const uint32_t* s_lnt = s_h + SB_SIM_H;
    uint32_t* s_x = smem + SB_SIM_TAB; uint32_t* s_s = s_x + T * WIN; uint32_t* s_g = s_s + T * SB;
    unsigned long long* s_bar = (unsigned long long*)(s_g + ((R * T * L + 3u) & ~3u));
    const uint32_t l = blockIdx.x / a.ntiles, tile = blockIdx.x % a.ntiles;
    const sb200_link lk = a.links[l];
    const uint64_t m0 = (uint64_t)tile * TM;
    const int64_t mlo = (int64_t)m0 - (int64_t)(L - 1);                              // first interpolated sample of the tile
    // input index of output m: (tau0 + m step + 2^23) >> 32; the window starts 3 before that of max(mlo, 0), rounded down to 4
    const uint64_t mfirst = mlo > 0 ? (uint64_t)mlo : 0ull;
    const int64_t lo = ((int64_t)((lk.tau0 + mfirst * lk.step + (1ull << 23)) >> 32) - 3) & ~3ll;
    for (uint32_t i = tid; i < R * T * L; i += SB_FIR_THREADS) s_g[i] = __ldg(a.taps + (uint64_t)l * (R * T * L) + i);
    stage_window(a.x + l * a.in_link, a.in_row, T, a.n_in, lo, WIN, s_x, WIN, a.tab, SB_SIM_TAB, s_tab, s_bar);

    // 1. s_t(m) for m = mlo + q, q < TM + L - 1 (0 for m < 0)
    for (uint32_t q = tid; q < TM + L - 1; q += SB_FIR_THREADS) {
        const int64_t m = mlo + (int64_t)q;
        if (m < 0) { for (uint32_t t = 0; t < T; t++) s_s[t * SB + q] = 0; continue; }
        const uint64_t tp = lk.tau0 + (uint64_t)m * lk.step + (1ull << 23);
        const uint32_t p = (uint32_t)(tp >> 24) & 255u, off = (uint32_t)((int64_t)(tp >> 32) - 3 - lo);
        const uint4 hw = *(const uint4*)(s_h + 4 * p);
        const uint32_t hv[4] = {hw.x, hw.y, hw.z, hw.w};
        for (uint32_t t = 0; t < T; t++) {
            const uint32_t* xs = s_x + t * WIN + off;
            int re = 1 << 13, im = 1 << 13;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const cs16 h2 = unpack(hv[k]), v0 = unpack(xs[2 * k]), v1 = unpack(xs[2 * k + 1]);   // taps 2k (low half), 2k + 1 (high half)
                re += h2.re * v0.re + h2.im * v1.re; im += h2.re * v0.im + h2.im * v1.im;
            }
            s_s[t * SB + q] = pack(mk(sat16(re >> 14), sat16(im >> 14)));
        }
    }
    __syncthreads();

    const bool ident = lk.phase_inc == 0u && (lk.phase0 >> 20) == 0u;                // NCO[0] = (2^14, 0): the rotation is the identity
    const uint32_t sigma = lk.noise_q8;
    for (uint32_t r = 0; r < R; r++) {
        // 2. u_r(m0 + tid + 256 j): s buffer word of output m, tap j is (L - 1) + (m - m0) - j
        int accr[J], acci[J];
#pragma unroll
        for (int j = 0; j < J; j++) accr[j] = acci[j] = 1 << 13;
        for (uint32_t t = 0; t < T; t++) {
            const uint32_t* g = s_g + (r * T + t) * L;
            const uint32_t* sp = s_s + t * SB + (L - 1) + tid;
            for (uint32_t jj = 0; jj < L; jj++, sp--) {                              // one tap at a time over the J outputs: a uniform word
                const cs16 gv = unpack(g[jj]);
#pragma unroll
                for (int j = 0; j < J; j++) {
                    const cs16 v = unpack(sp[SB_FIR_THREADS * j]);
                    accr[j] += gv.re * v.re - gv.im * v.im; acci[j] += gv.re * v.im + gv.im * v.re;   // the tap-sum limit keeps this from wrapping
                }
            }
        }
        uint32_t* yr = a.y + l * a.out_link + r * a.out_row;
#pragma unroll
        for (int j = 0; j < J; j += 2) {
            int vr[2], vi[2];
#pragma unroll
            for (int h = 0; h < 2; h++) {
                cs16 v = mk(sat16(accr[j + h] >> 14), sat16(acci[j + h] >> 14));
                if (!ident) {                                                        // 3. the carrier offset
                    const uint32_t m = (uint32_t)m0 + tid + SB_FIR_THREADS * (j + h);    // mod 2^32
                    v = nco_rotate_up(v, s_nco[(lk.phase0 + m * lk.phase_inc) >> 20]);
                }
                vr[h] = v.re; vi[h] = v.im;
            }
            if (sigma) {                                                             // 4. the noise (a uniform branch: every lane takes it)
                // outputs of group j + h of this warp: w0 + 256 h + [0, 32), pairs (w0 + 256 h) / 2 + [0, 16)
                const uint64_t w0 = m0 + SB_FIR_THREADS * j + (tid & ~31u);
                const uint64_t pair = (w0 >> 1) + (lane < 16u ? lane : (SB_FIR_THREADS / 2) + lane - 16u);
                const uint4 w = philox4x32_10(make_uint4((uint32_t)pair, (uint32_t)(pair >> 32), r, l), (uint32_t)a.seed, (uint32_t)(a.seed >> 32));
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int src = (int)(16u * h + (lane >> 1));
                    const uint32_t x0 = __shfl_sync(0xFFFFFFFFu, w.x, src), x1 = __shfl_sync(0xFFFFFFFFu, w.y, src);
                    const uint32_t x2 = __shfl_sync(0xFFFFFFFFu, w.z, src), x3 = __shfl_sync(0xFFFFFFFFu, w.w, src);
                    const bool odd = lane & 1u;                                      // m0 + 256 j + 32 w is even: lane parity is m's
                    int nre, nim;
                    sim_noise(odd ? x2 : x0, odd ? x3 : x1, sigma, s_nco, s_lnt, nre, nim);
                    vr[h] = sat16(vr[h] + nre); vi[h] = sat16(vi[h] + nim);
                }
            }
#pragma unroll
            for (int h = 0; h < 2; h++) {                                            // 5. coalesced stores
                const uint64_t m = m0 + tid + SB_FIR_THREADS * (j + h);
                if (m < a.n_out) yr[m] = pack(mk(vr[h], vi[h]));
            }
        }
    }
}

// Limits of the link records and tap sums that sb200_channel_sim checks on the device when either table is device memory: thread i checks
// link i / R's record (when i % R == 0) and the tap sum of (link i / R, row i % R); res[0] != 0 if any fails.
__global__ void __launch_bounds__(256) k_sim_check(const sb200_link* __restrict__ links, const int16_t* __restrict__ taps, uint32_t nlinks, uint32_t R, uint32_t T,
                                                  uint32_t L, uint32_t* __restrict__ res) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t bad = 0;
    if (i < (uint64_t)nlinks * R) {
        const uint64_t l = i / R;
        if (i % R == 0) {
            const sb200_link k = links[l];
            bad |= k.step < (1ull << 32) - (1ull << 24) || k.step > (1ull << 32) + (1ull << 24) || k.tau0 >= (1ull << 62) || k.noise_q8 >= (1u << 24);
        }
        const int16_t* g = taps + i * T * L * 2;
        uint32_t sum = 0;
        for (uint32_t q = 0; q < 2 * T * L; q++) sum += (uint32_t)abs((int)g[q]);
        bad |= sum > 65535u;
    }
    bad = __reduce_or_sync(0xFFFFFFFFu, bad);
    if ((threadIdx.x & 31) == 0 && bad) atomicOr(res, 1u);
}

} // namespace sb
