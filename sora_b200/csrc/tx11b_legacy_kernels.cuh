// sora_b200 — the legacy 802.11b transmit filter on the device: BB11BPMDSpreadFIR4SSE / BB11BPMDSpreadFIR4ASM (kernel/inc/bb/bbb.h:188-200,
// kernel/bb/dot11b/bbb_fir.c), the 37-tap pulse shaper BB11BPMDPacketGenSignal (bbb_tx.c:116-150) runs over the 4x zero-stuffed chip stream.
//
// The reference is a transposed-form filter: a group of four inputs adds its products to the partial sums of the 40 outputs it reaches, with
// saturating 16-bit adds, and a finished output is the saturating sum of its four lanes, (l0 + l2) + (l1 + l3), >> 8, packed to int8.  Read the
// other way round, output sample 4p + r of a frame is a fixed function of the ten input groups p-9 .. p (group q = input samples 8 + 4q .. 8 + 4q + 3:
// the routine starts at the second 16-byte block): lane i sums x[8 + 4q + i] * h[r + 4(p - q) - i] over q.  A lane's sum cannot saturate
// (it meets every fourth tap only: at most 195 * 128 = 24 960), so only the three adds of the lane tree need the clamp, and every output is
// independent: one thread per group of four outputs, ten 8-byte loads, ~80 multiply-adds with compile-time coefficients.
// The two bodies of the reference differ in the outer +-1 taps (DESIGN.md, legacy 802.11b transmit filter, has the why):
//   variant 0 (FIR37SSE_INTRINSIC, bbb_fir.c:413-566): in an even group outputs 1..3 take x[8+4p] * 1 as their newest contribution (row 0's
//     coefficients instead of rows 1..3); the oldest contribution of output r = 1 is missing and that of r = 2 is -x[2] of the even group at or
//     before p - 9 (instead of +x[2] of group p - 9);
//   variant 1 (FIR37SSE_INLINE, bbb_fir.c:137-386): the plain filter.
#pragma once
#include "tx11b_kernels.cuh"
#include "tx_frames.cuh"

namespace sb {

__host__ __device__ constexpr int fir37_h(int k) {
    constexpr int H[37] = {1, 0, -1, 0, 1, 0, -1, 0, 2, 0, -3, 0, 5, 0, -11, 0, 54, 128, 163, 128, 54, 0, -11, 0, 5, 0, -3, 0, 2, 0, -1, 0, 1, 0, -1, 0, 1};
    return (k >= 0 && k < 37) ? H[k] : 0;
}
__device__ __forceinline__ int fir37_sat16(int v) { return min(max(v, -32768), 32767); }

#define SB_FIR37_THREADS 128

// grid: x = frame, y = tiles of SB_FIR37_THREADS groups (grid-stride over the frame's groups)
template <int VARIANT>
__global__ void __launch_bounds__(SB_FIR37_THREADS) k_fir37_legacy(const int8_t* __restrict__ in, const uint64_t* __restrict__ off, const uint32_t* __restrict__ len,
                                                                  uint32_t nframes, int8_t* __restrict__ out) {
    const uint32_t f = blockIdx.x;
    if (f >= nframes) return;
    const uint32_t n_in = len[f], ngroups = (n_in >> 3) * 2u;
    const uint2* src = reinterpret_cast<const uint2*>(in + 2ull * off[f]);          // one group of four COMPLEX8 per 8-byte word (off is a multiple of 8 samples)
    uint2* dst = reinterpret_cast<uint2*>(out + 2ull * off[f]);
    const uint32_t nwords = n_in >> 2;                                               // whole groups of the input; samples past n_in read as zero
    for (uint32_t p = blockIdx.y * SB_FIR37_THREADS + threadIdx.x; p < ngroups; p += gridDim.y * SB_FIR37_THREADS) {
        int v[10][4][2];                                                             // v[m] = group p - m
#pragma unroll
        for (int m = 0; m < 10; m++) {
            const int64_t w = (int64_t)p - m + 2;                                    // word index of group q = p - m (sample 8 + 4q)
            uint2 x = make_uint2(0u, 0u);
            if (p >= (uint32_t)m && (uint64_t)w < nwords) x = __ldg(src + w);
            v[m][0][0] = (int8_t)(x.x); v[m][0][1] = (int8_t)(x.x >> 8); v[m][1][0] = (int8_t)(x.x >> 16); v[m][1][1] = (int8_t)(x.x >> 24);
            v[m][2][0] = (int8_t)(x.y); v[m][2][1] = (int8_t)(x.y >> 8); v[m][3][0] = (int8_t)(x.y >> 16); v[m][3][1] = (int8_t)(x.y >> 24);
        }
        int stale2[2] = {0, 0};                                                       // variant 0: x[2] of the even group at or before p - 9
        if (VARIANT == 0) {
            const uint32_t odd = (p + 1u) & 1u;                                       // p - 9 is odd when p is even
            if (!odd) { stale2[0] = v[9][2][0]; stale2[1] = v[9][2][1]; }
            else if (p >= 10u) {
                const int64_t w = (int64_t)p - 10 + 2; uint2 x = make_uint2(0u, 0u);
                if ((uint64_t)w < nwords) x = __ldg(src + w);
                stale2[0] = (int8_t)(x.y); stale2[1] = (int8_t)(x.y >> 8);
            }
        }
        const bool have9 = p >= 9u;                                                   // before that the partial sums are still the zeros they started as
        int y[4][2];
#pragma unroll
        for (int r = 0; r < 4; r++) {
#pragma unroll
            for (int c = 0; c < 2; c++) {
                int l[4];
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    int s = 0;
#pragma unroll
                    for (int m = 1; m < 9; m++) s += v[m][i][c] * fir37_h(r + 4 * m - i);
                    // oldest contribution (rows 36..39 of the table)
                    if (VARIANT == 1 || r == 0 || r == 3) s += v[9][i][c] * fir37_h(r + 36 - i);
                    else if (r == 2 && i == 2) s += have9 ? -stale2[c] : 0;             // row 38 made from the row-36 product of the even group: -x[2]
                    // newest contribution
                    if (VARIANT == 0 && r > 0) s += ((p & 1u) == 0) ? v[0][i][c] * fir37_h(0 - i) : v[0][i][c] * fir37_h(r - i);
                    else s += v[0][i][c] * fir37_h(r - i);
                    l[i] = s;
                }
                const int t = fir37_sat16(fir37_sat16(l[0] + l[2]) + fir37_sat16(l[1] + l[3])) >> 8;
                y[r][c] = min(max(t, -128), 127) & 0xFF;
            }
        }
        dst[p] = make_uint2((uint32_t)y[0][0] | ((uint32_t)y[0][1] << 8) | ((uint32_t)y[1][0] << 16) | ((uint32_t)y[1][1] << 24),
                            (uint32_t)y[2][0] | ((uint32_t)y[2][1] << 8) | ((uint32_t)y[3][0] << 16) | ((uint32_t)y[3][1] << 24));
    }
}

// ---- the legacy 802.11b encoder in front of that filter: BB11BPMDBufferTx4XWith{Long,Short}Header (kernel/bb/dot11b/bbb_tx.c:508-758) -----
// The reference walks look-up tables byte by byte (bbb_scramble.c, bbb_dbpsk.c, bbb_dqpsk.c, bbb_cck5.c, bbb_cck11.c); the scrambler register
// and the differential phase reference are the only serial state.  Split like k_tx11b_code / k_tx11b_shape:
//   k_tx11b_legacy_code    one thread per frame: PLCP frame (CRC-16), scrambler over PLCP + PSDU + FCS, phase reference; one 16-bit
//                          descriptor per byte: [7:0] scrambled byte, [9:8] phase in front of the byte in quarter turns, [10] odd CCK-11 symbol;
//   k_tx11b_legacy_spread  every output sample independently: a CTA stages the chips its 1024 samples depend on in shared memory (a chip is
//                          a closed form of one descriptor and the chip number, the tables' entries), then each thread writes 8 samples
//                          with one 128-bit store: the 4x zero-stuffed encoder output itself, or the 37-tap filter of BB11BPMDPacketGenSignal
//                          applied on the fly.  Fused, the stuffed stream never reaches memory, and only one input in four of the filter
//                          is non-zero: output 4p + r = (sum_{m=0..9} chip[p + 2 - m] * h[r + 4m]) >> 8 (input group p - m holds chip p + 2 - m
//                          in lane 0 and zeros elsewhere, groups before 0 do not exist: chips 0 and 1 never enter).  No lane sum can saturate
//                          (|chip| <= 128, sum |h[r + 4m]| <= 195), so the lane tree of k_fir37_legacy adds nothing.  Variant 0's quirks reduce
//                          to one: in an even group, outputs 1..3 take chip[p + 2] * 1 as their newest term (row 0's coefficient); the stale
//                          row-38 term reads lane 2, always zero here.
struct Tx11bLegacyJob {
    uint32_t rate_kbps, rate_code, short_preamble, fcs_in_payload;
    uint32_t data_chips_per_byte;        // 88 / 44 / 16 / 8; 0 for short preamble at 1 Mbps (the reference's switch has no such case)
    uint32_t filter;                     // 0 encoder output, 1 BB11BPMDSpreadFIR4SSE, 2 BB11BPMDSpreadFIR4ASM
    uint32_t desc_stride;                // descriptors per frame row
};

__global__ void __launch_bounds__(128) k_tx11b_legacy_code(const uint8_t* __restrict__ payload, const uint64_t* __restrict__ pay_off,
        const uint32_t* __restrict__ pay_len, uint32_t nframes, Tx11bLegacyJob job, const uint32_t* __restrict__ crcs, uint16_t* __restrict__ desc) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nframes) return;
    const uint8_t* p = payload + pay_off[f];
    const uint32_t len = job.fcs_in_payload ? pay_len[f] - 4u : pay_len[f], size = len + 4u;   // MPDU bytes, PSDU bytes (FCS included)
    uint16_t* d = desc + (size_t)f * job.desc_stride;
    uint8_t hdr[6];
    tx11b_plcp_header(hdr, job.rate_kbps, job.rate_code, size);
    const uint32_t fcs = crcs ? crcs[f] : 0u;
    const uint32_t plcp = tx11b_legacy_plcp_bytes(job.short_preamble), nsync = job.short_preamble ? 7u : 16u;
    const uint32_t n_dbpsk = job.short_preamble ? 9u : (job.rate_kbps == 1000 ? plcp + size : plcp);
    unsigned reg = job.short_preamble ? 0x1Bu : 0x6Cu;                                  // DOT11B_PLCP_{SHORT,LONG}_TX_SCRAMBLER_REGISTER
    unsigned q = 2u, odd = 0;                                                           // ref 0 = phase pi
    const uint32_t total = plcp + (job.data_chips_per_byte ? size : 0u);
    for (uint32_t i = 0; i < total; i++) {
        unsigned b;
        if (i < nsync) b = job.short_preamble ? 0x00u : 0xFFu;
        else if (i == nsync) b = job.short_preamble ? 0xCFu : 0xA0u;                   // SFD 0x05CF / 0xF3A0, little endian
        else if (i == nsync + 1u) b = job.short_preamble ? 0x05u : 0xF3u;
        else if (i < plcp) b = hdr[i - nsync - 2u];
        else if (i < plcp + len || job.fcs_in_payload) b = p[i - plcp];
        else b = (fcs >> (8u * (i - plcp - len))) & 0xFFu;
        const unsigned sb = tx11b_scramble(b, reg);
        d[i] = (uint16_t)(sb | (q << 8) | (odd << 10));
        if (i < n_dbpsk) {                                                              // DBPSK: pi per one bit
            unsigned par = sb; par ^= par >> 4; par ^= par >> 2; par ^= par >> 1;
            q = (q + 2u * (par & 1u)) & 3u;
        } else if (i < plcp || job.rate_kbps == 2000) {                                 // DQPSK: a rotation per dibit
            q = (q + q_of_dqpsk(sb) + q_of_dqpsk(sb >> 2) + q_of_dqpsk(sb >> 4) + q_of_dqpsk(sb >> 6)) & 3u;
        } else if (job.rate_kbps == 5500) {                                             // two CCK symbols, the second one odd
            q = (q + q_of_dqpsk(sb) + q_of_dqpsk(sb >> 4) + 2u) & 3u;
        } else {                                                                        // CCK 11: even / odd symbols alternate
            q = (q + q_of_dqpsk(sb) + 2u * odd) & 3u; odd ^= 1u;
        }
    }
}

// chip k of a frame from its descriptor row, as (re & 0xFF) | (im << 8): the entry of the reference's table the encoder copies
__device__ __forceinline__ uint32_t tx11b_legacy_chip(const uint16_t* __restrict__ d, uint32_t k, const Tx11bLegacyJob& job, uint32_t nchips) {
    if (k >= nchips) return 0u;
    const unsigned BARKER_NEG = 0x712u;                                                 // bit k set where Barker11[k] = -1
    const uint32_t ndb = job.short_preamble ? 9u * 88u : (job.rate_kbps == 1000 ? nchips : 24u * 88u);
    unsigned q; bool dbpsk = false;
    if (k < ndb) {                                                                      // DBPSK: +127 / -128 (bbb_dbpsk.c:17-19)
        const uint32_t byte = k / 88u, r = k - byte * 88u, bit = r / 11u, c = r - bit * 11u;
        const unsigned w = __ldg(d + byte);
        unsigned par = (w & 0xFFu) & ((2u << bit) - 1u); par ^= par >> 4; par ^= par >> 2; par ^= par >> 1;
        q = ((w >> 8) & 3u) + 2u * (par & 1u) + 2u * ((BARKER_NEG >> c) & 1u);
        dbpsk = true;
    } else {
        const uint32_t hc = tx11b_legacy_header_chips(job.short_preamble);
        uint32_t byte, r, cpb = job.data_chips_per_byte;
        if (k < hc) { cpb = 44u; byte = 9u + (k - ndb) / 44u; r = (k - ndb) % 44u; }     // short preamble: the header is DQPSK
        else { byte = tx11b_legacy_plcp_bytes(job.short_preamble) + (k - hc) / cpb; r = (k - hc) % cpb; }
        const unsigned w = __ldg(d + byte), sb = w & 0xFFu;
        q = (w >> 8) & 3u;
        if (cpb == 44u) {                                                               // DQPSK (bbb_dqpsk.c)
            const uint32_t s = r / 11u, c = r - s * 11u;
            for (uint32_t t = 0; t <= s; t++) q += q_of_dqpsk(sb >> (2u * t));
            q += 2u * ((BARKER_NEG >> c) & 1u);
        } else {                                                                        // CCK: chip i of phi1 .. phi4 (bbb_cck5.c, bbb_cck11.c)
            unsigned p2, p3, p4, i = r;
            if (cpb == 16u) {
                const unsigned n = (r < 8u) ? (sb & 15u) : (sb >> 4);
                q += q_of_dqpsk(sb); if (r >= 8u) q += q_of_dqpsk(sb >> 4) + 2u;
                p2 = 1u + 2u * ((n >> 2) & 1u); p3 = 0u; p4 = 2u * ((n >> 3) & 1u); i = r & 7u;
            } else {
                q += q_of_dqpsk(sb) + 2u * ((w >> 10) & 1u);
                p2 = q_of_cck11(sb >> 2); p3 = q_of_cck11(sb >> 4); p4 = q_of_cck11(sb >> 6);
            }
            if (!(i & 1u)) q += p2;                                                     // phi2 on chips 0, 2, 4, 6
            if (!(i & 2u)) q += p3;                                                     // phi3 on chips 0, 1, 4, 5
            if (!(i & 4u)) q += p4;                                                     // phi4 on chips 0 .. 3
            if (i == 3u || i == 6u) q += 2u;
        }
    }
    q &= 3u;                                                                            // 0: 1, 1: +j, 2: -1, 3: -j
    const uint32_t neg = dbpsk ? 0x80u : 0x81u;                                         // -128 (DBPSK) or -127
    const uint32_t a = (q & 2u) ? neg : 0x7Fu;
    return (q & 1u) ? (a << 8) : a;
}

#define SB_TX11B_LEGACY_THREADS 128
#define SB_TX11B_LEGACY_CHIPS (SB_TX11B_LEGACY_THREADS * 2 + 9)      // a CTA's 1024 samples = 256 chip periods, plus 9 of filter history

// grid: x = frame, y = tiles of 1024 samples of the slot; FILTER 0 = encoder output, 1 = SSE filter body, 2 = ASM body
template <int FILTER>
__global__ void __launch_bounds__(SB_TX11B_LEGACY_THREADS) k_tx11b_legacy_spread(const uint32_t* __restrict__ pay_len, Tx11bLegacyJob job,
        const uint16_t* __restrict__ desc, int8_t* __restrict__ out, uint64_t out_stride /*samples, multiple of 8*/, uint32_t* __restrict__ nsamples) {
    __shared__ uint16_t s_chip[SB_TX11B_LEGACY_CHIPS];
    const uint32_t f = blockIdx.x;
    const uint32_t size = job.fcs_in_payload ? pay_len[f] : pay_len[f] + 4u;
    const uint32_t nchips = tx11b_legacy_header_chips(job.short_preamble) + size * job.data_chips_per_byte;
    const uint32_t ns = tx11b_legacy_nsamples(size, job.short_preamble, job.data_chips_per_byte);
    const uint64_t s_blk = (uint64_t)blockIdx.y * (SB_TX11B_LEGACY_THREADS * 8);
    if (s_blk >= out_stride) return;
    if (blockIdx.y == 0 && threadIdx.x == 0 && nsamples) nsamples[f] = ns;
    const int64_t k_lo = (int64_t)(s_blk >> 2) + (FILTER ? 2 - 9 : 0);                 // first chip the CTA reads
    const bool inside = s_blk < ns;
    if (inside) {
        const uint16_t* d = desc + (size_t)f * job.desc_stride;
        for (int i = threadIdx.x; i < SB_TX11B_LEGACY_CHIPS; i += SB_TX11B_LEGACY_THREADS) {
            const int64_t k = k_lo + i;
            s_chip[i] = (uint16_t)((FILTER ? k >= 2 : k >= 0) && k < (int64_t)nchips ? tx11b_legacy_chip(d, (uint32_t)k, job, nchips) : 0u);
        }
    }
    __syncthreads();
    const uint64_t s0 = s_blk + threadIdx.x * 8u;
    if (s0 >= out_stride) return;
    uint32_t w[4] = {0u, 0u, 0u, 0u};                                                   // 8 COMPLEX8 samples
    if (inside && s0 < ns) {
        const int loc = threadIdx.x * 2;                                                // chip of this thread's first sample group, minus k_lo's offset
        if (FILTER == 0) {
            w[0] = s_chip[loc]; w[2] = s_chip[loc + 1];                                 // chip, three zeros, chip, three zeros
        } else {
#pragma unroll
            for (int g = 0; g < 2; g++) {
                const uint32_t p = (uint32_t)(s0 >> 2) + g;                             // filter output group
                int c[10][2];                                                           // c[m] = chip p + 2 - m
#pragma unroll
                for (int m = 0; m < 10; m++) { const uint32_t v = s_chip[loc + g + 9 - m]; c[m][0] = (int8_t)(v & 0xFFu); c[m][1] = (int8_t)(v >> 8); }
                uint32_t y[4];
#pragma unroll
                for (int r = 0; r < 4; r++) {
                    int a[2];
#pragma unroll
                    for (int x = 0; x < 2; x++) {
                        int s = 0;
#pragma unroll
                        for (int m = 1; m < 10; m++) s += c[m][x] * fir37_h(r + 4 * m);
                        const int h0 = (FILTER == 1 && r > 0 && (p & 1u) == 0) ? 1 : fir37_h(r);   // variant 0: even group, rows 1..3 read row 0
                        s += c[0][x] * h0;
                        a[x] = min(max(s >> 8, -128), 127) & 0xFF;
                    }
                    y[r] = (uint32_t)a[0] | ((uint32_t)a[1] << 8);
                }
                w[2 * g] = y[0] | (y[1] << 16); w[2 * g + 1] = y[2] | (y[3] << 16);
            }
        }
    }
    *reinterpret_cast<uint4*>(out + 2ull * ((uint64_t)f * out_stride + s0)) = make_uint4(w[0], w[1], w[2], w[3]);
}

}  // namespace sb
