// 802.11b transmit on sm_90a: the brick modulator graph of kernel/bb/demod11/fb11bmod_config.hpp:19-45
//   TBB11bSrc -> TSc741 -> TBB11bMRSelect -> {TBB11bDBPSKSpread, TBB11bDQPSKSpread, TCCK5Encode, TCCK11Encode}
//             -> TQuickPulseShaper -> TPackSample16to8 -> TModSink
// split where the data dependence allows it:
//   k_tx11b_code   one thread per frame: everything that is a recurrence over the byte stream — PLCP header (CRC-16), the
//                  self-synchronising 7-4-1 scrambler and the differential phase reference — leaving one 16-bit descriptor
//                  per byte: [7:0] the DBPSK/DQPSK phase code or the scrambled CCK 5.5 byte with [9:8] the phase reference in front of it;
//                  at 11 Mbps the symbol's four phase terms as quarter turns (m0 m1 + odd-symbol pi, m2, m3, m4).  ~20 integer instructions per byte.
//                  Reference: PHY_11b.hpp:82-151,216-293; scramble.hpp:9-91; barkerspread.hpp:25-41,129-156; cck.hpp:854-866,945-953.
//   k_tx11b_shape  every output sample independently: a CTA stages the chips its 2048 samples depend on in shared memory
//                  (chip = pure function of a descriptor and the chip number), then each thread runs the 5-input polyphase
//                  shaper for 8 consecutive samples and stores them with one or two 128-bit writes.  HBM-write bound:
//                  2 (COMPLEX8) or 4 (COMPLEX16) bytes per sample out, 0.5 descriptor bytes per chip in.
//                  Reference: barkerspread.hpp:48-65,160-188; cck.hpp:797-828,893-918; pulse.hpp:260-379; stdbrick.hpp:413-445,278-330.
#pragma once
#include "tx11a_kernels.cuh"
#include "tx_frames.cuh"

namespace sb {

struct Tx11bJob {
    uint32_t rate_kbps, rate_code;       // 1000 / 2000 / 5500 / 11000; PLCP SIGNAL byte (bb/bbb.h:47-50)
    uint32_t chips_per_byte;             // 88 / 44 / 16 / 8
    uint32_t lead, fmt16;                // zero samples in front of the frame; 0 = COMPLEX8 out, 1 = COMPLEX16 (<< 8)
    uint32_t init_phase;                 // CF_DifferentialMap::last_phase in front of the first byte
    uint32_t desc_stride;                // descriptors per frame row
    short taps[20];                      // h(8) .. h(-11), pulse.hpp:279-305 (built on the host from the reference's formula)
};

// quarter turns of the reference's two phase alphabets and the way back
//   DQPSKEncode[]  = {1, -j, +j, -1} (cck.hpp:766)      -> 0, 3, 1, 2
//   CCK11D3D2[]    = {1, -1, +j, -j} (cck.hpp:767)      -> 0, 2, 1, 3
__device__ __forceinline__ unsigned q_of_dqpsk(unsigned i) { return (0x9Cu >> (2u * (i & 3u))) & 3u; }      // 0,3,1,2 packed little end first
__device__ __forceinline__ unsigned dqpsk_of_q(unsigned q) { return (0x78u >> (2u * (q & 3u))) & 3u; }      // 0,2,3,1
__device__ __forceinline__ unsigned q_of_cck11(unsigned i) { return (0xD8u >> (2u * (i & 3u))) & 3u; }      // 0,2,1,3

// PLCP header of a PSDU of `size` bytes (PHY_11b.hpp:82-136, PLCPGetLength in bbb_tx.c:39-65): SIGNAL, SERVICE (length extension in
// bit 7), LENGTH in microseconds, CRC-16 (CalcCRC16, core/inc/CRC16.h:37-48)
__device__ __forceinline__ void tx11b_plcp_header(uint8_t (&hdr)[6], uint32_t rate_kbps, uint32_t rate_code, uint32_t size) {
    uint32_t plen, ext = 0;
    if (rate_kbps == 1000) plen = size << 3;
    else if (rate_kbps == 2000) plen = size << 2;
    else if (rate_kbps == 5500) plen = ((size << 4) - 1u) / 11u + 1u;
    else { plen = ((size << 3) - 1u) / 11u + 1u; if (plen * 11u - (size << 3) >= 8u) ext = 1; }
    hdr[0] = (uint8_t)rate_code; hdr[1] = (uint8_t)(ext << 7); hdr[2] = (uint8_t)plen; hdr[3] = (uint8_t)(plen >> 8);
    unsigned c = 0xFFFFu;
    for (int i = 0; i < 4; i++) { c ^= hdr[i]; for (int k = 0; k < 8; k++) c = (c & 1u) ? (c >> 1) ^ 0x8408u : c >> 1; }
    c = ~c & 0xFFFFu; hdr[4] = (uint8_t)c; hdr[5] = (uint8_t)(c >> 8);
}
// byte b through the self-synchronising 7-4-1 scrambler (TSc741, gc_ScramblerLUT[b][reg]): o_k = x_k ^ s_k ^ s_(k+3) where the 4-ago tap
// is still old state (k < 4), then the taps that already see new output bits; reg moves on to the byte's last seven output bits
__device__ __forceinline__ unsigned tx11b_scramble(unsigned b, unsigned& reg) {
    const unsigned lo = (b ^ reg ^ (reg >> 3)) & 0xFu;
    const unsigned mid = ((b >> 4) ^ (reg >> 4) ^ lo) & 0x7u;
    const unsigned top = ((b >> 7) ^ lo ^ (lo >> 3)) & 1u;
    const unsigned sb = lo | (mid << 4) | (top << 7);
    reg = sb >> 1;
    return sb;
}

__global__ void __launch_bounds__(128) k_tx11b_code(const uint8_t* __restrict__ payload, const uint64_t* __restrict__ pay_off, const uint32_t* __restrict__ pay_len,
                                                    uint32_t nframes, Tx11bJob job, const uint32_t* __restrict__ crcs, uint16_t* __restrict__ desc, uint32_t* __restrict__ final_phase) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nframes) return;
    const uint8_t* p = payload + pay_off[f]; const uint32_t len = pay_len[f], size = len + 4u;
    uint16_t* d = desc + (size_t)f * job.desc_stride;
    uint8_t hdr[6];
    tx11b_plcp_header(hdr, job.rate_kbps, job.rate_code, size);
    const uint32_t fcs = crcs[f];
    unsigned reg = 0x6C;                                                                // DOT11B_PLCP_LONG_TX_SCRAMBLER_REGISTER
    unsigned ref = job.init_phase & 3u, odd = 0;
    const uint32_t total = 24u + size;
    for (uint32_t i = 0; i < total; i++) {
        unsigned b;
        if (i < 16u) b = 0xFF; else if (i == 16u) b = 0xA0; else if (i == 17u) b = 0xF3;
        else if (i < 24u) b = hdr[i - 18u];
        else if (i < 24u + len) b = p[i - 24u];
        else b = (fcs >> (8u * (i - 24u - len))) & 0xFFu;
        const unsigned sb = tx11b_scramble(b, reg);
        unsigned word;
        if (i < 24u || job.rate_kbps == 1000) {                                         // DBPSK: running parity of the bits, from the reference phase
            unsigned c = sb; c ^= c << 1; c ^= c << 2; c ^= c << 4; c &= 0xFFu;
            if (ref & 1u) c ^= 0xFFu;
            word = c; ref = (c >> 7) ? 3u : 0u;                                         // "compatible to dqpsk": pi = 11
        } else if (job.rate_kbps == 2000) {                                             // DQPSK: four dibits, each a rotation
            unsigned ph = ref, c = 0;
#pragma unroll
            for (int k = 0; k < 8; k += 2) { ph = dqpsk_of_q(q_of_dqpsk(ph) + q_of_dqpsk(sb >> k)); c |= ph << k; }
            word = c; ref = c >> 6;
        } else if (job.rate_kbps == 5500) {                                             // two 4-bit CCK symbols; the second carries the odd-symbol pi
            word = sb | (ref << 8);
            ref = dqpsk_of_q(2u + q_of_dqpsk(ref) + q_of_dqpsk(sb) + q_of_dqpsk(sb >> 4));
        } else {                                                                        // 11 Mbps: the four phase terms of the symbol as quarter turns
            const unsigned q0 = (q_of_dqpsk(ref) + q_of_dqpsk(sb) + 2u * odd) & 3u;     // m0 m1 and the odd-symbol pi
            word = q0 | (q_of_cck11(sb >> 2) << 2) | (q_of_cck11(sb >> 4) << 4) | (q_of_cck11(sb >> 6) << 6);
            ref = dqpsk_of_q(q0); odd ^= 1u;
        }
        d[i] = (uint16_t)word;
    }
    if (final_phase) final_phase[f] = ref;                                              // what CF_DifferentialMap::last_phase is left at
}

// chip n of a frame from its descriptor row: one of 1, j, -1, -j as the integer re + 65536 * im, so that one 32-bit multiply-add
// per tap filters both components (the low half borrows from the high half when re < 0; tx11b_unborrow undoes it at the end)
template <uint32_t rate_kbps>
__device__ __forceinline__ int tx11b_chip(const uint16_t* __restrict__ d, uint32_t n) {
    const unsigned BARKER_NEG = 0x712u;                                                 // bit k set where Barker11[k] = -1 (barkerspread.hpp:7)
    unsigned q; bool flip = false;
    if (n < 2112u || rate_kbps == 1000) {
        const uint32_t byte = n / 88u, r = n - byte * 88u, bit = r / 11u, k = r - bit * 11u;
        q = ((__ldg(d + byte) >> bit) & 1u) ? 2u : 0u; flip = (BARKER_NEG >> k) & 1u;
    } else {
        const uint32_t m = n - 2112u;
        if (rate_kbps == 2000) {
            const uint32_t byte = m / 44u, r = m - byte * 44u, sym = r / 11u, k = r - sym * 11u;
            q = q_of_dqpsk(__ldg(d + 24u + byte) >> (2u * sym)); flip = (BARKER_NEG >> k) & 1u;
        } else if (rate_kbps == 5500) {
            const uint32_t byte = m >> 4, i = m & 15u; const unsigned w = __ldg(d + 24u + byte), sb = w & 0xFFu, ref = (w >> 8) & 3u;
            // CCK5D3D2 rows as quarter turns (cck.hpp:768-773): {1,0,1,2,1,0,3,0} {3,0,3,2,3,0,1,0} {3,2,3,0,1,0,3,0} {1,2,1,0,3,0,1,0}
            const unsigned half = (i < 8u) ? (sb & 15u) : (sb >> 4);
            unsigned row;
            switch (half >> 2) {                                                        // packed little end first: chip c at bits [2c+1:2c]
                case 0: row = 1u | (0u << 2) | (1u << 4) | (2u << 6) | (1u << 8) | (0u << 10) | (3u << 12) | (0u << 14); break;
                case 1: row = 3u | (0u << 2) | (3u << 4) | (2u << 6) | (3u << 8) | (0u << 10) | (1u << 12) | (0u << 14); break;
                case 2: row = 3u | (2u << 2) | (3u << 4) | (0u << 6) | (1u << 8) | (0u << 10) | (3u << 12) | (0u << 14); break;
                default: row = 1u | (2u << 2) | (1u << 4) | (0u << 6) | (3u << 8) | (0u << 10) | (1u << 12) | (0u << 14); break;
            }
            q = q_of_dqpsk(ref) + q_of_dqpsk(sb) + ((row >> (2u * (i & 7u))) & 3u);
            if (i >= 8u) q += 2u + q_of_dqpsk(sb >> 4);
        } else {
            const uint32_t byte = m >> 3, i = m & 7u; const unsigned w = __ldg(d + 24u + byte);
            q = w;                                                                      // bits above the low two are cut off at the end, so the terms go in unmasked
            if (!(i & 1u)) q += w >> 2;                                                 // m2 on chips 0, 2, 4, 6
            if (!(i & 2u)) q += w >> 4;                                                 // m3 on chips 0, 1, 4, 5
            if (!(i & 4u)) q += w >> 6;                                                 // m4 on chips 0 .. 3
            if (i == 3u || i == 6u) q += 2u;
        }
    }
    if (flip) q += 2u;
    q &= 3u;                                                                            // 0: 1, 1: +j, 2: -1, 3: -j
    const int v = 1 << ((q & 1u) << 4);                                                 // 1 or j
    return (q & 2u) ? -v : v;
}

#define SB_TX11B_THREADS 256
#define SB_TX11B_SPT 8                 // samples per thread
// pulse.hpp:279-305 evaluated once: h(8) .. h(-11).  The host recomputes them from the reference's formula on every call and refuses
// to launch if they ever differ (sb200_tx11b_batch); compile-time values let the aligned path drop the eight zero taps.
#define SB_TX11B_TAPS {-1, 0, 3, 0, -6, 0, 34, 80, 102, 80, 34, 0, -6, 0, 3, 0, -1, 0, 1, 0}
__host__ __device__ constexpr int tx11b_branch_max(int k) {                              // largest |output| of polyphase branch k for chips in {-1, 0, 1}
    constexpr int H[20] = SB_TX11B_TAPS; int a = 0;
    for (int j = 0; j < 5; j++) a += H[4 * j + k] < 0 ? -H[4 * j + k] : H[4 * j + k];
    return a;
}
static_assert(tx11b_branch_max(0) <= 127 && tx11b_branch_max(1) <= 127 && tx11b_branch_max(2) <= 127 && tx11b_branch_max(3) <= 127,
              "TPackSample16to8 (packsswb) never saturates on this shaper, so the pack is a plain byte extraction");
// Both halves are kept non-negative by a bias of 128 (|output| <= 127, see above), so the low half never borrows from the high one; the bias
// is bit 7 of the byte that goes out and is flipped back after the bytes are gathered.
#define SB_TX11B_BIAS 0x00800080u

// ALIGNED: lead is a multiple of 4, so a thread's 8 samples are the two whole shaper vectors of chips n and n + 1
template <bool ALIGNED, uint32_t RATE>
__global__ void __launch_bounds__(SB_TX11B_THREADS) k_tx11b_shape(const uint32_t* __restrict__ pay_len, Tx11bJob job, const uint16_t* __restrict__ desc,
        void* __restrict__ out, uint64_t out_stride /*samples per slot, multiple of 8*/, uint32_t* __restrict__ nsamples) {
    __shared__ int s_chip[SB_TX11B_THREADS * SB_TX11B_SPT / 4 + 8];
    const uint32_t f = blockIdx.x;                                                      // frames on x: the y extent stops at 65535
    const uint32_t len = pay_len[f], nc = tx11b_nchips(len, job.chips_per_byte), ns = tx11b_nsamples(nc);
    const uint32_t s_blk = blockIdx.y * (SB_TX11B_THREADS * SB_TX11B_SPT);              // first slot sample of this CTA (the host keeps slots below 2^27 samples)
    if (s_blk >= out_stride) return;
    if (blockIdx.y == 0 && threadIdx.x == 0 && nsamples) nsamples[f] = job.lead + ns;
    // chips the CTA's samples lean on: n_lo .. n_lo + count - 1 (four chips of history in front)
    const int m_lo = (int)s_blk - (int)job.lead;                                        // frame-relative index of the CTA's first sample
    const int n_lo = (m_lo >> 2) - 4;                                                   // arithmetic shift = floor
    const int count = SB_TX11B_THREADS * SB_TX11B_SPT / 4 + 6;
    const uint32_t s0 = s_blk + threadIdx.x * SB_TX11B_SPT;
    const int nvec = (int)nc + 5;                                                       // shaper output vectors, flush included
    const bool inside = m_lo + SB_TX11B_THREADS * SB_TX11B_SPT > 0 && m_lo < nvec * 4;   // does the CTA touch the frame at all?
    if (inside) {
        const uint16_t* d = desc + (size_t)f * job.desc_stride;
        for (int i = threadIdx.x; i < count; i += SB_TX11B_THREADS) {
            const int n = n_lo + i;
            s_chip[i] = (n >= 0 && n < (int)nc) ? tx11b_chip<RATE>(d, (uint32_t)n) : 0;
        }
    }
    __syncthreads();
    if (s0 >= out_stride) return;
    uint32_t t[SB_TX11B_SPT];                                                           // per sample: re + 128 in the low half, im + 128 in the high half
#pragma unroll
    for (int i = 0; i < SB_TX11B_SPT; i++) t[i] = SB_TX11B_BIAS;
    if (inside) {
        if (ALIGNED) {
            constexpr int H[20] = SB_TX11B_TAPS;
            const int nA = ((int)s0 - (int)job.lead) >> 2;                                  // exact: both are multiples of 4
#pragma unroll
            for (int c = 0; c < 2; c++) {
                const int n = nA + c;
                if (n < 0 || n >= nvec) continue;
                const int loc = n - n_lo;
                int x[5];
#pragma unroll
                for (int j = 0; j < 5; j++) x[j] = s_chip[loc - j];
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    int a = (int)SB_TX11B_BIAS;
#pragma unroll
                    for (int j = 0; j < 5; j++) if (H[4 * j + k] != 0) a += x[j] * H[4 * j + k];
                    t[4 * c + k] = (uint32_t)a;
                }
            }
        } else {
#pragma unroll
            for (int i = 0; i < SB_TX11B_SPT; i++) {
                const int m = (int)s0 + i - (int)job.lead;
                if (m < 0 || m >= nvec * 4) continue;
                const int n = (m >> 2) - n_lo, k = m & 3;
                int a = (int)SB_TX11B_BIAS;
#pragma unroll
                for (int j = 0; j < 5; j++) a += s_chip[n - j] * (int)job.taps[4 * j + k];
                t[i] = (uint32_t)a;
            }
        }
    }
    // TPackSample16to8 keeps the low byte of each component (never saturates, see above); COMPLEX16 output is that byte << 8
    if (job.fmt16) {
        uint4 a, b; const uint32_t F = 0x80008000u;     // the bias, now in the high byte of each 16-bit component
        a.x = __byte_perm(t[0], 0, 0x2404) ^ F; a.y = __byte_perm(t[1], 0, 0x2404) ^ F; a.z = __byte_perm(t[2], 0, 0x2404) ^ F; a.w = __byte_perm(t[3], 0, 0x2404) ^ F;
        b.x = __byte_perm(t[4], 0, 0x2404) ^ F; b.y = __byte_perm(t[5], 0, 0x2404) ^ F; b.z = __byte_perm(t[6], 0, 0x2404) ^ F; b.w = __byte_perm(t[7], 0, 0x2404) ^ F;
        uint4* o = (uint4*)((uint32_t*)out + (size_t)f * out_stride + s0);
        o[0] = a; o[1] = b;
    } else {
        uint4 a; const uint32_t F = 0x80808080u;
        a.x = __byte_perm(t[0], t[1], 0x6420) ^ F; a.y = __byte_perm(t[2], t[3], 0x6420) ^ F; a.z = __byte_perm(t[4], t[5], 0x6420) ^ F; a.w = __byte_perm(t[6], t[7], 0x6420) ^ F;
        *(uint4*)((uint16_t*)out + (size_t)f * out_stride + s0) = a;
    }
}

}  // namespace sb
