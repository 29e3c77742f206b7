// sora_b200 — 802.11a transmit kernels (sm_90a): SURVEY.md §8(f) rank 2, the reference's brick modulator on the device.
//
//   k_tx11a_preamble   one warp, once per handle: the 640-sample short/long training waveform exactly as TTS11aSrc builds it
//                      (Brick11/src/preamble11a.hpp:22-104: two fixed-point IFFT<128>, >> 4, periodic extension, GI2, window).
//   k_tx11a            one warp per OFDM symbol (symbol 0 = SIGNAL): every symbol is independent once the scrambler is read as
//                      a 127-periodic sequence and the encoder state as "the previous six scrambled bits":
//                      TBB11aSrc byte stream (PHY_11a.hpp:125-190) -> T11aSc (scramble.hpp:169-262) -> TConvEncode_12/23/34
//                      (conv_enc.hpp:5-280) -> T11aInterleave* (interleave.hpp:16-96) -> TMap11a* (mapper11a.hpp:13-298) ->
//                      T11aAddPilot (pilot.hpp:31-118) -> TIFFTx (fft.hpp:9-60: zero-stuffed IFFT<128>, >> 4, GI, window) ->
//                      TPackSample16to8 (stdbrick.hpp:413-445).
//   Output per frame: `lead` zero samples, 640 preamble samples, 160 per symbol, zeros up to the slot size; either COMPLEX8 (what
//   `demod11 -m` writes) or COMPLEX16 = COMPLEX8 << 8 (what ConvertModFile2DumpFile_8b feeds the receiver), so that a slot can go
//   straight into sb200_rx11a_batch.
#pragma once
#include "tables.cuh"
#include "viterbi_k7_common.cuh"
#include "tx_frames.cuh"

namespace sb {

// a * conj(w) >> 15 with the reference's negation of a.re (vector128.h:1215-1231 conj_mul_shift)
__device__ __forceinline__ cs16 conj_tw(cs16 a, cs16 w) {
    const int re = wadd(a.re * w.re, a.im * w.im), im = wadd(a.im * w.re, neg16(a.re) * w.im);
    return mk(sx16(re >> 15), sx16(im >> 15));
}
// radix-4 DIF butterfly of IFFTSSE<N> (ifft_r4dif.h:12-47); outputs at the same four slots: X(4k), X(4k+2), X(4k+1), X(4k+3)
__device__ __forceinline__ void ir4_butterfly(cs16& a, cs16& b, cs16& c, cs16& d, cs16 w1, cs16 w2, cs16 w3) {
    a = sra(a, 2); b = sra(b, 2); c = sra(c, 2); d = sra(d, 2);
    const cs16 ac = adds(a, c), bd = adds(b, d), a_c = subs(a, c), b_d = subs(b, d), jbd = mulj(b_d);
    a = adds(ac, bd);
    b = conj_tw(subs(ac, bd), w2);
    c = conj_tw(adds(a_c, jbd), w1);
    d = conj_tw(subs(a_c, jbd), w3);
}
// IFFTSSEEx<8> (ifft_r4dif.h:90-139) on eight consecutive points; negations are one's complements as in the SSE code
__device__ __forceinline__ void idft8(cs16 (&x)[8]) {
    cs16 a[4], b[4], s[4], d[4];
#pragma unroll
    for (int i = 0; i < 4; i++) { a[i] = sra(x[i], 3); b[i] = sra(x[4 + i], 3); d[i] = subs(a[i], b[i]); s[i] = adds(a[i], b[i]); }
    d[2] = mk(~d[2].im, d[2].re); d[3] = mk(~d[3].im, d[3].re);                             // upper two times j
    cs16 u[4] = {adds(d[0], d[2]), adds(d[1], d[3]), adds(cnot(d[2]), d[0]), adds(cnot(d[3]), d[1])};
    const cs16 W1 = mk(23169, -23169), W3 = mk(-23169, -23169), W0 = mk(32767, 0);       // wFFTLUT8 (fft_lut_twiddle.h)
    u[0] = conj_tw(u[0], W0); u[1] = conj_tw(u[1], W1); u[2] = conj_tw(u[2], W0); u[3] = conj_tw(u[3], W3);
    x[4] = adds(u[0], u[1]); x[5] = adds(cnot(u[1]), u[0]); x[6] = adds(u[2], u[3]); x[7] = adds(cnot(u[3]), u[2]);
    cs16 v[4] = {adds(s[0], s[2]), adds(s[1], s[3]), adds(cnot(s[2]), s[0]), adds(cnot(s[3]), s[1])};
    v[3] = mk(~v[3].im, v[3].re);
    x[0] = adds(v[0], v[1]); x[1] = adds(cnot(v[1]), v[0]); x[2] = adds(v[2], v[3]); x[3] = adds(cnot(v[3]), v[2]);
}
// IFFT<128> of the warp-private 128-word shared buffer (packed c16), in place; bin/time index i ends up at slot rev7(i)
__device__ __forceinline__ void warp_ifft128(uint32_t* x, const DevTablesTx& X, int lane) {
    __syncwarp();
    {   cs16 a = unpack(x[lane]), b = unpack(x[lane + 32]), c = unpack(x[lane + 64]), d = unpack(x[lane + 96]);
        ir4_butterfly(a, b, c, d, unpack(__ldg(X.tw128 + lane)), unpack(__ldg(X.tw128 + 32 + lane)), unpack(__ldg(X.tw128 + 64 + lane)));
        x[lane] = pack(a); x[lane + 32] = pack(b); x[lane + 64] = pack(c); x[lane + 96] = pack(d); }
    __syncwarp();
    {   const int base = (lane >> 3) * 32 + (lane & 7), j = lane & 7;
        cs16 a = unpack(x[base]), b = unpack(x[base + 8]), c = unpack(x[base + 16]), d = unpack(x[base + 24]);
        ir4_butterfly(a, b, c, d, unpack(__ldg(X.tw32 + j)), unpack(__ldg(X.tw32 + 8 + j)), unpack(__ldg(X.tw32 + 16 + j)));
        x[base] = pack(a); x[base + 8] = pack(b); x[base + 16] = pack(c); x[base + 24] = pack(d); }
    __syncwarp();
    if (lane < 16) {
        cs16 v[8];
#pragma unroll
        for (int i = 0; i < 8; i++) v[i] = unpack(x[8 * lane + i]);
        idft8(v);
#pragma unroll
        for (int i = 0; i < 8; i++) x[8 * lane + i] = pack(v[i]);
    }
    __syncwarp();
}
__device__ __forceinline__ int rev7(int i) { return (int)(__brev((unsigned)i) >> 25); }
__device__ __forceinline__ int pack8s(int v) { return v > 127 ? 127 : (v < -128 ? -128 : v); }

__global__ void __launch_bounds__(32) k_tx11a_preamble(DevTablesTx X) {
    __shared__ uint32_t s[128];
    const int lane = threadIdx.x;
    const int sts = (int)(unsigned short)(1.0 * 10720 * 1.472), lts = 10720;
    static const signed char L[53] = {1,1,-1,-1,1,1,-1,1,-1,1,1,1,1,1,1,-1,-1,1,1,-1,1,-1,1,1,1,1,0,
                                      1,-1,-1,1,1,-1,1,-1,1,-1,-1,-1,-1,-1,1,1,-1,-1,1,-1,1,-1,1,1,1,1};
    for (int i = lane; i < 128; i += 32) {
        int v = 0;
        if (i == 12 || i == 16 || i == 20 || i == 24 || i == 104 || i == 112 || i == 124) v = sts;
        if (i == 4 || i == 8 || i == 108 || i == 116 || i == 120) v = -sts;
        s[i] = pack(mk(v, v));
    }
    warp_ifft128(s, X, lane);
    for (int i = lane; i < 320; i += 32) { cs16 c = sra(unpack(s[rev7(i & 127)]), 4); if (i < 2 || i >= 318) c = sra(c, 1); X.preamble[i] = pack(c); }
    __syncwarp();
    for (int i = lane; i < 128; i += 32) {
        const int k = i < 64 ? i : i - 128; int v = 0;
        if (k >= -26 && k <= 26 && k != 0) v = L[k + 26] > 0 ? lts : -lts;
        s[i] = pack(mk(v, 0));
    }
    warp_ifft128(s, X, lane);
    for (int i = lane; i < 320; i += 32) {                                              // [GI2 = last 64 | T1 | T2]
        cs16 c = sra(unpack(s[rev7((i + 64) & 127)]), 4); if (i < 2 || i >= 318) c = sra(c, 1);
        X.preamble[320 + i] = pack(c);
    }
}

struct TxJob {
    uint32_t rate_code, nbpsc, code_rate, ndbps;   // SIGNAL rate bits, N_BPSC, CR_*, N_DBPS
    uint32_t ndbps_pad;                             // N_DBPS the padding rule uses (doubled at 9 Mbps, PHY_11a.hpp:113-116)
    uint32_t lead, fmt16;                           // zero samples in front of the preamble; 0 = COMPLEX8 out, 1 = COMPLEX16 (<< 8)
    uint32_t max_sym;                               // symbols per frame the grid covers (SIGNAL included)
};

// CRC-32 of every MPDU (what fb11amod_config.hpp:40 stores in CF_11aTxVector::crc32): one thread per frame
__global__ void __launch_bounds__(128) k_tx11a_crc(const uint8_t* __restrict__ payload, const uint64_t* __restrict__ pay_off, const uint32_t* __restrict__ pay_len,
                                                   uint32_t nframes, DevTables T, uint32_t* __restrict__ crcs) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nframes) return;
    const uint8_t* p = payload + pay_off[f]; const uint32_t n = pay_len[f];
    uint32_t c = 0xFFFFFFFFu;
    for (uint32_t i = 0; i < n; i++) c = (c >> 8) ^ __ldg(T.crc32 + ((c ^ p[i]) & 0xFFu));
    crcs[f] = ~c;
}

// ---- the per-symbol bit path the OFDM modulators share (k_tx11a, k_tx11a_legacy, k_tx11n) ------------------------------------------------
// even parity of the SIGNAL word into bit 17, folded over the word as the caller built it (a LENGTH of 4096 lands on the parity bit itself)
__device__ __forceinline__ uint32_t sig_parity(uint32_t w) {
    uint32_t p = w ^ (w >> 16); p ^= p >> 8; p ^= p >> 4; p ^= p >> 2; p ^= p >> 1;
    return w | (p & 1u) << 17;
}
// data bits of the 802.11a SIGNAL symbol: six zero bits of encoder history, then the 24 bits of the word
__device__ __forceinline__ void signal_bits(uint8_t* sd, uint32_t sig, int lane) {
    if (lane < 30) sd[lane] = lane < 6 ? 0 : (uint8_t)((sig >> (lane - 6)) & 1u);
}
// scrambled data bits d[j], j in [n0 - 6, n0 + nd), into sd[0 .. nd + 6): byte 0, 1 the SERVICE field, then the payload up to byte
// body_end, the FCS up to tail_at, the tail and the pad.  The scrambler is read as a 127-periodic sequence from `phase` (the seed's place in
// it; 255 = the all-zero state, no scrambling); the six tail bits are not scrambled (TAIL_SCRAMBLE: code & 0xC0).  Bits at or past `limit`
// are zero and not scrambled either (the FlushPort bytes of 802.11n).
__device__ __forceinline__ void scrambled_bits(uint8_t* sd, uint32_t n0, uint32_t nd, const uint8_t* pl, uint32_t body_end, uint32_t tail_at,
                                               uint32_t fcs, uint32_t phase, const DevTablesTx& X, int lane, uint32_t limit = 0xFFFFFFFFu) {
    for (uint32_t i = lane; i < nd + 6u; i += 32) {
        const int j = (int)n0 - 6 + (int)i;
        uint32_t bit = 0;
        if (j >= 0 && (uint32_t)j < limit) {
            const uint32_t by = (uint32_t)j >> 3, bi = (uint32_t)j & 7u;
            uint32_t raw = 0;
            if (by >= 2u && by < body_end) raw = pl[by - 2u]; else if (by >= body_end && by < tail_at) raw = (fcs >> (8u * (by - body_end))) & 0xFFu;
            const uint32_t scr = phase == 255u ? 0u : __ldg(X.scr_seq + (phase + (uint32_t)j) % 127u);
            bit = ((raw >> bi) & 1u) ^ scr;
            if (by == tail_at && bi < 6u) bit = 0;
        }
        sd[i] = (uint8_t)bit;
    }
}
// coded bit k of a symbol (puncture pattern of TConvEncode_12/23/34), straight from its data bits; puncture groups never straddle a
// symbol, so k is local to the symbol
__device__ __forceinline__ uint32_t coded_bit(const uint8_t* sd, uint32_t cr, uint32_t k) {
    uint32_t n, isb;
    if (cr == CR_12) { n = k >> 1; isb = k & 1u; }
    else if (cr == CR_34) { const uint32_t g = k >> 2, r = k & 3u; n = 3u * g + (r == 3u ? 2u : r >> 1); isb = (r == 1u || r == 3u); }
    else { const uint32_t g = k / 3u, r = k - 3u * g; n = 2u * g + (r == 2u ? 1u : 0u); isb = r == 1u; }          // rate 2/3: A0 B0 A1 (conv_enc.hpp:102-188)
    const uint8_t* d = sd + 6 + n;                      // d[0] = x, d[-1] = previous ...; generators 133 (A) and 171 (B) share taps 0, 2, 3, 6
    return (d[0] ^ d[-2] ^ d[-3] ^ d[-6] ^ (isb ? d[-1] : d[-5])) & 1u;
}
// data carrier d (AddPilot order: -(hw + 2) .. -1, then 1 .. hw + 2, pilots skipped) to its slot of the zero-stuffed IFFT<128> input
// (bins 32..63 move to 96..127); hw = 24 for 802.11a and the 802.11n SIG symbols, 26 for HT data
__device__ __forceinline__ int carrier_slot(int d, int hw) {
    int bin = d < hw ? 62 - hw + d : d - hw + 1;
    if (d < hw) { if (bin >= 43) bin++; if (bin >= 57) bin++; } else { if (bin >= 7) bin++; if (bin >= 21) bin++; }
    return bin < 32 ? bin : bin + 64;
}
// the pilots of carriers -21, -7, 7, 21 into their slots of the zero-stuffed IFFT<128> input
__device__ __forceinline__ void put_pilots(uint32_t* xs, int m21, int m7, int p7, int p21) {
    xs[43 + 64] = pack(mk(m21, 0)); xs[57 + 64] = pack(mk(m7, 0)); xs[7] = pack(mk(p7, 0)); xs[21] = pack(mk(p21, 0));
}
// T11aAddPilot (pilot.hpp:96-109) at amplitude a: polarity entry 127 for SIGNAL, then 0, 1, ... for the symbols behind it
__device__ __forceinline__ void pilots11a(uint32_t* xs, const DevTables& T, uint32_t sym, int a) {
    const int s = __ldg(T.pilot_neg + (sym == 0 ? 127u : (sym - 1u) % 127u)) ? -a : a;
    put_pilots(xs, s, s, s, -s);
}
// time sample behind output sample i (0 .. 159) of a symbol: the last 32 samples go in front as the guard interval
__device__ __forceinline__ uint32_t gi_sample(uint32_t i) { return i < 32u ? 96u + i : i - 32u; }

#define SB_TX_WARPS 4
__global__ void __launch_bounds__(32 * SB_TX_WARPS) k_tx11a(const uint8_t* __restrict__ payload, const uint64_t* __restrict__ pay_off, const uint32_t* __restrict__ pay_len,
        const uint8_t* __restrict__ seeds, uint32_t nframes, TxJob job, DevTables T, DevTablesTx X, const uint16_t* __restrict__ inv_deint,
        const uint32_t* __restrict__ crcs, void* __restrict__ out, uint64_t out_stride /*samples per slot*/, uint32_t* __restrict__ nsamples) {
    __shared__ uint32_t s_x[SB_TX_WARPS][128];
    __shared__ uint8_t s_d[SB_TX_WARPS][232];           // scrambled data bits of the symbol, six bits of history in front
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const uint32_t f = blockIdx.x;                         // frames on x (no 65535 limit), symbol groups on y
    const uint32_t sym = blockIdx.y * SB_TX_WARPS + wib;    // 0 = SIGNAL, 1.. = data; symbols >= job.max_sym do the preamble / zero fill
    if (f >= nframes) return;
    const uint32_t len = pay_len[f];
    const uint32_t nsym = tx11a_nsym(len, job.ndbps, job.ndbps_pad);
    const uint32_t used = job.lead + 640u + 160u * (1u + nsym);
    uint32_t* out16 = (uint32_t*)out + (size_t)f * out_stride; uint16_t* out8 = (uint16_t*)out + (size_t)f * out_stride;
    auto put = [&](uint32_t pos, cs16 c) {              // one complex sample through TPackSample16to8 (+ optional << 8)
        const int re = pack8s(c.re), im = pack8s(c.im);
        if (job.fmt16) out16[pos] = ((uint32_t)(re << 8) & 0xFFFFu) | ((uint32_t)(im << 8) << 16);
        else out8[pos] = (uint16_t)((re & 0xFF) | ((im & 0xFF) << 8));
    };
    if (sym >= job.max_sym) {                           // helper warps: lead zeros, preamble, trailing zeros
        const uint32_t helper = sym - job.max_sym, nhelp = gridDim.y * SB_TX_WARPS - job.max_sym;
        if (helper == 0 && lane == 0 && nsamples) nsamples[f] = used;
        for (uint64_t p = (uint64_t)helper * 32 + lane; p < out_stride; p += (uint64_t)nhelp * 32) {
            if (p >= job.lead && p < job.lead + 640u) put((uint32_t)p, unpack(X.preamble[p - job.lead]));
            else if (p < job.lead || p >= used) put((uint32_t)p, mk(0, 0));
        }
        return;
    }
    if (sym > nsym) return;
    if ((uint64_t)used > out_stride) return;            // the host checked this; never write outside the slot
    // ---- scrambled data bits d[j], j in [n0 - 6, n0 + nd) -----------------------------------------------------------------
    const uint32_t nd = sym == 0 ? 24u : job.ndbps, nbpsc = sym == 0 ? 1u : job.nbpsc, cr = sym == 0 ? (uint32_t)CR_12 : job.code_rate;
    const uint32_t n0 = sym == 0 ? 0u : (sym - 1u) * job.ndbps;
    uint8_t* sd = s_d[wib];
    if (sym == 0) signal_bits(sd, sig_parity(job.rate_code | ((len + 4u) << 5)), lane);
    else {
        const uint32_t seed = seeds ? seeds[f] : 0xFFu;
        // the FCS is CF_11aTxVector::crc32, computed by k_tx11a_crc
        scrambled_bits(sd, n0, nd, payload + pay_off[f], 2u + len, 6u + len, __ldg(crcs + f), __ldg(X.scr_phase + (seed >> 1)), X, lane);
    }
    __syncwarp();
    const uint16_t* inv = inv_deint + (nbpsc == 1 ? 0 : nbpsc == 2 ? 48 : nbpsc == 4 ? 144 : 336);     // air position -> coded index
    const int km = nbpsc == 1 ? 10720 : nbpsc == 2 ? (int)(short)(10720 / 1.414) : nbpsc == 4 ? (int)(short)(10720 / 3.162) : (int)(short)(10720 / 6.481);
    auto level = [&](uint32_t p0, uint32_t m) -> int {   // InitQamMapLut (mapper11a.hpp:17-46): first bit is the Gray MSB
        uint32_t bin = 0, acc = 0;
        for (uint32_t i = 0; i < m; i++) { acc ^= coded_bit(sd, cr, __ldg(inv + p0 + i)); bin = (bin << 1) | acc; }
        return (2 * (int)bin - ((1 << m) - 1)) * km;
    };
    uint32_t* xs = s_x[wib];
    for (int i = lane; i < 128; i += 32) xs[i] = 0;
    __syncwarp();
#pragma unroll
    for (int w = 0; w < 2; w++) {                       // lanes 0..23 place data carriers d = lane and lane + 24 (T11aAddPilot order: -26..-1, 1..26)
        const int dd = lane + 24 * w;
        if (lane < 24) {
            cs16 c;
            if (nbpsc == 1) c = mk(coded_bit(sd, cr, __ldg(inv + dd)) ? 10720 : -10720, 0);
            else { const uint32_t h = nbpsc >> 1; c = mk(level((uint32_t)dd * nbpsc, h), level((uint32_t)dd * nbpsc + h, h)); }
            xs[carrier_slot(dd, 24)] = pack(c);
        }
    }
    if (lane == 24) pilots11a(xs, T, sym, 10720);
    warp_ifft128(xs, X, lane);
    // ---- >> 4, guard interval, window, pack, store (fft.hpp:27-41) ----------------------------------------------------------
    const uint32_t base = job.lead + 640u + 160u * sym;
    for (uint32_t i = lane; i < 160u; i += 32) {
        cs16 c = sra(unpack(xs[rev7((int)gi_sample(i))]), 4);
        if (i < 2u || i >= 158u) c = sra(c, 1);
        put(base + i, c);
    }
}

} // namespace sb
