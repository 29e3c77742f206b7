// 802.11n two-stream HT-mixed-format transmit on sm_90a: the modulator graphs of kernel/bb/demod11/fb11nmod_config.hpp:74-171
// (CreatePreambleGraph11n, CreateSigGraph11n, CreateModGraph11n) driven like kernel/bb/demod11/fb11n_mod.cpp:44-70.
//   k_tx11n   one warp per (OFDM symbol, stream): symbols 0..2 are L-SIG / HT-SIG 1 / HT-SIG 2 (one spectrum, stream 2 delayed by
//             TCSD<2>), symbols 3.. are DATA.  As in k_tx11a nothing is carried from symbol to symbol: the scrambler is read as a
//             127-periodic sequence, the encoder state is the six scrambled bits in front of the symbol, the stream parser / HT
//             interleaver are an index map (host-built inverse of interleave.hpp:33-60), so every warp goes straight from payload bytes
//             to 160 output samples: scramble, encode + puncture, parse, interleave, map, T11nAddPilot, TIFFTxOnly (warp_ifft128, no
//             scaling), TCSD<4> on stream 2, TAddGI.  Helper warps copy the two preamble blocks (tables regenerated on the host from
//             their defining formula, tx11n tables) and zero the rest of the slot.
//             Reference: PHY_11n.hpp:13-134,244-281; _b_lsig.h; _b_htsig.h; scramble.hpp:169-262; conv_enc.hpp; _b_stream_parser.h:36-49;
//             interleave.hpp:16-60,115-118; mapper11n.hpp:26-46; mapper11a.hpp; pilot.hpp:31-118; pilot_11n.hpp:8-83; _b_dot11_pilot.h:3-46;
//             fft.hpp:62-101; csd.hpp:38-51; gi.hpp:32-41; preamble11n.hpp:9-80.
#pragma once
#include "tx11a_kernels.cuh"

namespace sb {

struct DevTablesTx11n {
    const uint32_t* pre;       // [2][1120] packed c16: per stream L-STF + L-LTF (640) then HT-STF + HT-LTF x 2 (480), cyclic shifts applied
    const uint8_t*  inv;       // [2 (BPSK, QPSK)][2 (stream)][104]: air position -> bit index inside the stream's share of the symbol
    const uint16_t* inv16;     // [2 (16-QAM, 64-QAM)][2 (stream)][312]: the same for the 16-QAM / 64-QAM interleavers
};
struct Tx11nJob {
    uint32_t mcs, nbpsc, code_rate, ndbps;   // 8..14; N_BPSCS; CR_12 / CR_23 / CR_34; N_DBPS over both streams
    uint32_t enc_in, parse_in;               // input bursts of the encoder and of the stream parser, bytes (conv_enc.hpp, streamparser.hpp)
    uint32_t lead, max_sym;                  // zero samples in front; symbols per frame the grid covers (3 SIG + data)
};
__host__ __device__ inline uint32_t tx11n_nsym_signalled(uint32_t len, uint32_t ndbps) { return ((len + 4u) * 8u + 16u + 6u + ndbps - 1u) / ndbps; }   // ht_symbol_count
// data symbols the graph emits: the Flush padding (FlushPort: encoder burst, then stream-parser burst) can add one
__host__ __device__ inline uint32_t tx11n_nsym_emitted(uint32_t len, const Tx11nJob& j, uint32_t* enc_bits, uint32_t* coded_bits) {
    const uint32_t ns = tx11n_nsym_signalled(len, j.ndbps);
    uint32_t bytes = (ns * j.ndbps + 7u) / 8u; bytes = (bytes + j.enc_in - 1u) / j.enc_in * j.enc_in;
    const uint32_t cbytes = j.code_rate == CR_12 ? 2u * bytes : j.code_rate == CR_34 ? bytes / 3u * 4u : bytes / 2u * 3u;
    if (enc_bits) *enc_bits = bytes * 8u; if (coded_bits) *coded_bits = cbytes * 8u;
    return (cbytes + j.parse_in - 1u) / j.parse_in;
}

#define SB_TX11N_WARPS 4
__global__ void __launch_bounds__(32 * SB_TX11N_WARPS) k_tx11n(const uint8_t* __restrict__ payload, const uint64_t* __restrict__ pay_off, const uint32_t* __restrict__ pay_len,
        const uint8_t* __restrict__ seeds, uint32_t nframes, Tx11nJob job, DevTables T, DevTablesTx X, DevTablesTx11n N, const uint16_t* __restrict__ inv_deint,
        const uint32_t* __restrict__ crcs, uint32_t* __restrict__ out0, uint32_t* __restrict__ out1, uint64_t out_stride /*samples per slot*/, uint32_t* __restrict__ nsamples) {
    __shared__ uint32_t s_x[SB_TX11N_WARPS][128];
    __shared__ uint8_t s_d[SB_TX11N_WARPS][480];        // scrambled data bits of the symbol (<= 468), six bits of history in front
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const uint32_t f = blockIdx.x;
    const uint32_t unit = blockIdx.y * SB_TX11N_WARPS + wib;       // (symbol, stream) pairs first, helper warps behind them
    if (f >= nframes) return;
    const uint32_t len = pay_len[f];
    uint32_t enc_bits, coded_bits; const uint32_t nsym = tx11n_nsym_emitted(len, job, &enc_bits, &coded_bits);
    const uint32_t ns_sig = tx11n_nsym_signalled(len, job.ndbps);
    const uint32_t used = job.lead + 640u + 480u + 480u + 160u * nsym;
    uint32_t* outs[2] = {out0 + (size_t)f * out_stride, out1 + (size_t)f * out_stride};
    if (unit >= 2u * job.max_sym) {                     // helper warps: lead zeros, the two preamble blocks, trailing zeros
        const uint32_t helper = unit - 2u * job.max_sym, nhelp = gridDim.y * SB_TX11N_WARPS - 2u * job.max_sym;
        if (helper == 0 && lane == 0 && nsamples) nsamples[f] = used;
        const uint32_t l0 = job.lead, h0 = job.lead + 640u + 480u;
        for (uint64_t p = (uint64_t)helper * 32 + lane; p < out_stride; p += (uint64_t)nhelp * 32) {
#pragma unroll
            for (int a = 0; a < 2; a++) {
                if (p >= l0 && p < l0 + 640u) outs[a][p] = __ldg(N.pre + a * 1120 + (p - l0));
                else if (p >= h0 && p < h0 + 480u) outs[a][p] = __ldg(N.pre + a * 1120 + 640 + (p - h0));
                else if (p < l0 || p >= used) outs[a][p] = 0;
            }
        }
        return;
    }
    const uint32_t sym = unit >> 1, iss = unit & 1u;    // sym 0..2 SIG, 3.. DATA
    if (sym >= 3u + nsym || (sym < 3u && iss)) return;  // the SIG symbols are one spectrum: stream 1's warp writes both antennas
    if ((uint64_t)used > out_stride) return;            // the host checked this; never write outside the slot
    uint8_t* sd = s_d[wib];
    uint32_t* xs = s_x[wib];
    for (int i = lane; i < 128; i += 32) xs[i] = 0;
    const bool sig = sym < 3u;
    if (sig) {
        // ---- L-SIG (6 Mbps, length that spans the HT part) + HT-SIG (MCS, length, CRC-8): 72 bits, PHY_11n.hpp:244-281 ----------------------
        const uint32_t nsym_all = ns_sig + 5u, lsig_len = (nsym_all * 24u - 16u - 6u) / 8u;
        uint32_t lsig = 0xBu | (lsig_len << 5); uint32_t p = lsig ^ (lsig >> 16); p ^= p >> 8; p ^= p >> 4; p ^= p >> 2; p ^= p >> 1; lsig |= (p & 1u) << 17;
        const uint32_t L4 = len + 4u;
        const uint32_t h0 = job.mcs | ((L4 & 0xFFFFu) << 8) | (3u << 24);                           // _b_htsig.h:49-53: mcs, length, smoothing | not sounding
        unsigned c = 0xFF;                                                                          // CalcCRC8 over 4 bytes and 2 tail bits (CRC8.h:28-50)
        for (int i = 0; i < 4; i++) { c ^= (h0 >> (8 * i)) & 0xFFu; for (int k = 0; k < 8; k++) c = (c & 1u) ? (c >> 1) ^ 0xE0u : c >> 1; }
        for (int k = 0; k < 2; k++) c = (c & 1u) ? (c >> 1) ^ 0xE0u : c >> 1;                        // the two tail bits are zero
        c = ~c & 0xFFu;
        const uint32_t h1 = ((c << 2) & 0xFFu) | ((c >> 6) << 8);                                   // bytes 4, 5
        // info bit j of the 72: [0, 24) L-SIG, [24, 56) h0, [56, 72) h1
        if (lane < 30) {
            const int j = (int)(24u * sym) - 6 + lane;
            uint32_t bit = 0;
            if (j >= 0) bit = j < 24 ? (lsig >> j) & 1u : j < 56 ? (h0 >> (j - 24)) & 1u : (h1 >> (j - 56)) & 1u;
            sd[lane] = (uint8_t)bit;
        }
    } else {
        // ---- scrambled data bits d[j], j in [n0 - 6, n0 + N_DBPS): TBB11nSrc through T11aSc, then the FlushPort zero bytes ---------------------
        const uint32_t n0 = (sym - 3u) * job.ndbps;
        const uint8_t* pl = payload + pay_off[f];
        const uint32_t seed = seeds ? seeds[f] : 0xABu, phase = __ldg(X.scr_phase + (seed >> 1));   // fb11nmod_config.hpp:52
        const uint32_t crc_at = 2u + len, tail_at = crc_at + 4u, src_bits = (ns_sig * job.ndbps + 7u) / 8u * 8u;
        const uint32_t crc = __ldg(crcs + f);
        for (uint32_t i = lane; i < job.ndbps + 6u; i += 32) {
            const int j = (int)n0 - 6 + (int)i;
            uint32_t bit = 0;
            if (j >= 0 && (uint32_t)j < src_bits) {
                const uint32_t by = (uint32_t)j >> 3, bi = (uint32_t)j & 7u;
                uint32_t raw = 0;
                if (by >= 2u && by < crc_at) raw = pl[by - 2u]; else if (by >= crc_at && by < tail_at) raw = (crc >> (8u * (by - crc_at))) & 0xFFu;
                const uint32_t scr = phase == 255u ? 0u : __ldg(X.scr_seq + (phase + (uint32_t)j) % 127u);
                bit = ((raw >> bi) & 1u) ^ scr;
                if (by == tail_at && bi < 6u) bit = 0;                                    // TAIL_SCRAMBLE: code & 0xC0
            }
            sd[i] = (uint8_t)bit;
        }
    }
    __syncwarp();
    const uint32_t cr = sig ? (uint32_t)CR_12 : job.code_rate;
    const uint32_t cbase = sig ? 0u : (sym - 3u) * 104u * job.nbpsc;                     // index of this symbol's first coded bit in the frame
    auto coded = [&](uint32_t k) -> uint32_t {           // coded bit k of this symbol (both streams' bits interleaved), as in k_tx11a
        if (!sig && cbase + k >= coded_bits) return 0u;  // behind the encoder's last burst: the stream parser's pad bytes
        uint32_t n, isb;
        if (cr == CR_12) { n = k >> 1; isb = k & 1u; }
        else if (cr == CR_34) { const uint32_t g = k >> 2, r = k & 3u; n = 3u * g + (r == 3u ? 2u : r >> 1); isb = (r == 1u || r == 3u); }
        else { const uint32_t g = k / 3u, r = k - 3u * g; n = 2u * g + (r == 2u ? 1u : 0u); isb = r == 1u; }          // rate 2/3: A0 B0 A1 (conv_enc.hpp:102-188)
        const uint8_t* d = sd + 6 + n;
        return isb ? (d[0] ^ d[-1] ^ d[-2] ^ d[-3] ^ d[-6]) & 1u : (d[0] ^ d[-2] ^ d[-3] ^ d[-5] ^ d[-6]) & 1u;
    };
    if (sig) {
        // T11aInterleaveBPSK + TSigMap11n (L-SIG on I, HT-SIG on Q, +-30339) + T11aAddPilot<30339> (index 127, 0, 1)
#pragma unroll
        for (int w = 0; w < 2; w++) {
            const int dd = lane + 24 * w;
            if (lane < 24) {
                int bin = dd < 24 ? 38 + dd : dd - 24 + 1;
                if (dd < 24) { if (bin >= 43) bin++; if (bin >= 57) bin++; } else { if (bin >= 7) bin++; if (bin >= 21) bin++; }
                const int v = coded(__ldg(inv_deint + dd)) ? 30339 : -30339;
                xs[bin < 32 ? bin : bin + 64] = pack(sym == 0 ? mk(v, 0) : mk(0, v));
            }
        }
        if (lane == 24) {
            const uint32_t pi = sym == 0 ? 127u : sym - 1u;
            const int s = __ldg(T.pilot_neg + pi) ? -30339 : 30339;
            xs[7] = pack(mk(s, 0)); xs[21] = pack(mk(-s, 0)); xs[57 + 64] = pack(mk(s, 0)); xs[43 + 64] = pack(mk(s, 0));
        }
    } else {
        // stream parser (even coded bits -> stream 1, odd -> stream 2) + T11nInterleave*_S1/_S2 + mapper + T11nAddPilot<iss>
        const uint8_t* inv = N.inv + ((job.nbpsc == 1 ? 0 : 2) + iss) * 104;
#pragma unroll
        for (int w = 0; w < 2; w++) {
            const int dd = lane + 26 * w;               // data carrier 0..51 in T11nAddPilot order: -28..-1 then 1..28
            if (lane < 26) {
                int bin = dd < 26 ? 36 + dd : dd - 26 + 1;
                if (dd < 26) { if (bin >= 43) bin++; if (bin >= 57) bin++; } else { if (bin >= 7) bin++; if (bin >= 21) bin++; }
                cs16 c;
                if (job.nbpsc == 1) c = mk(coded(2u * __ldg(inv + dd) + iss) ? 30339 : -30339, 0);
                else if (job.nbpsc == 2) c = mk(coded(2u * __ldg(inv + 2 * dd) + iss) ? 21453 : -21453, coded(2u * __ldg(inv + 2 * dd + 1) + iss) ? 21453 : -21453);
                else {                                  // TMap11aQAM16<9594> / TMap11aQAM64<4681> (mapper11a.hpp:16-41): Gray level of the M bits, first on air = most significant
                    const uint32_t M = job.nbpsc >> 1;  // stream parser: M bits to stream 1, M to stream 2, in turn (_b_stream_parser.h:140-275)
                    const uint16_t* iv = N.inv16 + ((job.nbpsc == 6 ? 2 : 0) + iss) * 312 + dd * job.nbpsc;
                    int lv[2];
#pragma unroll
                    for (int a = 0; a < 2; a++) {
                        uint32_t g = 0;
                        for (uint32_t t = 0; t < M; t++) { const uint32_t m = __ldg(iv + a * M + t); g = (g << 1) | coded((2u * (m / M) + iss) * M + m % M); }
                        uint32_t bin = g; for (uint32_t sh = g >> 1; sh; sh >>= 1) bin ^= sh;
                        lv[a] = ((int)bin * 2 - ((1 << M) - 1)) * (M == 2 ? 9594 : 4681);
                    }
                    c = mk(lv[0], lv[1]);
                }
                xs[bin < 32 ? bin : bin + 64] = pack(c);
            }
        }
        if (lane == 26) {                               // _b_dot11_pilot.h:7-35: polarity entry (n + 3) % 127, pattern row n & 3
            const uint32_t n = sym - 3u;
            const int s = __ldg(T.pilot_neg + (n + 3u) % 127u) ? -30339 : 30339;
            // rows {1,1,-1,-1},{1,-1,-1,1} | {1,-1,-1,1},{-1,-1,1,1} | {-1,-1,1,1},{-1,1,1,-1} | {-1,1,1,-1},{1,1,-1,-1}: bit set = minus, carrier order -21, -7, 7, 21
            const unsigned NEGS = 0xC993366Cu;                  // nibble (row * 2 + stream), low one first: bits 0..3 = the four carriers
            const unsigned nib = (NEGS >> (4u * ((n & 3u) * 2u + iss))) & 0xFu;
            xs[43 + 64] = pack(mk((nib & 1u) ? -s : s, 0)); xs[57 + 64] = pack(mk((nib & 2u) ? -s : s, 0));
            xs[7] = pack(mk((nib & 4u) ? -s : s, 0)); xs[21] = pack(mk((nib & 8u) ? -s : s, 0));
        }
    }
    warp_ifft128(xs, X, lane);
    // ---- TCSD (stream 2: 2 vectors for the SIG symbols, 4 for DATA), TAddGI, store as COMPLEX16 ---------------------------------------------------
    const uint32_t shift = iss ? (sig ? 8u : 16u) : 0u;
    const uint32_t base = job.lead + 640u + (sig ? 160u * sym : 480u + 480u + 160u * (sym - 3u));
    if (sig && iss == 0) {                              // one spectrum, two antennas: the first stream's warp writes both
        for (uint32_t i = lane; i < 160u; i += 32) {
            const uint32_t t = i < 32u ? 96u + i : i - 32u;
            outs[0][base + i] = xs[rev7((int)t)];
            outs[1][base + i] = xs[rev7((int)((t + 128u - 8u) & 127u))];
        }
    } else if (!sig) {
        for (uint32_t i = lane; i < 160u; i += 32) {
            const uint32_t t = i < 32u ? 96u + i : i - 32u;
            outs[iss][base + i] = xs[rev7((int)((t + 128u - shift) & 127u))];
        }
    }
}

}  // namespace sb
