// sora_b200 — the legacy 802.11a transmitter on the device (sm_90a): BB11ATxFrameMod / BB11ATxBufferMod6M (kernel/bb/dot11a/dot11/atx_fe.c,
// atx_tpl_imp.h:5-58) at SampleRate 40 or 44, the reference's other 802.11a modulator next to the brick one of tx11a_kernels.cuh.
//
//   k_tx11a_legacy   one warp per run of SB_TXL_RUN consecutive OFDM symbols of one frame (symbol 0 = SIGNAL), plus helper warps per frame
//                    for the preamble and the zero fill.  Per symbol: the scrambled bits (the scrambler as a 127-periodic sequence from the
//                    0xFF state, atx_tpl.h:18, the encoder state as the six scrambled bits in front of the symbol) -> puncturing -> the
//                    interleaver -> the lutst/mapa_* levels -> pilots +-10720 (PILOTSGN; SIGNAL polarity 0) -> IFFT64x (the zero-stuffed
//                    IFFT<128> of tx11a_kernels.cuh, then a wrapping << 2, ifft64x.h:6-24) -> CopyGI -> Window (ofdmsymbol.h:19-46) ->
//                    UpsampleAndCopyNT (ofdmsymbol.h:48-75).
//   The one dependency between symbols is the Window's carry: three samples of symbol k-1 (3/4, 1/2, 1/4 of its samples 32..34, taken
//   before symbol k-1's own window touches its samples 0..3) are saturating-added into samples 0..3 of symbol k, and the first once more
//   with a plain 16-bit add.  A run carries it in registers and computes the symbol in front of it once more for the first carry; the
//   preamble seeds the carry of SIGNAL from its samples 512..514.
//   At 44 Msps every 160-sample chunk is upsampled afresh into 176 (Upsample40MTo44M_160, inc/bb/mod/upsample.h:85-144).  Output k = 11 h + s
//   of a chunk x is  s == 0: M(x[10 h], 11),  else M(x[10 h + s - 1], s) + M(x[10 h + s], 11 - s)  (16-bit wrap), M(v, a) = pmulhrsw(v,
//   a * 0x7fff / 11).  Output 175 reads x[160], one sample behind the chunk: for SIGNAL and data symbols that is cSymbol44M[0] in
//   BB11A_TX_VECTOR (bba.h:161-165), the chunk's own first 44 Msps output; for preamble chunks 0-2 the next chunk's first sample; for
//   chunk 3 zero (DESIGN.md §1).  Copy_NT: >> 6, saturated to int8 (copynt.h:16-26).
//   Frame slot: preamble (640 | 704), SIGNAL and data symbols (160 | 176 each), the 8-sample tail (the last carry, at 44 through
//   Upsample40MTo44M_3, then four zeros), zeros to the end of the slot.  Every store is 16 bytes (eight COMPLEX8 samples).
#pragma once
#include "tx11a_kernels.cuh"
#include "tx_frames.cuh"

namespace sb {

struct Tx11aLegacyJob {
    uint32_t rate_code, nbpsc, code_rate, ndbps;    // SIGNAL rate bits, N_BPSC, CR_*, N_DBPS
    uint32_t sr44;                                  // 0: 40 Msps, 1: 44 Msps
    uint32_t fcs_in_payload;                        // 1: the payload's last four bytes are the FCS; 0: CRC-32 appended
    uint32_t runs;                                  // symbol warps per frame (the rest of the frame's warps are helpers)
};

#define SB_TXL_WARPS 4
#ifndef SB_TXL_RUN
#define SB_TXL_RUN 8
#endif

__constant__ short c_txl_lev[14] = {-7580, 7580, -10169, -3389, 3389, 10169, -11578, -8270, -4962, -1654, 1654, 4962, 8270, 11578};   // lutst/mapa_*.c

__device__ __forceinline__ int txl_mulhrs(int x, int a) { return (x * ((a * 0x7fff) / 11) + 16384) >> 15; }   // pmulhrsw by S1(a), a in 0 .. 11
// output k (0 .. 175) of Upsample40MTo44M_160 over the chunk read through in(i), i in 0 .. 160
template <class In> __device__ __forceinline__ cs16 txl_up44(const In& in, int k) {
    const int h = k / 11, s = k - 11 * h, b = 10 * h;
    if (s == 0) { const cs16 x = in(b); return mk(txl_mulhrs(x.re, 11), txl_mulhrs(x.im, 11)); }
    const cs16 x = in(b + s - 1), y = in(b + s);
    return mk(sx16(txl_mulhrs(x.re, s) + txl_mulhrs(y.re, 11 - s)), sx16(txl_mulhrs(x.im, s) + txl_mulhrs(y.im, 11 - s)));
}
__device__ __forceinline__ uint32_t txl_pack2(cs16 a, cs16 b) {   // two samples through Copy_NT (psraw 6, packsswb)
    const uint32_t ar = (uint32_t)pack8s(a.re >> 6) & 0xFFu, ai = (uint32_t)pack8s(a.im >> 6) & 0xFFu;
    const uint32_t br = (uint32_t)pack8s(b.re >> 6) & 0xFFu, bi = (uint32_t)pack8s(b.im >> 6) & 0xFFu;
    return ar | (ai << 8) | (br << 16) | (bi << 24);
}
template <class Get> __device__ __forceinline__ uint4 txl_pack8(const Get& g) {
    return make_uint4(txl_pack2(g(0), g(1)), txl_pack2(g(2), g(3)), txl_pack2(g(4), g(5)), txl_pack2(g(6), g(7)));
}

__global__ void __launch_bounds__(32 * SB_TXL_WARPS) k_tx11a_legacy(const uint8_t* __restrict__ payload, const uint64_t* __restrict__ pay_off,
        const uint32_t* __restrict__ pay_len, uint32_t nframes, Tx11aLegacyJob job, DevTables T, DevTablesTx X, const uint16_t* __restrict__ inv_deint,
        const uint32_t* __restrict__ crcs, const uint32_t* __restrict__ pre, int8_t* __restrict__ out, uint64_t out_stride /*samples per slot*/,
        uint32_t* __restrict__ nsamples) {
    __shared__ uint32_t s_x[SB_TXL_WARPS][128];
    __shared__ uint32_t s_w[SB_TXL_WARPS][164];            // the windowed symbol (cSymbol) and, at 44 Msps, the over-read sample behind it
    __shared__ uint8_t s_d[SB_TXL_WARPS][232];             // scrambled data bits of the symbol, six bits of history in front
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const uint32_t f = blockIdx.x;
    const uint32_t w = blockIdx.y * SB_TXL_WARPS + wib;
    if (f >= nframes) return;
    const uint32_t len = pay_len[f], L = job.fcs_in_payload ? len : len + 4u;
    const uint32_t nsym = tx11a_legacy_nsym(L, job.ndbps);
    const uint32_t chunk = job.sr44 ? 176u : 160u, sig_end = tx11a_legacy_signal(nsym, job.sr44), padded = tx11a_legacy_padded(nsym, job.sr44);
    uint4* slot = (uint4*)(out + (size_t)f * out_stride * 2u);          // 8 samples per uint4
    if ((uint64_t)padded > out_stride) return;                          // the host checked this; never write outside the slot
    if (w >= job.runs) {                                                // helper warps: preamble, then zeros from the tail's end to the slot's end
        const uint32_t helper = w - job.runs, nhelp = gridDim.y * SB_TXL_WARPS - job.runs;
        if (helper == 0 && lane == 0 && nsamples) nsamples[f] = padded;
        const uint32_t npre = chunk / 2u, z0 = sig_end / 8u, nz = (uint32_t)(out_stride / 8u) - z0;
        for (uint32_t q = helper * 32u + lane; q < npre + nz; q += nhelp * 32u) {
            if (q >= npre) { slot[z0 + (q - npre)] = make_uint4(0, 0, 0, 0); continue; }
            if (!job.sr44) { slot[q] = txl_pack8([&](int j) { return unpack(__ldg(pre + 8u * q + j)); }); continue; }
            const uint32_t c = q / 22u, k0 = 8u * (q - 22u * c);
            const auto in = [&](int i) { return i < 160 ? unpack(__ldg(pre + 160u * c + i)) : (c < 3u ? unpack(__ldg(pre + 160u * (c + 1u))) : mk(0, 0)); };
            slot[q] = txl_pack8([&](int j) { return txl_up44(in, (int)k0 + j); });
        }
        return;
    }
    const uint32_t s_first = w * SB_TXL_RUN;
    if (s_first > nsym) return;
    const uint32_t s_last = s_first + SB_TXL_RUN - 1u < nsym ? s_first + SB_TXL_RUN - 1u : nsym;
    uint32_t* xs = s_x[wib]; uint32_t* ws = s_w[wib]; uint8_t* sd = s_d[wib];
    const uint8_t* pl = payload + pay_off[f];
    const uint32_t crc = job.fcs_in_payload ? 0u : __ldg(crcs + f);
    const uint32_t phase = __ldg(X.scr_phase + 0x7Fu);                 // Scramble11a: bReg = 0xFF, no random seed (atx_tpl.h:18)
    const uint16_t* inv = inv_deint + (job.nbpsc == 1 ? 0 : job.nbpsc == 2 ? 48 : job.nbpsc == 4 ? 144 : 336);   // air position -> coded index
    // IFFT64x of symbol `sym` into xs (slot rev7(i) holds time sample i, before the << 2)
    auto ifft_symbol = [&](uint32_t sym) {
        const uint32_t nd = sym == 0 ? 24u : job.ndbps, nbpsc = sym == 0 ? 1u : job.nbpsc, cr = sym == 0 ? (uint32_t)CR_12 : job.code_rate;
        const uint32_t n0 = sym == 0 ? 0u : (sym - 1u) * job.ndbps;
        __syncwarp();
        if (sym == 0) signal_bits(sd, sig_parity(job.rate_code | (L << 5)), lane);        // GetSignal (atx.h:78-97): LENGTH 4096 lands on the parity bit
        else scrambled_bits(sd, n0, nd, pl, 2u + len, 2u + L, crc, phase, X, lane);          // the six tail bits, not scrambled (atx_tpl.h:52)
        __syncwarp();
        const uint16_t* iv = sym == 0 ? inv_deint : inv;
        const int lev0 = nbpsc == 2 ? 0 : nbpsc == 4 ? 2 : 6;
        auto level = [&](uint32_t p0, uint32_t m) -> int {             // Gray-decoded bin, first bit on air = most significant
            uint32_t bin = 0, acc = 0;
            for (uint32_t i = 0; i < m; i++) { acc ^= coded_bit(sd, cr, __ldg(iv + p0 + i)); bin = (bin << 1) | acc; }
            return c_txl_lev[lev0 + bin];
        };
        for (int i = lane; i < 128; i += 32) xs[i] = 0;
        __syncwarp();
#pragma unroll
        for (int h = 0; h < 2; h++) {                                   // AddPilot's carrier order: -26..-1, then 1..26
            const int dd = lane + 24 * h;
            if (lane < 24) {
                cs16 c;
                if (nbpsc == 1) c = mk(coded_bit(sd, cr, __ldg(iv + dd)) ? 10720 : -10720, 0);
                else { const uint32_t hb = nbpsc >> 1; c = mk(level((uint32_t)dd * nbpsc, hb), level((uint32_t)dd * nbpsc + hb, hb)); }
                xs[carrier_slot(dd, 24)] = pack(c);
            }
        }
        if (lane == 24) pilots11a(xs, T, sym, 10720);
        warp_ifft128(xs, X, lane);
    };
    auto raw = [&](int t) { const cs16 v = unpack(xs[rev7(t)]); return mk(sx16(v.re << 2), sx16(v.im << 2)); };   // psllw 2, wraps
    cs16 last0, last1, last2;                                           // info->cWindow[0..2] ([3] stays zero)
    auto carry_from = [&](cs16 a, cs16 b, cs16 c) {
        last0 = mk(sx16(a.re - (a.re >> 2)), sx16(a.im - (a.im >> 2))); last1 = sra(b, 1); last2 = sra(c, 2);
    };
    if (s_first == 0) carry_from(unpack(__ldg(pre + 512)), unpack(__ldg(pre + 513)), unpack(__ldg(pre + 514)));   // CopyPreamble16_NT
    else { ifft_symbol(s_first - 1u); carry_from(raw(0), raw(1), raw(2)); }
    for (uint32_t sym = s_first; sym <= s_last; sym++) {
        ifft_symbol(sym);
        for (int i = lane; i < 160; i += 32) {                          // CopyGI + Window
            cs16 v = raw((int)gi_sample(i));
            if (i < 4) {
                if (i == 0) v = sra(v, 2); else if (i == 1) v = sra(v, 1); else if (i == 2) v = mk(sx16(v.re - (v.re >> 2)), sx16(v.im - (v.im >> 2)));
                const cs16 l = i == 0 ? last0 : i == 1 ? last1 : i == 2 ? last2 : mk(0, 0);
                v = adds(v, l);
                if (i == 0) v = mk(sx16(v.re + last0.re), sx16(v.im + last0.im));
            }
            ws[i] = pack(v);
        }
        carry_from(raw(0), raw(1), raw(2));
        __syncwarp();
        uint4* o = slot + (size_t)(4u + sym) * (chunk / 8u);
        if (!job.sr44) {
            if (lane < 20) o[lane] = txl_pack8([&](int j) { return unpack(ws[8 * lane + j]); });
        } else {
            if (lane == 0) { const cs16 x = unpack(ws[0]); ws[160] = pack(mk(txl_mulhrs(x.re, 11), txl_mulhrs(x.im, 11))); }   // cSymbol[160] = cSymbol44M[0]
            __syncwarp();
            const auto in = [&](int i) { return unpack(ws[i]); };
            if (lane < 22) o[lane] = txl_pack8([&](int j) { return txl_up44(in, 8 * lane + j); });
        }
        if (sym == nsym && lane == 0) {                                 // UpsampleTailAndCopyNT: the last carry, four zeros
            const cs16 t[4] = {last0, last1, last2, mk(0, 0)};
            const auto in = [&](int i) { return i < 4 ? t[i] : mk(0, 0); };
            slot[sig_end / 8u - 1u] = txl_pack8([&](int j) { return j >= 4 ? mk(0, 0) : job.sr44 ? txl_up44(in, j) : t[j]; });
        }
    }
}

} // namespace sb
