// ORACLE — TEST INFRASTRUCTURE ONLY (see ops.h).
// The reference's LEGACY 802.11a transmitter (BB11ATxFrameMod / BB11ATxBufferMod6M, kernel/bb/dot11a/dot11/atx_fe.c, atx_tpl_imp.h:5-58) as a
// whole, at SampleRate 40 or 44: what tx11a_legacy.cpp restates at 40 Msps (pinned there by usr/HwVeri/data/ofdm.bin and the legacy_tx
// vectors), plus the 40 -> 44 Msps upsampler, LENGTH 4096, the RCB zero padding and an FCS sent as it is.  The symbol stages are those of
// tx11a_legacy.cpp, stopped before Copy_NT so that the 16-bit symbol can be upsampled; at 40 Msps the two entry points agree sample for
// sample (tests/test_cpu_oracle_tx11a_legacy_tx.py).  Built on its own, with the oracle sources it needs, into
// oracle/libsora_oracle_tx11a44.so (oracle/tx11a_legacy44.mk).
#include "tx11a.h"
#include "rx11a.h"
#include <cstring>
#include <vector>

namespace sbo {

void tx11a_encode_bits(const std::vector<uint8_t>& bytes, int cr, std::vector<uint8_t>& coded);   // tx11a.cpp: rate-1/2 mother code + puncturing, one coded bit per byte

namespace {
struct LRate { uint32_t kbps; uint8_t code; int nbpsc; int cr; int ndbps; };
const LRate LR[8] = {{6000, 0xB, 1, CR_12, 24}, {9000, 0xF, 1, CR_34, 36}, {12000, 0xA, 2, CR_12, 48}, {18000, 0xE, 2, CR_34, 72},
                     {24000, 0x9, 4, CR_12, 96}, {36000, 0xD, 4, CR_34, 144}, {48000, 0x8, 6, CR_23, 192}, {54000, 0xC, 6, CR_34, 216}};
inline int16_t level(int nbpsc, int bin) {              // bin = Gray-decoded index 0 .. 2^(nbpsc/2) - 1, smallest = most negative
    static const int16_t L2[2] = {-7580, 7580}, L4[4] = {-10169, -3389, 3389, 10169}, L6[8] = {-11578, -8270, -4962, -1654, 1654, 4962, 8270, 11578};
    return nbpsc == 2 ? L2[bin] : nbpsc == 4 ? L4[bin] : L6[bin];
}
inline int16_t sat_add16(int a, int b) { int s = a + b; return (int16_t)(s > 32767 ? 32767 : s < -32768 ? -32768 : s); }
inline int8_t pack_nt(int16_t v) { int s = v >> 6; return (int8_t)(s > 127 ? 127 : s < -128 ? -128 : s); }

struct LegacyTx {
    c16 last[4];                                        // info->cWindow[0..3]
    // one OFDM symbol from ncbps coded bits (one per byte): interleave, map, pilots, IFFT64x, CopyGI, Window -> info->cSymbol, the 160
    // COMPLEX16 samples UpsampleAndCopyNT reads (the same stages as LegacyTx::symbol of tx11a_legacy.cpp, stopped before Copy_NT)
    void symbol16(const uint8_t* coded, int nbpsc, bool pilot_neg, c16* sym) {
        const Tables& T = tables();
        const int ncbps = 48 * nbpsc;
        const uint16_t* dm = nbpsc == 1 ? T.deint48 : nbpsc == 2 ? T.deint96 : nbpsc == 4 ? T.deint192 : T.deint288;
        uint8_t air[288];
        for (int k = 0; k < ncbps; k++) air[dm[k]] = coded[k];
        alignas(16) c16 f[64]; memset(f, 0, sizeof f);
        const int h = nbpsc / 2;
        auto lev = [&](const uint8_t* b) -> int16_t {                         // first bit on air is the most significant Gray bit
            int g = 0; for (int i = 0; i < h; i++) g = (g << 1) | b[i];
            int bin = 0, acc = 0; for (int i = h - 1; i >= 0; i--) { acc ^= (g >> i) & 1; bin = (bin << 1) | acc; }
            return level(nbpsc, bin);
        };
        int d = 0;
        for (int pass = 0; pass < 2; pass++)                                  // AddPilot's carrier order: -26..-1 then 1..26, pilots skipped
            for (int i = pass ? 1 : 38; i <= (pass ? 26 : 63); i++) {
                if (i == 43 || i == 57 || i == 7 || i == 21) continue;
                const uint8_t* b = air + d * nbpsc; d++;
                if (nbpsc == 1) { f[i].re = b[0] ? 10720 : -10720; f[i].im = 0; }
                else { f[i].re = lev(b); f[i].im = lev(b + h); }
            }
        const int16_t one = 32 * 335;                                         // OFDM_ONE
        const int s = pilot_neg ? -1 : 1;
        f[7].re = (int16_t)(s * one); f[21].re = (int16_t)(-s * one); f[57].re = (int16_t)(s * one); f[43].re = (int16_t)(s * one);
        alignas(16) c16 t[128], o[128];
        memset(t, 0, sizeof t); memcpy(t, f, 32 * sizeof(c16)); memcpy(t + 96, f + 32, 32 * sizeof(c16));
        ifft128((v128*)t, (v128*)o);
        for (int i = 0; i < 128; i++) { sym[32 + i].re = (int16_t)((uint16_t)o[i].re << 2); sym[32 + i].im = (int16_t)((uint16_t)o[i].im << 2); }   // psllw 2
        memcpy(sym, sym + 128, 32 * sizeof(c16));                             // CopyGI
        // Window
        sym[0].re >>= 2; sym[0].im >>= 2; sym[1].re >>= 1; sym[1].im >>= 1;
        sym[2].re = (int16_t)(sym[2].re - (sym[2].re >> 2)); sym[2].im = (int16_t)(sym[2].im - (sym[2].im >> 2));
        for (int i = 0; i < 4; i++) { sym[i].re = sat_add16(sym[i].re, last[i].re); sym[i].im = sat_add16(sym[i].im, last[i].im); }
        sym[0].re = (int16_t)(sym[0].re + last[0].re); sym[0].im = (int16_t)(sym[0].im + last[0].im);
        last[0].re = (int16_t)(sym[32].re - (sym[32].re >> 2)); last[0].im = (int16_t)(sym[32].im - (sym[32].im >> 2));
        last[1].re = (int16_t)(sym[33].re >> 1); last[1].im = (int16_t)(sym[33].im >> 1);
        last[2].re = (int16_t)(sym[34].re >> 2); last[2].im = (int16_t)(sym[34].im >> 2);
        last[3].re = last[3].im = 0;
    }
};
}

// ---- 40 -> 44 Msps: Upsample40MTo44M_160 / _3 (inc/bb/mod/upsample.h:44-144), lane for lane on SSE ------------------------------------
// compute_4 (upsample.h:44-62) on four input samples v:   m0 = mulhrs(v, row0[idx]), m1 = mulhrs(v, row1[idx]),
//   out = { resi[3] + m0[0], m1[0] + m1[1], m0[1] + m0[2], m1[2] + m1[3] },  resi = m0;
// mul_shift<15> = pmulhrsw (vector128.h:1252, rounds: SONE * x is not x for |x| > 16384), concat_extract<12> = palignr (:552),
// permutate<1,0,3,2> = pshufd (:688), add = paddw (:603, wraps), and / or with _ODD_MASK / _EVEN_MASK.  Coefficients S1(x) = x * 0x7fff / 11.
namespace {
inline int16_t up_s1(int x) { return (int16_t)(x * 0x7fff / 11); }
struct Up44 {
    v128 r0[3], r1[3];
    Up44() {
        static const int a0[3][4] = {{11, 2, 9, 4}, {7, 6, 5, 8}, {3, 10, 1, 0}}, a1[3][4] = {{1, 10, 3, 8}, {5, 6, 7, 4}, {9, 2, 0, 0}};   // g_coff1_row0 / _row1
        for (int i = 0; i < 3; i++) {
            r0[i] = _mm_setr_epi16(up_s1(a0[i][0]), up_s1(a0[i][0]), up_s1(a0[i][1]), up_s1(a0[i][1]), up_s1(a0[i][2]), up_s1(a0[i][2]), up_s1(a0[i][3]), up_s1(a0[i][3]));
            r1[i] = _mm_setr_epi16(up_s1(a1[i][0]), up_s1(a1[i][0]), up_s1(a1[i][1]), up_s1(a1[i][1]), up_s1(a1[i][2]), up_s1(a1[i][2]), up_s1(a1[i][3]), up_s1(a1[i][3]));
        }
    }
    v128 compute_4(v128 vin, v128& resi, int idx) const {
        const v128 odd = _mm_setr_epi16(-1, -1, 0, 0, -1, -1, 0, 0), even = _mm_setr_epi16(0, 0, -1, -1, 0, 0, -1, -1);
        v128 xx1 = _mm_mulhrs_epi16(vin, r0[idx]);
        const v128 xx3 = resi; resi = xx1;
        xx1 = _mm_alignr_epi8(xx1, xx3, 12);
        v128 xx2 = _mm_shuffle_epi32(xx1, _MM_SHUFFLE(2, 3, 0, 1));
        const v128 yy1 = _mm_and_si128(_mm_add_epi16(xx1, xx2), odd);
        xx1 = _mm_mulhrs_epi16(vin, r1[idx]);
        xx2 = _mm_shuffle_epi32(xx1, _MM_SHUFFLE(2, 3, 0, 1));
        const v128 yy2 = _mm_and_si128(_mm_add_epi16(xx1, xx2), even);
        return _mm_or_si128(yy1, yy2);
    }
    // reads in[0 .. 164): the last step loads in[160 .. 163] one vector past the 160 inputs, and in[160] enters output 175
    void up160(const c16* in, c16* out) const {
        const c16* pv = in; c16* po = out; v128 resi = _mm_setzero_si128(), rr1, vin, vin1;
        int idx = 0, cnt = 160;
        while (true) {
            vin = ld(pv + 4 * idx++); rr1 = compute_4(vin, resi, 0); st(po, rr1); po += 4;
            vin = ld(pv + 4 * idx++); rr1 = compute_4(vin, resi, 1); st(po, rr1); po += 4;
            vin = ld(pv + 4 * idx++); rr1 = compute_4(vin, resi, 2); st(po, rr1); po += 3;
            vin1 = ld(pv + 4 * idx++); vin = _mm_alignr_epi8(vin1, vin, 8); rr1 = compute_4(vin, resi, 0); st(po, rr1); po += 4;
            vin = vin1; vin1 = ld(pv + 4 * idx++); vin = _mm_alignr_epi8(vin1, vin, 8); rr1 = compute_4(vin, resi, 1); st(po, rr1); po += 4;
            vin = vin1; vin1 = ld(pv + 4 * idx); vin = _mm_alignr_epi8(vin1, vin, 8); rr1 = compute_4(vin, resi, 2);
            cnt -= 20;
            if (cnt == 0) break;
            st(po, rr1); po += 3;
        }
        alignas(16) c16 r[4]; st(r, rr1);
        *po++ = r[0]; *po++ = r[1]; *po++ = r[2];
    }
    void up3(const c16* in4, c16* out4) const { v128 resi = _mm_setzero_si128(); st(out4, compute_4(ld(in4), resi, 0)); }
};
const Up44& up44() { static const Up44 u; return u; }
}

// The whole of BB11ATxFrameMod / BB11ATxBufferMod6M at SampleRate 40 or 44 (atx_tpl_imp.h:5-58, ofdmsymbol.h:48-94, atx_tpl.h:69-83):
//   * 44: every 160-sample chunk (the four preamble chunks, SIGNAL, each data symbol) is upsampled afresh into 176, then Copy_NT; the
//     over-read sample in[160] is the next preamble chunk's first sample for preamble chunks 0-2, zero for chunk 3 (past PREAMBLE40_11A_LUT,
//     which the reference does not define; DESIGN.md §1), and for SIGNAL / data the first 44 Msps output of the same symbol: cSymbol[160]
//     is cSymbol44M[0] in BB11A_TX_VECTOR (bba.h:161-165), which the first store of the same call has just written.  The tail is
//     Upsample40MTo44M_3 over cWindow, four zero samples, Copy_NT of 8.
//   * LENGTH = len (+ 4 with append_crc) may be 4096, which atx_fe.c:23 admits and GetSignal shifts into the parity bit (atx.h:78-97).
//   * the signal, (640 + 160 (1 + nsym)) (x 11/10 at 44) + 8 samples, is zero padded to a multiple of 128 bytes = 64 samples
//     (ALIGN_WITH_RCB_BUFFER_PADDING_ZERO, core/inc/_tx_manager2.h:29-38).
// Returns the padded sample count (0: bad rate / sample rate / length, or cap too small); *signal_samples = the samples before the padding.
static size_t modulate_ex(const uint8_t* mpdu, uint32_t len, int append_crc, uint32_t rate_kbps, uint32_t sample_rate, const c16* preamble640,
                                int8_t* out, size_t cap, size_t* signal_samples) {
    const LRate* ri = nullptr; for (auto& r : LR) if (r.kbps == rate_kbps) ri = &r;
    if (!ri || (!mpdu && len) || !preamble640 || (sample_rate != 40 && sample_rate != 44)) return 0;
    const Tables& T = tables();
    const uint32_t L = len + (append_crc ? 4u : 0u);
    if (L > 4096u) return 0;
    const uint32_t nsym = (22u + 8u * L + (uint32_t)ri->ndbps - 1u) / (uint32_t)ri->ndbps;
    const size_t chunk = sample_rate == 44 ? 176 : 160;
    const size_t sig = chunk * (4 + 1 + (size_t)nsym) + 8, total = (sig + 63) & ~(size_t)63;
    if (total > cap) return 0;
    if (signal_samples) *signal_samples = sig;
    const Up44& U = up44();
    alignas(16) c16 buf[160 + 177 + 3];                 // cSymbol[160] immediately followed by cSymbol44M[176 + 1], as in BB11A_TX_VECTOR
    c16* const s40 = buf; c16* const s44 = buf + 160;
    int8_t* o = out;
    auto emit = [&](const c16* x, size_t n) { for (size_t i = 0; i < n; i++) { o[2 * i] = pack_nt(x[i].re); o[2 * i + 1] = pack_nt(x[i].im); } o += 2 * n; };
    auto chunk_out = [&](const c16* in164) {            // UpsampleAndCopyNT of one 160-sample chunk
        if (sample_rate == 44) { U.up160(in164, s44); emit(s44, 176); } else emit(in164, 160);
    };
    {   alignas(16) c16 pre[640 + 4]; memcpy(pre, preamble640, 640 * sizeof(c16)); memset(pre + 640, 0, 4 * sizeof(c16));
        for (int c = 0; c < 4; c++) chunk_out(pre + 160 * c); }                               // CopyPreamble16_NT
    LegacyTx tx;
    const c16* pt = preamble640 + 512;
    tx.last[0].re = (int16_t)(pt[0].re - (pt[0].re >> 2)); tx.last[0].im = (int16_t)(pt[0].im - (pt[0].im >> 2));
    tx.last[1].re = (int16_t)(pt[1].re >> 1); tx.last[1].im = (int16_t)(pt[1].im >> 1);
    tx.last[2].re = (int16_t)(pt[2].re >> 2); tx.last[2].im = (int16_t)(pt[2].im >> 2);
    tx.last[3].re = tx.last[3].im = 0;
    memset(s44, 0, 177 * sizeof(c16));
    {   uint32_t sg = ri->code | (L << 5);                                                   // GetSignal: L = 4096 lands on bit 17
        uint32_t p = sg ^ (sg >> 16); p ^= p >> 8; p ^= p >> 4; p ^= p >> 2; p ^= p >> 1; sg |= (p & 1u) << 17;
        std::vector<uint8_t> b = {(uint8_t)sg, (uint8_t)(sg >> 8), (uint8_t)(sg >> 16)}, coded;
        tx11a_encode_bits(b, CR_12, coded);
        tx.symbol16(coded.data(), 1, false, s40); chunk_out(s40);
    }
    const uint32_t nbytes = (nsym * (uint32_t)ri->ndbps + 7u) / 8u;
    std::vector<uint8_t> data(nbytes + 8, 0);
    if (len) memcpy(data.data() + 2, mpdu, len);
    if (append_crc) { uint32_t crc = 0xFFFFFFFFu; for (uint32_t i = 0; i < len; i++) crc = (crc >> 8) ^ T.crc32_lut[mpdu[i] ^ (crc & 0xFF)]; crc = ~crc; memcpy(data.data() + 2 + len, &crc, 4); }
    uint8_t reg = 0xFF;
    for (uint32_t i = 0; i < nbytes; i++) {
        reg = T.scramble_lut[reg >> 1];
        data[i] = (uint8_t)(data[i] ^ reg);
        if (i == 2 + L) data[i] &= 0xC0;
    }
    data.resize(nbytes);
    std::vector<uint8_t> coded; tx11a_encode_bits(data, ri->cr, coded);
    const int ncbps = 48 * ri->nbpsc;
    coded.resize((size_t)nsym * ncbps + 8, 0);
    unsigned st7 = 0x7F; uint8_t seq[127], pneg[127];
    for (int i = 0; i < 127; i++) { unsigned b = ((st7 >> 6) ^ (st7 >> 3)) & 1; st7 = ((st7 << 1) | b) & 0x7F; seq[i] = (uint8_t)b; }
    for (int i = 0; i < 127; i++) pneg[i] = seq[(i + 1) % 127];                           // lutst/pilotsgn.c: entry i = p_{i+1}
    for (uint32_t s = 0; s < nsym; s++) { tx.symbol16(coded.data() + (size_t)s * ncbps, ri->nbpsc, pneg[s % 127] != 0, s40); chunk_out(s40); }
    if (sample_rate == 44) {                                                                 // UpsampleTailAndCopyNT
        alignas(16) c16 w[8]; memcpy(w, tx.last, 4 * sizeof(c16)); memset(w + 4, 0, 4 * sizeof(c16));
        U.up3(w, w); emit(w, 8);
    } else { alignas(16) c16 w[8]; memcpy(w, tx.last, 4 * sizeof(c16)); memset(w + 4, 0, 4 * sizeof(c16)); emit(w, 8); }
    memset(o, 0, 2 * (total - sig));
    return total;
}

} // namespace sbo

extern "C" {
// the whole transmitter: returns the padded sample count (0: bad rate / sample rate / length, or cap too small)
uint64_t sbo_tx11a_legacy_modulate_ex(const uint8_t* mpdu, uint32_t len, int append_crc, uint32_t rate_kbps, uint32_t sample_rate, const int16_t* preamble640,
                                      int8_t* out, uint64_t cap_samples, uint64_t* signal_samples) {
    size_t sig = 0;
    const size_t n = sbo::modulate_ex(mpdu, len, append_crc, rate_kbps, sample_rate, (const sbo::c16*)preamble640, out, (size_t)cap_samples, &sig);
    if (signal_samples) *signal_samples = sig;
    return n;
}
// Upsample40MTo44M_160: reads in[0 .. 164);  Upsample40MTo44M_3
void sbo_tx11a_legacy_upsample44_160(const int16_t* in164, int16_t* out176) { sbo::up44().up160((const sbo::c16*)in164, (sbo::c16*)out176); }
void sbo_tx11a_legacy_upsample44_3(const int16_t* in4, int16_t* out4) { sbo::up44().up3((const sbo::c16*)in4, (sbo::c16*)out4); }
}
