// ORACLE — TEST INFRASTRUCTURE ONLY (see ops.h).  802.11a transmit restatement; see tx11a.h.
#include "tx11a.h"
#include "rx11a.h"
#include <cstring>
#include <vector>

namespace sbo {

void tx11a_encode_bits(const std::vector<uint8_t>& bytes, int cr, std::vector<uint8_t>& coded);

static const int16_t BPSK_MOD = 10720;                                  // mapper11a.hpp:8-11
static inline int16_t kmod_of(int nbpsc) { return nbpsc == 1 ? BPSK_MOD : nbpsc == 2 ? (int16_t)(BPSK_MOD / 1.414) : nbpsc == 4 ? (int16_t)(BPSK_MOD / 3.162) : (int16_t)(BPSK_MOD / 6.481); }

struct RateInfo { uint32_t kbps; uint8_t code; int nbpsc; int cr; int ndbps; };
static const RateInfo RATES[8] = {{6000, 0xB, 1, CR_12, 24}, {9000, 0xF, 1, CR_34, 36}, {12000, 0xA, 2, CR_12, 48}, {18000, 0xE, 2, CR_34, 72},
                                  {24000, 0x9, 4, CR_12, 96}, {36000, 0xD, 4, CR_34, 144}, {48000, 0x8, 6, CR_23, 192}, {54000, 0xC, 6, CR_34, 216}};
static const RateInfo* rate_info(uint32_t kbps) { for (auto& r : RATES) if (r.kbps == kbps) return &r; return nullptr; }

// IFFTx of one 64-carrier symbol: zero-stuffed IFFT<128>, >> 4, 32-sample GI, window (fft.hpp:9-60)
void tx11a_ifftx(const c16* f64, c16* out160) {
    alignas(16) c16 t[128], o[128];
    memset(t, 0, sizeof t); memcpy(t, f64, 32 * sizeof(c16)); memcpy(t + 96, f64 + 32, 32 * sizeof(c16));
    ifft128((v128*)t, (v128*)o);
    for (int i = 0; i < 128; i++) { out160[32 + i].re = (int16_t)(o[i].re >> 4); out160[32 + i].im = (int16_t)(o[i].im >> 4); }
    memcpy(out160, out160 + 128, 32 * sizeof(c16));
    for (int i : {0, 1, 158, 159}) { out160[i].re >>= 1; out160[i].im >>= 1; }
}
static inline int8_t pack8(int16_t v) { return (int8_t)(v > 127 ? 127 : v < -128 ? -128 : v); }   // TPackSample16to8: packsswb (stdbrick.hpp:413-445)
void tx11a_pack8(const c16* in, size_t n, int8_t* out) { for (size_t i = 0; i < n; i++) { out[2 * i] = pack8(in[i].re); out[2 * i + 1] = pack8(in[i].im); } }

void tx11a_preamble16(c16* lut) {
    alignas(16) c16 t[128], o[128];
    const int16_t sts = (int16_t)(uint16_t)(1.0 * BPSK_MOD * 1.472), lts = BPSK_MOD;
    memset(t, 0, sizeof t);
    auto set = [&](int k, int s) { t[k].re = t[k].im = (int16_t)(s * sts); };
    set(4, -1); set(8, -1); set(12, 1); set(16, 1); set(20, 1); set(24, 1); set(104, 1); set(108, -1); set(112, 1); set(116, -1); set(120, -1); set(124, 1);
    ifft128((v128*)t, (v128*)o);
    for (int i = 0; i < 128; i++) { lut[i].re = (int16_t)(o[i].re >> 4); lut[i].im = (int16_t)(o[i].im >> 4); }
    for (int i = 128; i < 320; i++) lut[i] = lut[i - 128];                                  // forward overlapping copy = periodic extension
    for (int i : {0, 1, 318, 319}) { lut[i].re >>= 1; lut[i].im >>= 1; }
    memset(t, 0, sizeof t);
    static const int8_t L[53] = {1,1,-1,-1,1,1,-1,1,-1,1,1,1,1,1,1,-1,-1,1,1,-1,1,-1,1,1,1,1,0,
                                 1,-1,-1,1,1,-1,1,-1,1,-1,-1,-1,-1,-1,1,1,-1,-1,1,-1,1,-1,1,1,1,1};
    for (int k = 1; k <= 26; k++) { t[k].re = (int16_t)(L[k + 26] > 0 ? lts : -lts); t[128 - k].re = (int16_t)(L[26 - k] > 0 ? lts : -lts); }
    ifft128((v128*)t, (v128*)o);
    for (int i = 0; i < 128; i++) { lut[384 + i].re = (int16_t)(o[i].re >> 4); lut[384 + i].im = (int16_t)(o[i].im >> 4); }
    memcpy(lut + 512, lut + 384, 128 * sizeof(c16));
    memcpy(lut + 320, lut + 576, 64 * sizeof(c16));                                          // GI2
    for (int i : {320, 321, 638, 639}) { lut[i].re >>= 1; lut[i].im >>= 1; }
}

uint32_t tx11a_nsym(uint32_t len, uint32_t rate_kbps) {
    const RateInfo* ri = rate_info(rate_kbps); if (!ri) return 0;
    const uint32_t nd = rate_kbps == 9000 ? 2u * ri->ndbps : (uint32_t)ri->ndbps;
    const uint32_t dbytes = 2u + (len + 4u) + 1u, bits = dbytes * 8u;
    const uint32_t padded = (bits + nd - 1u) / nd * nd;
    return (bits + ((padded - bits + 7u) / 8u) * 8u) / ri->ndbps;
}

// T11Interleave (interleave.hpp:16-96): coded bit k of the symbol goes on air at deint[k]; one bit per byte both sides
void tx11a_interleave(const uint8_t* coded, int nbpsc, uint8_t* air) {
    const Tables& T = tables();
    const uint16_t* dm = nbpsc == 1 ? T.deint48 : nbpsc == 2 ? T.deint96 : nbpsc == 4 ? T.deint192 : T.deint288;
    for (int k = 0; k < 48 * nbpsc; k++) air[dm[k]] = coded[k];
}

// TMap11a* (mapper11a.hpp:13-298): 48 * nbpsc air bits -> 48 points.  Levels are (2b - (2^m - 1)) * kmod with the Gray code read first bit
// most significant (InitQamMapLut: bit-reverse, Gray -> binary)
void tx11a_map(const uint8_t* air, int nbpsc, c16* d48) {
    const int16_t km = kmod_of(nbpsc); const int h = nbpsc / 2;
    auto level = [&](const uint8_t* b, int m) -> int16_t {
        int g = 0; for (int i = 0; i < m; i++) g = (g << 1) | b[i];
        int bin = 0, acc = 0; for (int i = m - 1; i >= 0; i--) { acc ^= (g >> i) & 1; bin = (bin << 1) | acc; }
        return (int16_t)((2 * bin - ((1 << m) - 1)) * km);
    };
    for (int d = 0; d < 48; d++) {
        const uint8_t* b = air + d * nbpsc;
        if (nbpsc == 1) { d48[d].re = b[0] ? BPSK_MOD : (int16_t)-BPSK_MOD; d48[d].im = 0; }
        else { d48[d].re = level(b, h); d48[d].im = level(b + h, h); }
    }
}

// T11aAddPilot<> (pilot.hpp:10-119): data on carriers 38..63 then 1..26 around the pilots, pilots by PilotSgn[pilot_index], then the index
// advances (wrapping 127 -> 0 past 126); DC and the guard carriers stay 0
void tx11a_add_pilot(const c16* d48, unsigned& pilot_index, c16* f64) {
    memset(f64, 0, 64 * sizeof(c16));
    int d = 0;
    for (int pass = 0; pass < 2; pass++)
        for (int i = pass ? 1 : 38; i <= (pass ? 26 : 63); i++) {
            if (i == 43 || i == 57 || i == 7 || i == 21) continue;
            f64[i] = d48[d++];
        }
    static const uint8_t* neg = nullptr; static uint8_t negtab[128];
    if (!neg) { unsigned st = 0x7F; uint8_t seq[127]; for (int i = 0; i < 127; i++) { unsigned o = ((st >> 6) ^ (st >> 3)) & 1; st = ((st << 1) | o) & 0x7F; seq[i] = (uint8_t)o; }
                for (int i = 0; i < 127; i++) negtab[i] = seq[(i + 1) % 127]; negtab[127] = 0; neg = negtab; }   // PilotSgn (pilot.hpp:10-28): [i] = p_{i+1}, [127] = SIGNAL
    const int s = neg[pilot_index] ? -1 : 1;
    f64[7].re = (int16_t)(s * BPSK_MOD); f64[21].re = (int16_t)(-s * BPSK_MOD); f64[57].re = (int16_t)(s * BPSK_MOD); f64[43].re = (int16_t)(s * BPSK_MOD);
    pilot_index++; if (pilot_index >= 127) pilot_index = 0;
}

// one OFDM symbol worth of coded bits -> 160 samples: the stages above, TIFFTx, TPackSample16to8
static void symbol_out(const uint8_t* coded /*ncbps bits, one per byte*/, int nbpsc, unsigned& pilot_index, int8_t* out) {
    uint8_t air[288]; c16 d[48], f[64], td[160];
    tx11a_interleave(coded, nbpsc, air);
    tx11a_map(air, nbpsc, d);
    tx11a_add_pilot(d, pilot_index, f);
    tx11a_ifftx(f, td);
    tx11a_pack8(td, 160, out);
}

// T11aSc (scramble.hpp:170-262): per byte, ctrl 0 passes it (NO_SCRAMBLE), 1 steps the register and XORs (DO_SCRAMBLE), anything else
// steps, XORs and keeps the top two bits (TAIL_SCRAMBLE: the six tail bits leave the encoder as zeros)
void tx11a_scramble(const uint8_t* in, const uint8_t* ctrl, size_t n, uint8_t& reg, uint8_t* out) {
    const Tables& T = tables();
    for (size_t i = 0; i < n; i++) {
        if (ctrl[i] == 0) { out[i] = in[i]; continue; }
        reg = T.scramble_lut[reg >> 1];
        out[i] = (uint8_t)(in[i] ^ reg);
        if (ctrl[i] != 1) out[i] &= 0xC0;
    }
}

// rate-1/2 mother code, bits LSB first, then puncturing (conv_enc.hpp:5-280): returns coded bits, one per byte
void tx11a_encode_bits(const std::vector<uint8_t>& bytes, int cr, std::vector<uint8_t>& coded) {
    unsigned s = 0; coded.clear();
    size_t n = bytes.size() * 8;
    for (size_t i = 0; i < n; i++) {
        const unsigned x = (bytes[i >> 3] >> (i & 7)) & 1;
        const unsigned a = (x ^ (s >> 4) ^ (s >> 3) ^ (s >> 1) ^ s) & 1, b = (x ^ s ^ (s >> 3) ^ (s >> 4) ^ (s >> 5)) & 1;
        s = (s >> 1) | (x << 5);
        const size_t ph = cr == CR_34 ? i % 3 : cr == CR_23 ? i % 2 : 0;
        if (cr == CR_12) { coded.push_back((uint8_t)a); coded.push_back((uint8_t)b); }
        else if (cr == CR_34) { if (ph == 0) { coded.push_back((uint8_t)a); coded.push_back((uint8_t)b); } else if (ph == 1) coded.push_back((uint8_t)a); else coded.push_back((uint8_t)b); }
        else { if (ph == 0) { coded.push_back((uint8_t)a); coded.push_back((uint8_t)b); } else coded.push_back((uint8_t)a); }
    }
}

size_t tx11a_modulate(const uint8_t* payload, uint32_t len, uint32_t rate_kbps, uint8_t sc_seed, int8_t* out, size_t cap, uint32_t tail_zeros) {
    const RateInfo* ri = rate_info(rate_kbps);
    if (!ri || !payload || len + 4u > 4095u) return 0;
    const Tables& T = tables();
    const uint32_t nsym = tx11a_nsym(len, rate_kbps);
    const size_t total = 640 + 160 * (size_t)(1 + nsym) + tail_zeros;
    if (total > cap) return 0;
    // preamble through the 16 -> 8 bit pack
    c16 pre[640]; tx11a_preamble16(pre);
    tx11a_pack8(pre, 640, out);
    unsigned pilot_index = 127;
    // SIGNAL: rate code, reserved, LENGTH (incl. FCS), even parity, 6 tail bits; never scrambled, always 6 Mbps (ieee80211a_cmn.h B11aGetPLCPSignal)
    {
        uint32_t sig = ri->code | ((len + 4u) << 5);
        uint32_t p = sig ^ (sig >> 16); p ^= p >> 8; p ^= p >> 4; p ^= p >> 2; p ^= p >> 1; sig |= (p & 1u) << 17;
        std::vector<uint8_t> b = {(uint8_t)sig, (uint8_t)(sig >> 8), (uint8_t)(sig >> 16)}, coded;
        tx11a_encode_bits(b, CR_12, coded);
        symbol_out(coded.data(), 1, pilot_index, out + 2 * 640);
    }
    // DATA: SERVICE, MPDU, CRC-32, tail byte, pad (TBB11aSrc::Process, PHY_11a.hpp:125-190) through T11aSc (scramble.hpp:169-262)
    uint32_t crc = 0xFFFFFFFFu; for (uint32_t i = 0; i < len; i++) crc = (crc >> 8) ^ T.crc32_lut[payload[i] ^ (crc & 0xFF)]; crc = ~crc;
    const uint32_t nbytes = nsym * ri->ndbps / 8u;
    std::vector<uint8_t> data(nbytes, 0);
    memcpy(data.data() + 2, payload, len); memcpy(data.data() + 2 + len, &crc, 4);
    std::vector<uint8_t> ctrl(nbytes, 1); ctrl[2 + len + 4] = 2;                // TBB11aSrc: DO_SCRAMBLE, TAIL_SCRAMBLE on the tail byte
    uint8_t reg = sc_seed;
    tx11a_scramble(data.data(), ctrl.data(), nbytes, reg, data.data());
    std::vector<uint8_t> coded; tx11a_encode_bits(data, ri->cr, coded);
    const int ncbps = 48 * ri->nbpsc;
    for (uint32_t s = 0; s < nsym; s++) symbol_out(coded.data() + (size_t)s * ncbps, ri->nbpsc, pilot_index, out + 2 * (640 + 160 * (size_t)(1 + s)));
    memset(out + 2 * (640 + 160 * (size_t)(1 + nsym)), 0, 2 * (size_t)tail_zeros);
    return total;
}

} // namespace sbo
