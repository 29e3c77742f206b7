// ORACLE — TEST INFRASTRUCTURE ONLY (see ops.h).
// K=7 (133,171) soft-decision Viterbi with the reference's uint8 path metrics:
//   wrapping byte adds, survivor mark in the metric LSB, unsigned byte min, min-subtract
//   normalisation with the LSB masked, traceback on the LSB of stored columns.
// Follows kernel/bb/Brick11/src/viterbicore.h:36-261 (Viterbi_sig11) and :269-556 (TViterbiCore).
#include "viterbi.h"

namespace sbo {

static const v128 kEven = _mm_set1_epi8((char)0xFE);
static const v128 kOne = _mm_set1_epi8(1);

static inline v128 dup_lo(v128 a) { return _mm_unpacklo_epi8(a, a); }
static inline v128 dup_hi(v128 a) { return _mm_unpackhi_epi8(a, a); }

void ViterbiCore::reset() {
    if (col.empty()) col.resize((size_t)(max_steps + 2) * 4);
    cur = col.data(); steps = 0;
    cur[0] = _mm_set_epi8(0x30, 0x30, 0x30, 0x30, 0x30, 0x30, 0x30, 0x30, 0x30, 0x30, 0x30, 0x30, 0x30, 0x30, 0x30, 0x00);
    cur[1] = cur[2] = cur[3] = _mm_set1_epi8(0x30);            // viterbilut.h:22-32
}

// one trellis step with both coded bits present (viterbicore.h:294-372)
void ViterbiCore::step_ab(unsigned sa, unsigned sb) {
    const Tables& T = tables();
    const v128* A = (const v128*)T.vit_ma[sa * 8]; const v128* B = (const v128*)T.vit_mb[sb * 8];
    for (int g = 0; g < 4; g++) {
        v128 lo = cur[g >> 1], hi = cur[2 + (g >> 1)];
        v128 r0 = (g & 1) ? dup_hi(lo) : dup_lo(lo);
        v128 r1 = (g & 1) ? dup_hi(hi) : dup_lo(hi);
        r0 = _mm_and_si128(_mm_add_epi8(_mm_add_epi8(r0, A[2 * g]), B[2 * g]), kEven);
        r1 = _mm_or_si128(_mm_add_epi8(_mm_add_epi8(r1, A[2 * g + 1]), B[2 * g + 1]), kOne);
        cur[4 + g] = _mm_min_epu8(r0, r1);
    }
    cur += 4; steps++;
}
// one trellis step with a single coded bit (the other punctured) (viterbicore.h:374-443)
void ViterbiCore::step_one(bool use_b, unsigned s) {
    const Tables& T = tables();
    const v128* M = use_b ? (const v128*)T.vit_mb[s * 8] : (const v128*)T.vit_ma[s * 8];
    for (int g = 0; g < 4; g++) {
        v128 lo = cur[g >> 1], hi = cur[2 + (g >> 1)];
        v128 r0 = (g & 1) ? dup_hi(lo) : dup_lo(lo);
        v128 r1 = (g & 1) ? dup_hi(hi) : dup_lo(hi);
        r0 = _mm_and_si128(_mm_add_epi8(r0, M[2 * g]), kEven);
        r1 = _mm_or_si128(_mm_add_epi8(r1, M[2 * g + 1]), kOne);
        cur[4 + g] = _mm_min_epu8(r0, r1);
    }
    cur += 4; steps++;
}
void ViterbiCore::normalize() {                               // viterbicore.h:445-465
    v128 m = _mm_min_epu8(_mm_min_epu8(cur[0], cur[1]), _mm_min_epu8(cur[2], cur[3]));
    m = _mm_min_epu8(m, _mm_srli_si128(m, 8)); m = _mm_min_epu8(m, _mm_srli_si128(m, 4));
    m = _mm_min_epu8(m, _mm_srli_si128(m, 2)); m = _mm_min_epu8(m, _mm_srli_si128(m, 1));
    v128 sub = _mm_set1_epi8((char)(_mm_cvtsi128_si32(m) & 0xFE));
    for (int i = 0; i < 4; i++) cur[i] = _mm_sub_epi8(cur[i], sub);
}
// state with the smallest (metric, index) key plus its mark bit in bit 6 (viterbicore.h:468-520)
static inline int best_state(const v128* c) {
    const uint8_t* m = (const uint8_t*)c;
    unsigned best = 0xFFFFFFFFu;
    for (unsigned s = 0; s < 64; s++) { unsigned key = ((unsigned)m[s] << 8) | (s << 2); if (key < best) best = key; }
    return (int)((best >> 2) & 0x7F);
}
void ViterbiCore::traceback(uint8_t* out, uint32_t nbits, uint32_t lookahead) {   // viterbicore.h:468-555
    int pos = best_state(cur);
    const v128* tb = cur;
    for (uint32_t i = 0; i < lookahead; i++) {
        tb -= 4; pos = (pos >> 1) & 0x3F;
        pos |= (((const uint8_t*)tb)[pos] & 1) << 6;
    }
    uint8_t* po = out + (nbits >> 3);
    for (uint32_t i = 0; i < (nbits >> 3); i++) {
        uint8_t ch = 0;
        for (int j = 0; j < 8; j++) {
            ch = (uint8_t)((ch << 1) | ((pos >> 6) & 1));
            tb -= 4; pos = (pos >> 1) & 0x3F;
            pos |= (((const uint8_t*)tb)[pos] & 1) << 6;
        }
        *--po = ch;
    }
}

// SIGNAL field: 48 soft values, R=1/2, 24 steps, normalise every 8, full traceback (viterbicore.h:36-261)
uint32_t viterbi_signal(const uint8_t soft[48]) {
    ViterbiCore v; v.max_steps = 24; v.reset();
    for (int i = 0; i < 24; i++) {
        v.step_ab(soft[2 * i], soft[2 * i + 1]);
        if ((v.steps & 7) == 0) v.normalize();
    }
    v.normalize();
    uint8_t out[4] = {0, 0, 0, 0};
    v.traceback(out, 24, 0);
    uint32_t w = out[0] | (out[1] << 8) | (out[2] << 16);
    return w >> 6;                                            // viterbi.hpp:39
}

// Whole-block decode with the brick's cadence (viterbi.hpp:104-237): groups per code rate, normalise
// when (steps & 7)==0 after a group, windowed traceback depth/lookahead, final flush.
// `nsoft` need not be a multiple of 48 here; the brick's 48-byte bursts only bound the granularity.  A trailing partial puncture group is
// not decoded: the brick keeps it buffered for the next burst, and the device stops at the last whole group too.
size_t viterbi_decode_block(ViterbiCore& v, const uint8_t* soft, size_t nsoft, int code_rate,
                            uint32_t frame_len_bytes, uint32_t depth, uint32_t look, uint8_t* out, uint32_t& ob_count) {
    size_t produced = 0;
    const uint32_t prefix = 6;
    const uint32_t end = frame_len_bytes * 8 + 16 + prefix;
    const size_t group = code_rate == CR_12 ? 2 : code_rate == CR_34 ? 4 : 3;
    size_t i = 0;
    while (i + group <= nsoft) {
        if (code_rate == CR_12) { v.step_ab(soft[i], soft[i + 1]); i += 2; }
        else if (code_rate == CR_34) { v.step_ab(soft[i], soft[i + 1]); v.step_one(false, soft[i + 2]); v.step_one(true, soft[i + 3]); i += 4; }
        else { v.step_ab(soft[i], soft[i + 1]); v.step_one(false, soft[i + 2]); i += 3; }
        uint32_t t = v.steps;
        if ((t & 7) == 0) v.normalize();
        uint32_t nout = 0, la = 0;
        if (t >= end) { nout = end - ob_count - prefix; la = t - end; }
        else if (t >= ob_count + depth + look + prefix) { nout = depth; la = look + (t - (ob_count + depth + look + prefix)) % 8; }
        if (nout) {
            v.traceback(out + produced, nout, la);
            ob_count += nout; produced += nout >> 3;
        }
    }
    return produced;
}

} // namespace sbo
