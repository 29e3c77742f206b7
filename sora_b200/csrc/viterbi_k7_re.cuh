// sora_b200 — batched K=7 (133,171) soft Viterbi, v3 "history-carrying" kernel for sm_90a.
//
// Arithmetic contract (bit-exact with kernel/bb/Brick11/src/viterbicore.h:269-556 driven like
// kernel/bb/Brick11/src/viterbi.hpp:104-237): path metrics are the reference's uint8 values, whose LSB is the survivor mark and whose upper
// seven bits m7 are the metric proper (every branch metric is even, viterbilut.h, so the mark never carries into m7):
//     new = min_u8( (old[p] + bm) & 0xFE , (old[p+32] + bm') | 1 )   ==   m7' = min(a7, b7) mod 128 with ties to the even candidate,
//     decision d = (b7 < a7).
//
// Machine mapping (the quad / in-place trellis of v2, viterbi_k7_quad.cuh, with different bookkeeping):
//   * 4 lanes per code block, 16 metrics per lane, two per register as 16-bit halves; m7 sits in bits 9..15 of its half, so the uint8 wrap is the
//     half's own carry-out.  Every add is a per-half SIMD add (VIADD.16x2, or the add inside VIADDMNMX.U16x2): nothing crosses halves.
//   * The low byte of a half carries the survivor HISTORY of the path that ends in that state: trellis step t gives the odd candidate bit
//     j = (t - 1) mod 8 (folded into its branch-metric constant) and leaves it clear in the even candidate.  Bits j+1..8 are still zero in both
//     candidates, so a metric tie is decided by bit j exactly like the reference's LSB mark decides it (even wins), bits below j are never
//     reached by the compare, and the min moves the winner's history along for free.  One fused VIADDMNMX.U16x2 (DPX add-min) plus one
//     VIADD.16x2 per register and step is the whole add-compare-select: no role masks, no per-step gathering of decision bits.
//   * Every 8 steps each half holds the eight decisions of its survivor over the block (register exchange over 8 columns): four PRMTs line
//     the 16 history bytes of a lane up in slot-address order and one 128-bit store puts them into a shared-memory ring:
//     entry [block][code block][slot] = 64 bytes per 8 columns, the same 8 bytes per column a plain decision matrix needs.
//   * Traceback jumps a whole block per lookup: the history byte h of slot A gives the eight decoded bits, and the slot eight columns earlier
//     is a fixed bit permutation of h rotated by the phase of the block boundary (K=7 replaces all six state bits in six steps).
//     A window of 256+24..31 columns costs ~37 byte loads instead of 280 64-bit word look-ups.
//   * The 8 code blocks of a warp run in lockstep (the caller hands every launch a dense list of the frames of its code rate), so the
//     path-metric exchange is a plain full-mask SHFL.BFLY; 24 steps (lcm of the 6-step phase cycle and the 8-step history block) without a
//     traceback trigger run as one branch-free instruction stream, everything else goes through a 6-step path with the event checks.
//   * The kernel emits the decoded bytes (SERVICE + PSDU, still scrambled).  Descrambler, CRC-32 and the verdict (scramble.hpp:269-355,
//     PHY_11a.hpp:609-702) run in k_sink11a, one thread per frame, after it.
// Instruction rates that shape this (tools/microbench/pipes.cu on an H100 SXM, 400 W limit): VIADDMNMX.U16x2 + IMAD/VIADD issue together at
// ~0.9 per cycle per sub-partition; VIMNMX + two adds (the v2 ACS) at 0.74; LOP3 and PRMT at 0.5.
#pragma once
#include "viterbi_k7_quad.cuh"
#include <type_traits>

namespace sb {

#define SB_VR_FR 8                         // code blocks per CTA (one warp)
#define SB_VR_NB 38                        // ring entries of 8 columns: depth + lookahead + 7 <= 288 columns = 36 entries, + the running one + 1

// Windowed traceback (viterbi.hpp:205-237) from slot A0 at time t over la + nout columns; the newest block (kp = t mod 8 columns, 0 = a whole
// one) is in ring entry e.  The walk is a chain of dependent shared-memory look-ups, one per 8 columns, done by one lane of the quad; it only
// collects the history bytes it passes, newest first, into the quad's scratch row `hb`: byte 0 = the kp decisions of the running block (right
// aligned; absent when kp = 0), then one byte per block, bit 7 = the newest column of the block.  vr_emit turns the row into output bytes.
// Kept out of line: it runs once per `depth` steps and must not sit in the instruction stream of the step loop.
#define SB_VR_HB 52                                          // >= (7 + 31 + 256 + 6) / 8 + 2; 13 words: rows of neighbouring lanes fall into different banks
template <int FR>
__device__ __noinline__ void vr_traceback(const uint8_t* __restrict__ ring_b, uint8_t* __restrict__ hb, uint32_t e, const uint32_t A0, const uint32_t t, uint32_t todo) {
    uint32_t A = A0, j = 0;
    uint32_t tt = t;                                         // time of the newest column not yet walked
    const uint32_t kp = t & 7u;
    if (kp) {                                                // running block: kp decisions in bits 0..kp-1, one slot-address bit changes per column
        const uint32_t h = (uint32_t)ring_b[e * (FR * 64) + A];
        const uint32_t take = min(kp, todo);
        for (uint32_t c = 0; c < take; c++) {                // column tt - c was produced at phase (tt - c - 1) mod 6: bit 5 - phase is replaced
            const uint32_t b = 5u - (tt - c - 1u) % 6u, d = (h >> (kp - 1u - c)) & 1u;
            A = (A & ~(1u << b)) | (d << b);
        }
        hb[j++] = (uint8_t)(h & ((1u << kp) - 1u));
        todo -= take; tt -= kp; e = e ? e - 1u : SB_VR_NB - 1u;
    }
    uint32_t ph = tt % 6u;                                   // phase of the block boundary the walk stands on
    const uint8_t* rp = ring_b + e * (FR * 64);
    while (todo >= 8u) {
        const uint32_t h = (uint32_t)rp[A];
        hb[j++] = (uint8_t)h;
        const uint32_t r = __brev(h) >> 24;                  // r bit i = h bit 7 - i = decision of column tt - i
        const uint32_t G = (r & 0x3Cu) | (r >> 6);           // slot-address bit (i - ph) mod 6 <- column tt - i, the two oldest overriding i = 0, 1
        A = ((G | (G << 6)) >> ph) & 63u;
        todo -= 8u; ph = ph >= 2u ? ph - 2u : ph + 4u;       // (tt - 8) mod 6
        rp = rp == ring_b ? ring_b + (SB_VR_NB - 1u) * (FR * 64) : rp - FR * 64;
    }
    if (todo) hb[j++] = rp[A];         // oldest block of the window: only its newest `todo` columns count
    hb[j] = 0; hb[j + 1] = 0;
}
// The nout / 8 decoded bytes of a window from the scratch row: bit k of the walk (k = 0 the newest column) sits at row bit (8 - kp) % 8 + k,
// counted from bit 7 of byte 0; the first la bits are only looked through, byte m of the output (m = 0 the LAST byte of the window) is the
// eight bits from la + 8 m on, newest in bit 7.  All four lanes of the quad take part; byte m goes to op[first + nbytes - 1 - m].
__device__ __forceinline__ void vr_emit(const uint8_t* __restrict__ hb, uint8_t* __restrict__ op, const uint32_t out_cap, const uint32_t first, const uint32_t nbytes,
                                        const uint32_t kp, const uint32_t la, const uint32_t q, const uint32_t nl) {
    const uint32_t s0 = ((8u - kp) & 7u) + la, sh = s0 & 7u, i0 = s0 >> 3;
    for (uint32_t m = q; m < nbytes; m += nl) {
        const uint32_t v = ((uint32_t)hb[i0 + m] << 8) | hb[i0 + m + 1u];
        const uint32_t at = first + nbytes - 1u - m;
        if (at < out_cap) op[at] = (uint8_t)(v >> (8u - sh));
    }
}
__device__ __noinline__ uint32_t vr_best_slot(uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3, uint32_t r4, uint32_t r5, uint32_t r6, uint32_t r7,
                                              const uint32_t q, const uint32_t tm, const uint32_t tn, const unsigned QM) {
    const uint32_t R[8] = {r0, r1, r2, r3, r4, r5, r6, r7};
    return vr_best_core<2>(R, q, tm, tn, QM);
}
__device__ __noinline__ uint32_t vr_best_slot16(uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3, uint32_t r4, uint32_t r5, uint32_t r6, uint32_t r7,
                                                uint32_t r8, uint32_t r9, uint32_t r10, uint32_t r11, uint32_t r12, uint32_t r13, uint32_t r14, uint32_t r15,
                                                const uint32_t q, const uint32_t tm, const uint32_t tn, const unsigned QM) {
    const uint32_t R[16] = {r0, r1, r2, r3, r4, r5, r6, r7, r8, r9, r10, r11, r12, r13, r14, r15};
    return vr_best_core<1>(R, q, tm, tn, QM);
}


template <int CODE_RATE, int LB>
struct VrDecoder {
    static constexpr int NR = 8 << (2 - LB), NL = 1 << LB, FR = 32 >> LB;                        // registers per lane, lanes per code block, code blocks per warp
    static constexpr uint32_t GROUP = CODE_RATE == CR_12 ? 2u : CODE_RATE == CR_34 ? 4u : 3u;   // soft bytes per puncture group
    static constexpr uint32_t GSTEPS = CODE_RATE == CR_12 ? 1u : CODE_RATE == CR_34 ? 3u : 2u;  // trellis steps per group
    static constexpr uint32_t CHUNK_BYTES = 6u / GSTEPS * GROUP;                                // 12 (R=1/2), 9 (2/3), 8 (3/4) soft bytes per 6 steps
    uint32_t R[NR];
    VrLane LC;
    uint32_t kc[2];        // 28 << 8 and 14 << 8 in both halves, as registers
    uint32_t mk[8], mkA[2][4], mkB[2][4], mkH[4], mkL[4];   // history marks 0x00010001 << j as registers; per lane-pair phase and chunk; T = 5 halves
    unsigned QM; int q;
    uint4* ring_q; const uint8_t* ring_b; uint8_t* hb;   // hb: the quad's traceback scratch row (SB_VR_HB bytes of shared memory)
    const uint8_t* sp; uint8_t* op; uint32_t out_cap, nsoft;
    uint32_t depth, look, end, ob, next_tb, nraw, wslot;
    bool done;

    __device__ __forceinline__ void fetch(const uint32_t pos, uint32_t (&a)[3]) const {
        if (pos + CHUNK_BYTES > nsoft) { a[0] = a[1] = a[2] = 0; return; }
        if constexpr (CODE_RATE == CR_34) { const uint2 v = __ldg((const uint2*)(sp + pos)); a[0] = v.x; a[1] = v.y; a[2] = 0; }
        else if constexpr (CODE_RATE == CR_12) { a[0] = __ldg((const uint32_t*)(sp + pos)); a[1] = __ldg((const uint32_t*)(sp + pos + 4)); a[2] = __ldg((const uint32_t*)(sp + pos + 8)); }
        else { uint32_t b[9];
#pragma unroll
               for (int i = 0; i < 9; i++) b[i] = __ldg(sp + pos + i);
               // keep every puncture group inside one word: w0 = b0 b1 b2 -, w1 = b3 b4 b5 -, w2 = b6 b7 b8 -
               a[0] = b[0] | (b[1] << 8) | (b[2] << 16); a[1] = b[3] | (b[4] << 8) | (b[5] << 16); a[2] = b[6] | (b[7] << 8) | (b[8] << 16); }
    }
    // the history bytes of this lane (low byte of every half: 16 or 32), in slot-address order, into ring entry `e`
    __device__ __forceinline__ void store_hist(const uint32_t e) {
#pragma unroll
        for (int i = 0; i < NR / 8; i++) {
            uint4 w;
            w.x = __byte_perm(R[8 * i + 0], R[8 * i + 1], 0x6420); w.y = __byte_perm(R[8 * i + 2], R[8 * i + 3], 0x6420);
            w.z = __byte_perm(R[8 * i + 4], R[8 * i + 5], 0x6420); w.w = __byte_perm(R[8 * i + 6], R[8 * i + 7], 0x6420);
            ring_q[e * (FR * 4) + i] = w;
        }
    }
    __device__ __forceinline__ void clear_hist() {
#pragma unroll
        for (int r = 0; r < NR; r++) R[r] &= 0xFE00FE00u;
    }
    __device__ __forceinline__ void next_slot() { wslot = wslot == SB_VR_NB - 1u ? 0u : wslot + 1u; }
    // viterbi.hpp:177-180 -> viterbicore.h:445-465: subtract (smallest byte & 0xFE) = the smallest m7; `mask` names the lanes that take part
    __device__ __forceinline__ void normalize(const unsigned mask) {
        uint32_t m = __vminu2(__vminu2(__vminu2(R[0], R[1]), __vminu2(R[2], R[3])), __vminu2(__vminu2(R[4], R[5]), __vminu2(R[6], R[7])));
        if constexpr (NR >= 16) m = __vminu2(m, __vminu2(__vminu2(__vminu2(R[8], R[9]), __vminu2(R[10], R[11])), __vminu2(__vminu2(R[12], R[13]), __vminu2(R[14], R[15]))));
        if constexpr (NR == 32) {
            uint32_t m2 = __vminu2(__vminu2(__vminu2(R[16], R[17]), __vminu2(R[18], R[19])), __vminu2(__vminu2(R[20], R[21]), __vminu2(R[22], R[23])));
            m2 = __vminu2(m2, __vminu2(__vminu2(__vminu2(R[24], R[25]), __vminu2(R[26], R[27])), __vminu2(__vminu2(R[28], R[29]), __vminu2(R[30], R[31]))));
            m = __vminu2(m, m2);
        }
        m = min(m & 0xFFFFu, m >> 16) >> 9;             // smallest m7 of this lane
        if constexpr (LB >= 1) m = min(m, __shfl_xor_sync(mask, m, 1));
        if constexpr (LB == 2) m = min(m, __shfl_xor_sync(mask, m, 2));
        const uint32_t mv = m * 0x02000200u;
#pragma unroll
        for (int r = 0; r < NR; r++) R[r] -= mv;        // every half >= m << 9: no borrow between halves, histories untouched
    }
    // windowed traceback from slot A0 at time t (viterbi.hpp:205-237): one lane of the quad walks the ring (vr_traceback)
    __device__ __forceinline__ void traceback(const uint32_t A0, const uint32_t t, const uint32_t la, const uint32_t nout) {
        __syncwarp(QM);
        if (q == 0) vr_traceback<FR>(ring_b, hb, wslot, A0, t, la + nout);
        __syncwarp(QM);
        vr_emit(hb, op, out_cap, nraw, nout >> 3, t & 7u, la, (uint32_t)q, (uint32_t)NL);
        nraw += nout >> 3;
        __syncwarp(QM);
    }
    // traceback trigger at time t (a puncture-group boundary), viterbi.hpp:182-203; tm = t mod 6
    __device__ __forceinline__ void trigger(const uint32_t t, const uint32_t tm) {
        if (t < next_tb) return;
        uint32_t nout, la;
        if (t >= end) { nout = end - ob - 6u; la = t - end; }
        else { nout = depth; la = look + (t - (ob + depth + look + 6u)) % 8u; }
        if (nout) {                                     // uniform inside the quad
            uint32_t A0;
            if constexpr (LB == 2) A0 = vr_best_slot(R[0], R[1], R[2], R[3], R[4], R[5], R[6], R[7], (uint32_t)q, tm, (t - 1u) & 7u, QM);
            else A0 = vr_best_slot16(R[0], R[1], R[2], R[3], R[4], R[5], R[6], R[7], R[8], R[9], R[10], R[11], R[12], R[13], R[14], R[15], (uint32_t)q, tm, (t - 1u) & 7u, QM);
            if (t & 7u) store_hist(wslot);              // mid-block: the partial histories of the running block (a block end has just stored its own)
            traceback(A0, t, la, nout);
            ob += nout;
        }
        if (ob + 6u >= end && t >= end) done = true;
        next_tb = min(end, ob + depth + look + 6u);
        if (next_tb <= t) next_tb = t + 1u;              // a frame shorter than the prefix: re-evaluate at every group
    }
    // steps S .. 23 of a 24-step stretch that starts at a multiple of 24 and holds no traceback trigger: no branches at all
    template <int S> __device__ __forceinline__ void fast(const uint32_t (&w)[4][3]) {
        if constexpr (S < 24) {
            constexpr int T = S % 6, J = S % 8, I = S / 6;
            const uint32_t cb = vr_bm<CODE_RATE, T>(w[I]);
            const uint32_t KC = kc[vr_ksum<CODE_RATE, T>() == 28u ? 0 : 1];
            if constexpr (T < LB) vr_step<T, true, LB>(R, cb, LC, KC, mkA[T][I], mkB[T][I], 0xFFFFFFFFu);
            else if constexpr (T <= 4) vr_step<T, true, LB>(R, cb, LC, KC, mk[J], 0u, 0xFFFFFFFFu);
            else vr_step<T, true, LB>(R, cb, LC, KC, mkH[I], mkL[I], 0xFFFFFFFFu);
            if constexpr ((S + 1) % 8 == 0) {
                store_hist(wslot); next_slot();
                if constexpr ((S + 1) % GSTEPS == 0) normalize(0xFFFFFFFFu);
                clear_hist();
            }
            fast<S + 1>(w);
        }
    }
    // steps s .. 5 of a 6-step chunk that starts at time tb (a multiple of 6), with every event check; quads that are not `live` only keep step
    template <int s> __device__ __forceinline__ void slow(const uint32_t (&w)[3], const uint32_t tb, const bool live) {
        if constexpr (s < 6) {
            const uint32_t t = tb + s + 1u;
            vr_step_rt<s, true, LB>(R, vr_bm<CODE_RATE, s>(w), LC, kc[vr_ksum<CODE_RATE, s>() == 28u ? 0 : 1], 0x00010001u << ((t - 1u) & 7u), 0xFFFFFFFFu);
            const bool blk = (t & 7u) == 0u;            // uniform over the warp
            if (blk) store_hist(wslot);
            if constexpr ((s + 1) % GSTEPS == 0) {
                if (blk) normalize(0xFFFFFFFFu);
                if (live && !done) trigger(t, (s + 1) % 6);
            }
            if (blk) { clear_hist(); next_slot(); }
            slow<s + 1>(w, tb, live);
        }
    }
};

// Work lists: the frames of every code rate, densely, so that each rate's launch runs warps of eight live code blocks.
// cnt[3] must be zero on entry; list holds 3 x nframes entries.
__global__ void k_vit_lists(const FrameInfo* __restrict__ info, uint32_t nframes, uint32_t* __restrict__ cnt, uint32_t* __restrict__ list) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t rate = 3u;
    if (f < nframes) { const FrameInfo fi = info[f]; if (fi.status == E_SUCCESS && fi.code_rate < 3u) rate = fi.code_rate; }
#pragma unroll
    for (uint32_t r = 0; r < 3u; r++) {                 // one atomic per warp and rate
        const unsigned m = __ballot_sync(0xFFFFFFFFu, rate == r);
        if (m == 0u) continue;
        const int leader = __ffs(m) - 1; uint32_t base = 0;
        if ((int)(threadIdx.x & 31) == leader) base = atomicAdd(cnt + r, (uint32_t)__popc(m));
        base = __shfl_sync(0xFFFFFFFFu, base, leader);
        if (rate == r) list[(size_t)r * nframes + base + (uint32_t)__popc(m & ((1u << (threadIdx.x & 31)) - 1u))] = f;
    }
}

// list / cnt: work list of this code rate (k_vit_lists) or null = frames 0 .. nframes-1 with the uniform parameters of `job`.
template <int CODE_RATE, int LB = 2>
__global__ void __launch_bounds__(32) k_viterbi_re(const uint8_t* __restrict__ soft, uint64_t soft_stride, uint32_t nframes,
        const uint32_t* __restrict__ list, const uint32_t* __restrict__ cnt, const FrameInfo* __restrict__ info, VitJob job,
        uint8_t* __restrict__ out, uint64_t out_stride, uint32_t raw_off, uint32_t* __restrict__ nraw_out) {
    using D = VrDecoder<CODE_RATE, LB>;
    constexpr int FR = D::FR, NL = D::NL;               // code blocks per warp (8 | 16), lanes per code block (4 | 2)
    __shared__ uint4 s_ring[SB_VR_NB][FR][4];          // entry: history bytes of the 64 slots of every code block over 8 columns
    __shared__ uint8_t s_hb[FR][SB_VR_HB];             // traceback scratch: the history bytes a walk passed, per code block
    constexpr unsigned FULL = 0xFFFFFFFFu;
    const uint32_t nvalid = list ? __ldg(cnt + CODE_RATE) : (job.code_rate == (uint32_t)CODE_RATE ? nframes : 0u);
    if (blockIdx.x * FR >= nvalid) return;              // whole CTA
    const int lane = threadIdx.x & 31, q = lane & (NL - 1), fb = lane >> LB;
    const uint32_t idx = blockIdx.x * FR + fb;
    const bool valid = idx < nvalid;
    const uint32_t f = !valid ? 0u : list ? __ldg(list + (size_t)CODE_RATE * nframes + idx) : idx;
    uint32_t L = job.frame_len;
    D d;
    d.nsoft = job.nsoft;
    if (valid && info) { const FrameInfo fi = info[f]; L = fi.length; d.nsoft = fi.soft_bytes; }
    if (!valid) d.nsoft = 0;
    d.q = q; d.QM = (NL == 4 ? 0xFu : NL == 2 ? 0x3u : 0x1u) << (lane & ~(NL - 1));
    d.depth = job.depth; d.look = job.lookahead;
    d.sp = soft + (size_t)f * soft_stride;
    d.op = out + (size_t)f * out_stride + raw_off;
    d.out_cap = (uint32_t)(out_stride - raw_off < 0xFFFFFFFFull ? out_stride - raw_off : 0xFFFFFFFFull);
#pragma unroll
    for (int t = 0; t < 6; t++) {
        const int lc = vq_cls(vq_rol6(q << (6 - LB), t) & 31);     // class contribution of this lane's address bits at phase t
        const int K = vr_kcls(t);
        d.LC.sel[t][0] = vq_sel(0 ^ lc, 0 ^ K ^ lc); d.LC.sel[t][1] = vq_sel(1 ^ lc, 1 ^ K ^ lc);
    }
    if constexpr (LB >= 1) {
        d.LC.bA[0] = (q >> (LB - 1)) & 1; d.LC.bB[0] = 1u - d.LC.bA[0]; // pair bit at T = 0 is address bit 5 (the top lane bit), at T = 1 (LB = 2) address bit 4
        d.LC.bA[1] = q & 1;               d.LC.bB[1] = 1u - d.LC.bA[1];
    } else { d.LC.bA[0] = d.LC.bA[1] = 0u; d.LC.bB[0] = d.LC.bB[1] = 0u; }   // one lane per code block: no lane-pair phase
    {   // history marks as run-time values (z is always 0, which the compiler cannot know): they must stay register operands
        const uint32_t z = (uint32_t)(soft_stride >> 63);
        d.kc[0] = 0x1C001C00u + z; d.kc[1] = 0x0E000E00u + z;
#pragma unroll
        for (int j = 0; j < 8; j++) d.mk[j] = (0x00010001u << j) + z;
#pragma unroll
        for (int i = 0; i < 4; i++) {                   // chunk i of a 24-step stretch: its steps 0, 1, 5 are steps 6i, 6i+1, 6i+5
            d.mkA[0][i] = d.LC.bA[0] * d.mk[(6 * i) % 8];     d.mkB[0][i] = d.LC.bB[0] * d.mk[(6 * i) % 8];
            d.mkA[1][i] = d.LC.bA[1] * d.mk[(6 * i + 1) % 8]; d.mkB[1][i] = d.LC.bB[1] * d.mk[(6 * i + 1) % 8];
            d.mkH[i] = d.mk[(6 * i + 5) % 8] & 0xFFFF0000u;   d.mkL[i] = d.mk[(6 * i + 5) % 8] & 0x0000FFFFu;
        }
    }
    // initial metrics (viterbilut.h:22-32): state 0 -> 0x00, others 0x30; at t=0 state == address; byte value v sits at v << 8
#pragma unroll
    for (int r = 0; r < D::NR; r++) d.R[r] = 0x30003000u;
    if (q == 0) d.R[0] = 0x30000000u;
    d.end = L * 8u + 16u + 6u; d.ob = 0; d.nraw = 0; d.wslot = 0; d.done = !valid;
    d.next_tb = min(d.end, d.depth + d.look + 6u);      // first time a traceback can fire (viterbi.hpp:182-203)
    uint4* const ring0 = &s_ring[0][0][0];              // this CTA's ring: [entry][code block][4 x 16 bytes]
    d.ring_q = ring0 + fb * 4 + q * (4 / NL);     // + entry * (FR * 4): this lane's 16 / 32 / 64 bytes of the code block's 64 (LB = 0: + group * FR)
    d.ring_b = (const uint8_t*)(ring0 + fb * 4);        // + entry * (FR * 64) + slot
    d.hb = s_hb[fb];

    // lockstep part: all eight code blocks of the warp advance together, 24 or 6 steps at a time; the soft values of the next four chunks
    // are always in registers
    uint32_t tb = 0, pos = 0, phase24 = 0;              // time and soft position at the start of the next chunk (uniform); (tb / 6) mod 4
    uint32_t w[4][3];
#pragma unroll
    for (int c = 0; c < 4; c++) d.fetch(pos + c * D::CHUNK_BYTES, w[c]);
    bool stale = false;                                 // out of input while others kept stepping (cannot happen with whole-symbol inputs)
    for (;;) {
        const bool more = !d.done && pos + D::CHUNK_BYTES <= d.nsoft;
        if (!__any_sync(FULL, more)) break;
        if (!more && !d.done) stale = true;
        const bool fast_ok = d.done || (tb + 24u < d.next_tb && pos + 4u * D::CHUNK_BYTES <= d.nsoft);
        if (phase24 == 0u && __all_sync(FULL, fast_ok)) {
            uint32_t n[4][3];
#pragma unroll
            for (int c = 0; c < 4; c++) d.fetch(pos + (4 + c) * D::CHUNK_BYTES, n[c]);
            d.template fast<0>(w);
#pragma unroll
            for (int c = 0; c < 4; c++) { w[c][0] = n[c][0]; w[c][1] = n[c][1]; w[c][2] = n[c][2]; }
            tb += 24u; pos += 4u * D::CHUNK_BYTES;
            continue;
        }
        uint32_t n[3];
        d.fetch(pos + 4u * D::CHUNK_BYTES, n);
        d.template slow<0>(w[0], tb, more);
#pragma unroll
        for (int c = 0; c < 3; c++) { w[c][0] = w[c + 1][0]; w[c][1] = w[c + 1][1]; w[c][2] = w[c + 1][2]; }
        w[3][0] = n[0]; w[3][1] = n[1]; w[3][2] = n[2];
        tb += 6u; pos += D::CHUNK_BYTES; phase24 = (phase24 + 1u) & 3u;
    }
    // tail: whole puncture groups that do not fill a 6-step chunk (standalone API with arbitrary nsoft): per code block, phases at run time
    if (!d.done && !stale) {
        uint32_t k = 0;                                 // steps into the chunk at tb
        auto step_rt = [&](const uint32_t Cbase, const uint32_t KC) {
            const uint32_t mark = 0x00010001u << ((tb + k) & 7u);
            switch (k) { case 0: vr_step_rt<0, false, LB>(d.R, Cbase, d.LC, KC, mark, d.QM); break; case 1: vr_step_rt<1, false, LB>(d.R, Cbase, d.LC, KC, mark, d.QM); break;
                         case 2: vr_step_rt<2, false, LB>(d.R, Cbase, d.LC, KC, mark, d.QM); break; case 3: vr_step_rt<3, false, LB>(d.R, Cbase, d.LC, KC, mark, d.QM); break;
                         case 4: vr_step_rt<4, false, LB>(d.R, Cbase, d.LC, KC, mark, d.QM); break; default: vr_step_rt<5, false, LB>(d.R, Cbase, d.LC, KC, mark, d.QM); }
            k++;
            if (((tb + k) & 7u) == 0u) d.store_hist(d.wslot);
        };
        auto block_end = [&]() { if (((tb + k) & 7u) == 0u) { d.clear_hist(); d.next_slot(); } };
        while (!d.done && pos + D::GROUP <= d.nsoft) {
            uint32_t g = __ldg(d.sp + pos) | ((uint32_t)__ldg(d.sp + pos + 1) << 8);
            if (D::GROUP > 2) g |= (uint32_t)__ldg(d.sp + pos + 2) << 16;
            if (D::GROUP > 3) g |= (uint32_t)__ldg(d.sp + pos + 3) << 24;
            pos += D::GROUP;
            step_rt(vq_bm_ab<0>(g), d.kc[0]);
            if (D::GSTEPS >= 2) { block_end(); step_rt(vq_bm_a<2>(g), d.kc[1]); }
            if (D::GSTEPS >= 3) { block_end(); step_rt(vq_bm_b<3>(g), d.kc[1]); }
            const uint32_t t = tb + k;
            if ((t & 7u) == 0u) d.normalize(d.QM);
            d.trigger(t, k == 6 ? 0u : k);
            block_end();
            if (k == 6) { k = 0; tb += 6; }
        }
    }
    if (valid && q == 0) nraw_out[f] = d.nraw;
}

// Descrambler + frame sink after the Viterbi kernel, one thread per frame (T11aDesc, scramble.hpp:269-355; TBB11aFrameSink, PHY_11a.hpp:609-702):
// raw bytes (SERVICE + scrambled PSDU) sit at row + 14 so that the PSDU starts 16-byte aligned at row + 16; the descrambled PSDU goes to row + 0.
// The first SERVICE byte is dropped, the second seeds the register (byte >> 1), then out = byte ^ lut[reg], reg advances by eight bits per byte.
// Both recurrences are taken off the per-byte dependency chain: the masks a 7-bit register produces byte after byte are one cycle of 127
// values (x^7 + x^4 + 1 is primitive, 8 and 127 are coprime), so the mask of byte i is s_seq[(position of the seed + i) mod 127] — four
// independent look-ups per word — and the CRC-32 goes four bytes per step through the three derived tables of the sliced form
// (T_k[i] = T_{k-1}[i] >> 8 ^ T_0[T_{k-1}[i] & 0xFF]); the words that touch the FCS or the end of the data take the byte-wise path.
__global__ void __launch_bounds__(128) k_sink11a(uint8_t* __restrict__ out, uint64_t out_stride, uint32_t nframes, const FrameInfo* __restrict__ info,
                                                 DevTables T, uint32_t* __restrict__ status_io, uint32_t* __restrict__ crc_out) {
    __shared__ uint32_t s_crc[4][256];                 // CRC-32 (reflected 0xEDB88320, core/inc/CRC32.h:76) and its three sliced companions
    __shared__ uint8_t s_scr[128];
    __shared__ uint8_t s_seq[136];                     // [0, 127): the cycle of masks, [127, 130): its first three again, [132, 136): zeros (the all-zero register)
    __shared__ uint8_t s_pos[128];                     // 7-bit register -> position of its first mask in the cycle (register 0: 132)
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_crc[0][i] = __ldg(T.crc32 + i);
    for (int i = threadIdx.x; i < 128; i += blockDim.x) s_scr[i] = __ldg(T.scramble + i);
    __syncthreads();
    for (int k = 1; k < 4; k++) {
        for (int i = threadIdx.x; i < 256; i += blockDim.x) { const uint32_t v = s_crc[k - 1][i]; s_crc[k][i] = (v >> 8) ^ s_crc[0][v & 0xFFu]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        uint32_t reg = 1;
        for (int k = 0; k < 127; k++) { const uint32_t m = s_scr[reg]; s_seq[k] = (uint8_t)m; s_pos[reg] = (uint8_t)k; reg = m >> 1; }
        s_seq[127] = s_seq[0]; s_seq[128] = s_seq[1]; s_seq[129] = s_seq[2]; s_seq[130] = s_seq[131] = 0;
        s_seq[132] = s_seq[133] = s_seq[134] = s_seq[135] = 0; s_pos[0] = 132;
    }
    __syncthreads();
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nframes) return;
    const FrameInfo fi = info[f];
    if (fi.status != E_SUCCESS) return;                 // the front end already reached a terminal code: nothing was decoded
    const uint32_t L = fi.length, nraw = status_io[f];  // bytes the Viterbi kernel produced (SERVICE included)
    uint8_t* row = out + (size_t)f * out_stride;
    uint32_t verdict = E_FAILED, fcs = 0, crc = 0xFFFFFFFFu;
    if (nraw >= 2u) {
        const uint32_t reg0 = row[15] >> 1;
        uint32_t p = s_pos[reg0]; const uint32_t pstep = reg0 ? 4u : 0u;
        const uint32_t have = min(nraw - 2u, L);        // PSDU bytes available
        const uint32_t cap = (uint32_t)(out_stride < 0xFFFFFFFFull ? out_stride : 0xFFFFFFFFull);
        for (uint32_t i0 = 0; i0 < have; i0 += 16u) {
            const uint4 v = *(const uint4*)(row + 16 + i0);
            uint32_t w[4] = {v.x, v.y, v.z, v.w}, o4[4];
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const uint32_t m = (uint32_t)s_seq[p] | ((uint32_t)s_seq[p + 1] << 8) | ((uint32_t)s_seq[p + 2] << 16) | ((uint32_t)s_seq[p + 3] << 24);
                p += pstep; if (p >= 127u && pstep) p -= 127u;
                const uint32_t ow = w[j] ^ m, i = i0 + 4u * j;
                o4[j] = ow;
                if (i + 7u < L && i + 3u < have) {       // the whole word is data under the CRC
                    const uint32_t c = crc ^ ow;
                    crc = s_crc[3][c & 0xFFu] ^ s_crc[2][(c >> 8) & 0xFFu] ^ s_crc[1][(c >> 16) & 0xFFu] ^ s_crc[0][c >> 24];
                } else {
#pragma unroll
                    for (int b = 0; b < 4; b++) {
                        const uint32_t ib = i + b, o = (ow >> (8 * b)) & 0xFFu;
                        if (ib < have) {
                            if (ib + 4u < L) crc = (crc >> 8) ^ s_crc[0][(crc ^ o) & 0xFFu];
                            else if (L >= 4u) fcs |= o << (8u * (ib + 4u - L));
                        }
                    }
                }
            }
            if (i0 + 16u <= have && i0 + 16u <= cap) *(uint4*)(row + i0) = make_uint4(o4[0], o4[1], o4[2], o4[3]);
            else for (uint32_t i = i0; i < have && i < cap; i++) row[i] = (uint8_t)(o4[(i - i0) >> 2] >> (8u * ((i - i0) & 3u)));
        }
        if (have == L && L >= 4u) verdict = (~crc == fcs) ? (uint32_t)E_FRAME_OK : (uint32_t)E_CRC32_FAIL;
        else fcs = 0;                                   // frame_crc32 is only set once the last FCS byte arrived (PHY_11a.hpp:688)
    }
    status_io[f] = verdict; crc_out[f] = fcs;
}

} // namespace sb
