// sora_b200 — batched K=7 (133,171) soft Viterbi, "lane" kernel for sm_90a: ONE LANE PER CODE BLOCK, six-column history blocks.
//
// Arithmetic contract: the same as viterbi_k7_re.cuh (bit-exact with kernel/bb/Brick11/src/viterbicore.h:269-556 driven like
// kernel/bb/Brick11/src/viterbi.hpp:104-237); the add-compare-select is that file's vr_step — one fused VIADDMNMX.U16x2 and one
// VIADD.16x2 per register and trellis step, the survivor history riding in the low byte of every 16-bit metric.
//
// What is different, and why (DESIGN.md §4):
//   * A lane owns all 64 states of a code block (32 registers); a warp decodes 32 code blocks.  No lane ever needs another lane's
//     metrics: no shuffle, no quad mask, no per-lane selector — every PRMT selector and pairing distance is a compile-time constant.
//     The per-warp overhead of a step (branch-metric construction, fetch, loop) is spread over 32 code blocks instead of 8:
//     0.63x the instructions of the four-lanes-per-block kernel for the same work (measured).
//   * The 24-step unrolled stream of viterbi_k7_re.cuh (lcm of the 6-step trellis phase and its 8-column history block) does not
//     survive this widening: 1 800 instructions of straight-line code per warp, every warp at another place in it — the measured
//     kernels stall on instruction fetch (2.8 - 4.3 warps per issue slot waiting for instructions).  Here the loop body is ONE 6-step
//     chunk.  With six-column history blocks (HB = 6) everything in it is a constant of the phase; with eight-column blocks (HB = 8, the
//     default: a quarter less ring traffic, fewer look-ups per window) the mark of a step is a warp-uniform run-time shift and the block
//     ends are three uniform branches.
//   * The survivor ring (up to 67 entries x 64 bytes per code block = 134 KB per warp) cannot live in shared memory; it is a per-CTA slab
//     of global memory, written with one fully coalesced 128-bit store per 16 states (512 contiguous bytes per warp and instruction)
//     and read back with ld.global.cg.  Every lane walks its own window — 32 walks per warp instruction, where the quad kernel has 8 —
//     and packs the decoded bits on the way; there is no scratch row and no second pass.  The rings of all resident warps do not fit
//     L2: this is HBM traffic (6 GB written, 4.6 GB read per 65 536 frames) that the kernel trades for instructions.
//   * The walk is a chain of dependent look-ups of ~1 400 cycles each.  DEFER (default) takes it off the critical path: the trigger only
//     starts it, the step loop does one look-up per chunk (VlDecoder::walk_tick), the forward pass never waits.
//   DESIGN.md, "The Viterbi kernel", has the measurements behind each of these.
#pragma once
#include "viterbi_k7_common.cuh"

namespace sb {

#define SB_VL_FR 32                        // code blocks per CTA (one warp), one lane each
#define SB_VL_NB 50                        // ring entries of 6 columns: depth + lookahead + 7 <= 288 columns = 48 entries, + the running one + 1
#define SB_VL_NB8 38                       // ring entries of 8 columns: 288 / 8 = 36 entries, + the running one + 1
#define SB_VL_NB8D 67                      // the same when the walk is deferred (one look-up per 6-step chunk): entry e - k is read 6 k steps after the
                                           // trigger, by when the writer is 0.75 k entries further: 1.75 x 37 entries, + 2
#define SB_VL_ENTRY (SB_VL_FR * 4)         // uint4 per ring entry of a CTA: [16-slot group][code block]

// L2 eviction priority of the ring traffic and of the soft-value stream (kernel argument `flags`): the ring is re-used in place every 300
// columns, the soft values are read once.  bit 0: ring stores and look-ups evict_last; bit 1: soft-value loads evict_first.
#ifndef SB_HOST_EMU
__device__ __forceinline__ uint64_t vl_policy(const int kind) {          // 0 normal, 1 evict_last, 2 evict_first
    uint64_t p;
    if (kind == 1) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    else if (kind == 2) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    else asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void vl_st128(uint4* p, const uint4 w, const uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1, %2, %3, %4}, %5;" :: "l"(p), "r"(w.x), "r"(w.y), "r"(w.z), "r"(w.w), "l"(pol) : "memory");
}
__device__ __forceinline__ uint32_t vl_ld8(const uint8_t* p, const uint64_t pol) {
    uint32_t v; asm volatile("ld.global.cg.L2::cache_hint.u8 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol) : "memory"); return v;
}
__device__ __forceinline__ uint2 vl_ld64(const uint8_t* p, const uint64_t pol) {
    uint2 v; asm volatile("ld.global.nc.L2::cache_hint.v2.b32 {%0, %1}, [%2], %3;" : "=r"(v.x), "=r"(v.y) : "l"(p), "l"(pol)); return v;
}
#else        // host emulation: plain memory
inline uint64_t vl_policy(const int) { return 0; }
inline void vl_st128(uint4* p, const uint4 w, const uint64_t) { *p = w; }
inline uint32_t vl_ld8(const uint8_t* p, const uint64_t) { return *p; }
inline uint2 vl_ld64(const uint8_t* p, const uint64_t) { return *(const uint2*)p; }
#endif

// Windowed traceback from slot A0 at time t over la + nout columns (viterbi.hpp:205-237), by one lane for its own code block.
// The newest block (kp = t mod 6 columns; 0 = a whole one) is in ring entry e.  Walking n columns back from a slot replaces its
// top n address bits by the reversed history bits of those columns (column c was produced at phase (c - 1) mod 6, which replaces
// address bit 5 - phase); the decoded bits are the history bits themselves, newest first.  The first la bits are only looked
// through; after them every eight bits make one output byte, newest bit in bit 7, the LAST byte of the window first (op[first + nbytes - 1]).
// A free function of plain values, kept out of line: it runs once per `depth` steps and must not sit in the instruction stream of the
// step loop — and the decoder's registers must never have their address taken.
__device__ __noinline__ void vl_traceback(const uint8_t* __restrict__ ring_b, uint8_t* __restrict__ op, const uint32_t out_cap, uint32_t e,
                                          const uint32_t A0, const uint32_t t, const uint32_t la, const uint32_t nout, const uint32_t first, const uint64_t pol) {
    constexpr uint32_t EB = SB_VL_ENTRY * 16u;          // bytes per ring entry of the CTA
    uint32_t A = A0, todo = la + nout, acc = 0;
    int nb = -(int)la;                                   // valid bits in acc (negative: still inside the look-ahead)
    uint32_t at = first + (nout >> 3);                   // the next output byte goes to op[at - 1]
    uint32_t eo = e * EB;                                // byte offset of the ring entry the walk stands in (32-bit arithmetic throughout)
    auto emit = [&]() { if (nb >= 8) { --at; if (at < out_cap) op[at] = (uint8_t)(acc >> (nb - 8)); nb -= 8; } };   // at most one byte per block: nb < 8 before it
    auto back = [&]() { eo = eo ? eo - EB : (SB_VL_NB - 1u) * EB; };
    auto hist = [&]() { return vl_ld8(ring_b + (eo + (A >> 4) * (SB_VL_FR * 16u) + (A & 15u)), pol) & 63u; };
    const uint32_t kp = t % 6u;
    if (kp) {                                            // running block: kp columns, history bits kp-1 .. 0 (todo >= 8 > kp always)
        const uint32_t h = hist(), low = (1u << (6u - kp)) - 1u;
        acc = h & ((1u << kp) - 1u); nb += (int)kp;
        A = (A & low) | ((__brev(h) >> 26) & ~low);
        todo -= kp; back(); emit();
    }
#pragma unroll 1
    while (todo >= 6u) {                                 // whole blocks: six decoded bits per look-up, the slot six columns back is the reversed byte
        const uint32_t h = hist();
        acc = (acc << 6) | h; nb += 6;
        A = __brev(h) >> 26;
        todo -= 6u; back(); emit();
    }
    if (todo) { acc = (acc << todo) | (hist() >> (6u - todo)); nb += (int)todo; emit(); }   // the old end of the window: only the newest columns of its block count
}

// The same walk over EIGHT-column history blocks (HB = 8: 64 B of ring per 8 columns instead of per 6, 38 entries instead of 50; the block
// boundary then falls on any even phase).  Eight decoded bits per look-up; the slot eight columns back is the bit permutation of
// viterbi_k7_re.cuh's vr_traceback: address bit (i - ph) mod 6 <- decision of column tt - i, the two oldest columns overriding i = 0, 1.
__device__ __noinline__ void vl_traceback8(const uint8_t* __restrict__ ring_b, uint8_t* __restrict__ op, const uint32_t out_cap, uint32_t e,
                                           const uint32_t A0, const uint32_t t, const uint32_t la, const uint32_t nout, const uint32_t first, const uint64_t pol) {
    constexpr uint32_t EB = SB_VL_ENTRY * 16u;
    uint32_t A = A0, todo = la + nout, acc = 0;
    int nb = -(int)la;
    uint32_t at = first + (nout >> 3);
    uint32_t eo = e * EB;
    auto emit = [&]() { if (nb >= 8) { --at; if (at < out_cap) op[at] = (uint8_t)(acc >> (nb - 8)); nb -= 8; } };   // nb < 8 before a block, < 16 after it
    auto back = [&]() { eo = eo ? eo - EB : (SB_VL_NB8 - 1u) * EB; };
    auto hist = [&]() { return vl_ld8(ring_b + (eo + (A >> 4) * (SB_VL_FR * 16u) + (A & 15u)), pol); };
    uint32_t tt = t;                                     // time of the newest column not yet walked
    const uint32_t kp = t & 7u;
    if (kp) {                                            // running block: kp columns, one slot-address bit changes per column
        const uint32_t h = hist();
        for (uint32_t c = 0; c < kp; c++) {              // column tt - c was produced at phase (tt - c - 1) mod 6: bit 5 - phase is replaced
            const uint32_t b = 5u - (tt - c - 1u) % 6u, d = (h >> (kp - 1u - c)) & 1u;
            A = (A & ~(1u << b)) | (d << b);
        }
        acc = h & ((1u << kp) - 1u); nb += (int)kp;
        todo -= kp; tt -= kp; back(); emit();
    }
    uint32_t ph = tt % 6u;                               // phase of the block boundary the walk stands on
#pragma unroll 1
    while (todo >= 8u) {
        const uint32_t h = hist();
        acc = (acc << 8) | h; nb += 8;
        const uint32_t r = __brev(h) >> 24;              // r bit i = h bit 7 - i = decision of column tt - i
        const uint32_t G = (r & 0x3Cu) | (r >> 6);
        A = ((G | (G << 6)) >> ph) & 63u;
        todo -= 8u; ph = ph >= 2u ? ph - 2u : ph + 4u;   // (tt - 8) mod 6
        back(); emit();
    }
    if (todo) { acc = (acc << todo) | (hist() >> (8u - todo)); nb += (int)todo; emit(); }
}

// HB: columns per history block, 6 (the trellis period: constants everywhere, the smallest loop body) or 8 (a quarter less ring traffic and
// a smaller ring; the mark of a step and the block boundaries become run-time, warp-uniform values).
// DEFER (HB = 8 only): the walk does not happen at the trigger.  Every look-up of a walk is a dependent L2 / HBM round trip of ~1 400 cycles,
// 34 of them per window, and ncu's source view puts 30 % of all stall samples on the one instruction that consumes the loaded byte; other warps
// do not cover that (starting them apart changes nothing, a walk prefetching its window neither — measured).  So the trigger only records where
// the walk starts and issues its first load; after that the step loop performs ONE look-up per 6-step chunk — consume the byte loaded a chunk
// ago, move to the slot eight columns back, issue the next load — and the forward pass never waits: a window's walk is finished 37 chunks =
// 222 steps after its trigger, before the next trigger (256 steps).  The ring keeps 29 more entries for the walk to still find its oldest ones.
template <int CODE_RATE, int HB, bool DEFER = false>
struct VlDecoder {
    static_assert(!DEFER || HB == 8, "the deferred walk is written for 8-column history blocks");
    static constexpr uint32_t NB = HB == 6 ? SB_VL_NB : DEFER ? SB_VL_NB8D : SB_VL_NB8;
    uint32_t wk_todo, wk_A, wk_eo, wk_acc, wk_at, wk_ph, wk_h; int wk_nb;      // deferred walk: columns left (0 = none in flight), slot, ring entry
                                                                               // offset, bit accumulator, next output byte, phase, the byte in flight, valid bits
    static constexpr uint32_t GROUP = CODE_RATE == CR_12 ? 2u : CODE_RATE == CR_34 ? 4u : 3u;   // soft bytes per puncture group
    static constexpr uint32_t GSTEPS = CODE_RATE == CR_12 ? 1u : CODE_RATE == CR_34 ? 3u : 2u;  // trellis steps per group
    static constexpr uint32_t CHUNK_BYTES = 6u / GSTEPS * GROUP;                                // soft bytes per 6 steps
    uint32_t R[32];        // slot address = register << 1 | half; state index of a slot at time t = rol6(address, t mod 6)
    VrLane LC;             // selectors of vr_step: constants here (no lane part), kept in the struct the step function takes
    uint32_t kc[2];        // 28 << 8 and 14 << 8 in both halves
    uint32_t mk[5], mkH, mkL;   // history mark of phase T = 0x00010001 << T as registers (IMAD-side adds, see vr_step); phase 5 split by half
    uint4* ring_q; const uint8_t* ring_b; uint64_t pol_ring, pol_soft;
    const uint8_t* sp; uint8_t* op; uint32_t out_cap, nsoft;
    uint32_t depth, look, end, ob, next_tb, nraw, wslot;
    bool done;

    __device__ __forceinline__ void fetch(const uint32_t pos, uint32_t (&a)[3]) const {
        if (pos + CHUNK_BYTES > nsoft) { a[0] = a[1] = a[2] = 0; return; }
        if constexpr (CODE_RATE == CR_34) { const uint2 v = vl_ld64(sp + pos, pol_soft); a[0] = v.x; a[1] = v.y; a[2] = 0; }
        else if constexpr (CODE_RATE == CR_12) { a[0] = __ldg((const uint32_t*)(sp + pos)); a[1] = __ldg((const uint32_t*)(sp + pos + 4)); a[2] = __ldg((const uint32_t*)(sp + pos + 8)); }
        else { uint32_t b[9];
#pragma unroll
               for (int i = 0; i < 9; i++) b[i] = __ldg(sp + pos + i);
               a[0] = b[0] | (b[1] << 8) | (b[2] << 16); a[1] = b[3] | (b[4] << 8) | (b[5] << 16); a[2] = b[6] | (b[7] << 8) | (b[8] << 16); }
    }
    // the 64 history bytes of this code block (low byte of every half, slot-address order) into ring entry e
    __device__ __forceinline__ void store_hist(const uint32_t e) {
#pragma unroll
        for (int i = 0; i < 4; i++) {
            uint4 w;
            w.x = __byte_perm(R[8 * i + 0], R[8 * i + 1], 0x6420); w.y = __byte_perm(R[8 * i + 2], R[8 * i + 3], 0x6420);
            w.z = __byte_perm(R[8 * i + 4], R[8 * i + 5], 0x6420); w.w = __byte_perm(R[8 * i + 6], R[8 * i + 7], 0x6420);
            vl_st128(ring_q + e * SB_VL_ENTRY + i * SB_VL_FR, w, pol_ring);
        }
    }
    __device__ __forceinline__ void clear_hist() {
#pragma unroll
        for (int r = 0; r < 32; r++) R[r] &= 0xFE00FE00u;
    }
    __device__ __forceinline__ void next_slot() { wslot = wslot == NB - 1u ? 0u : wslot + 1u; }
    // viterbi.hpp:177-180 -> viterbicore.h:445-465: subtract the smallest m7 from every metric
    __device__ __forceinline__ void normalize() {
        uint32_t m = R[0];
#pragma unroll
        for (int r = 1; r < 32; r++) m = __vminu2(m, R[r]);
        m = min(m & 0xFFFFu, m >> 16) >> 9;
        const uint32_t mv = m * 0x02000200u;
#pragma unroll
        for (int r = 0; r < 32; r++) R[r] -= mv;        // every half >= m << 9: no borrow between halves, histories untouched
    }
    // slot of the best state at time t (tm = t mod 6, tn = (t - 1) mod 6 = bit of the newest mark), viterbicore.h:468-520
    __device__ __forceinline__ uint32_t best_slot(const uint32_t tm, const uint32_t tn) const { return vr_best_core<0>(R, 0u, tm, tn, 0u); }

    // traceback trigger at time t (a puncture-group boundary), viterbi.hpp:182-203; tm = t mod 6
    __device__ __forceinline__ void trigger(const uint32_t t, const uint32_t tm) {
        if (t < next_tb) return;
        uint32_t nout, la;
        if (t >= end) { nout = end - ob - 6u; la = t - end; }
        else { nout = depth; la = look + (t - (ob + depth + look + 6u)) % 8u; }
        if (nout) {
            const uint32_t A0 = best_slot(tm, HB == 6 ? (tm ? tm - 1u : 5u) : ((t - 1u) & 7u));
            if (HB == 6 ? tm != 0u : (t & 7u) != 0u) store_hist(wslot);   // mid-block: the partial histories of the running block (a block end has just stored its own)
            if constexpr (HB == 6) vl_traceback(ring_b, op, out_cap, wslot, A0, t, la, nout, nraw, pol_ring);
            else if constexpr (DEFER) walk_start(A0, t, la, nout);
            else vl_traceback8(ring_b, op, out_cap, wslot, A0, t, la, nout, nraw, pol_ring);
            nraw += nout >> 3; ob += nout;
        }
        if (ob + 6u >= end && t >= end) done = true;
        next_tb = min(end, ob + depth + look + 6u);
        if (next_tb <= t) next_tb = t + 1u;              // a frame shorter than the prefix: re-evaluate at every group
    }
    // ---- deferred walk (DEFER): vl_traceback8 cut into its look-ups ----
    __device__ __forceinline__ uint32_t walk_load() const {
        return vl_ld8(ring_b + (wk_eo + (wk_A >> 4) * (SB_VL_FR * 16u) + (wk_A & 15u)), pol_ring);
    }
    __device__ __forceinline__ void walk_back() { wk_eo = wk_eo ? wk_eo - SB_VL_ENTRY * 16u : (NB - 1u) * (SB_VL_ENTRY * 16u); }
    __device__ __forceinline__ void walk_emit() { if (wk_nb >= 8) { --wk_at; if (wk_at < out_cap) op[wk_at] = (uint8_t)(wk_acc >> (wk_nb - 8)); wk_nb -= 8; } }
    // one look-up: consume the byte in flight, step eight columns back (or finish with the newest columns of the window's oldest block), load the next
    __device__ __forceinline__ void walk_tick() {
        if (wk_todo == 0u) return;
        const uint32_t h = wk_h;
        if (wk_todo >= 8u) {
            wk_acc = (wk_acc << 8) | h; wk_nb += 8;
            const uint32_t r = __brev(h) >> 24;                          // r bit i = h bit 7 - i = decision of column tt - i
            const uint32_t G = (r & 0x3Cu) | (r >> 6);
            wk_A = ((G | (G << 6)) >> wk_ph) & 63u;
            wk_todo -= 8u; wk_ph = wk_ph >= 2u ? wk_ph - 2u : wk_ph + 4u;
            walk_back(); walk_emit();
            if (wk_todo) wk_h = walk_load();
        } else { wk_acc = (wk_acc << wk_todo) | (h >> (8u - wk_todo)); wk_nb += (int)wk_todo; wk_todo = 0u; walk_emit(); }
    }
    __device__ __forceinline__ void walk_drain() { while (wk_todo) walk_tick(); }
    // at a trigger: finish a walk that is still in flight (windows shorter than a walk: standalone calls with a small depth), take the running
    // block at once (its entry was stored a moment ago), and leave the first whole-block load in flight
    __device__ __forceinline__ void walk_start(const uint32_t A0, const uint32_t t, const uint32_t la, const uint32_t nout) {
        walk_drain();
        wk_A = A0; wk_todo = la + nout; wk_acc = 0u; wk_nb = -(int)la; wk_at = nraw + (nout >> 3); wk_eo = wslot * (SB_VL_ENTRY * 16u);
        uint32_t tt = t; const uint32_t kp = t & 7u;
        if (kp) {
            const uint32_t h = walk_load();
            for (uint32_t c = 0; c < kp; c++) {                          // column tt - c was produced at phase (tt - c - 1) mod 6: bit 5 - phase is replaced
                const uint32_t b = 5u - (tt - c - 1u) % 6u, d = (h >> (kp - 1u - c)) & 1u;
                wk_A = (wk_A & ~(1u << b)) | (d << b);
            }
            wk_acc = h & ((1u << kp) - 1u); wk_nb += (int)kp;
            wk_todo -= kp; tt -= kp; walk_back(); walk_emit();
        }
        wk_ph = tt % 6u;
        if (wk_todo) wk_h = walk_load();
    }

    template <int s> __device__ __forceinline__ void step(const uint32_t cb, const uint32_t tb) {
        const uint32_t KC = kc[vr_ksum<CODE_RATE, s>() == 28u ? 0 : 1];
        if constexpr (HB == 8) vr_step_rt<s, true, 0>(R, cb, LC, KC, 0x00010001u << ((tb + s) & 7u), 0xFFFFFFFFu);    // tb is warp-uniform: the mark lives in a uniform register
        else if constexpr (s <= 4) vr_step<s, true, 0>(R, cb, LC, KC, mk[s], 0u, 0xFFFFFFFFu);
        else vr_step<5, true, 0>(R, cb, LC, KC, mkH, mkL, 0xFFFFFFFFu);
    }
    // steps s .. 5 of the 6-step chunk that starts at time tb (a multiple of 6).  CHECK = false: no traceback trigger falls into the
    // chunk for any lane of the warp (the hot loop); CHECK = true: every group boundary is checked, lanes that are not `live` only keep step.
    // Normalisation (viterbi.hpp:177-180) comes when (t & 7) == 0 at a group boundary: t is even only after an odd s.
    template <int s, bool CHECK> __device__ __forceinline__ void chunk(const uint32_t (&w)[3], const uint32_t tb, const bool live) {
        if constexpr (s < 6) {
            step<s>(vr_bm<CODE_RATE, s>(w), tb);
            const uint32_t t = tb + s + 1u;
            // block boundary: HB = 6 after the last step of every chunk; HB = 8 when (t & 7) == 0, which only an odd s can reach (tb is even)
            const bool blk = HB == 6 ? s == 5 : ((s & 1) && (t & 7u) == 0u);
            if (blk) store_hist(wslot);
            if constexpr ((s + 1) % GSTEPS == 0) {
                if constexpr (s & 1) { if ((t & 7u) == 0u) normalize(); }
                if constexpr (CHECK) { if (live && !done) trigger(t, (s + 1) % 6); }
            }
            if (blk) { clear_hist(); next_slot(); }
            chunk<s + 1, CHECK>(w, tb, live);
        }
    }
};

// list / cnt: work list of this code rate (k_vit_lists) or null = frames 0 .. nframes-1 with the uniform parameters of `job`.
// 16 resident one-warp CTAs per SM = 128 registers per thread, the out-of-line traceback included (without the bound the callee's own
// registers are added on top and the SM holds 12 warps: measured 4.8 ms instead of 4.2).
// gring: SB_VL_NB * SB_VL_ENTRY uint4 per CTA.
template <int CODE_RATE, int HB = 6, bool DEFER = false>
__global__ void __launch_bounds__(32, 16) k_viterbi_lane(const uint8_t* __restrict__ soft, uint64_t soft_stride, uint32_t nframes,
        const uint32_t* __restrict__ list, const uint32_t* __restrict__ cnt, const FrameInfo* __restrict__ info, VitJob job,
        uint8_t* __restrict__ out, uint64_t out_stride, uint32_t raw_off, uint32_t* __restrict__ nraw_out, uint4* __restrict__ gring, uint32_t flags) {
    using D = VlDecoder<CODE_RATE, HB, DEFER>;
    constexpr unsigned FULL = 0xFFFFFFFFu;
    const uint32_t nvalid = list ? __ldg(cnt + CODE_RATE) : (job.code_rate == (uint32_t)CODE_RATE ? nframes : 0u);
    if (blockIdx.x * SB_VL_FR >= nvalid) return;        // whole CTA
    const int lane = threadIdx.x & 31;
    const uint32_t idx = blockIdx.x * SB_VL_FR + lane;
    const bool valid = idx < nvalid;
    const uint32_t f = !valid ? 0u : list ? __ldg(list + (size_t)CODE_RATE * nframes + idx) : idx;
    uint32_t L = job.frame_len;
    D d;
    d.nsoft = job.nsoft;
    if (valid && info) { const FrameInfo fi = info[f]; L = fi.length; d.nsoft = fi.soft_bytes; }
    if (!valid) d.nsoft = 0;
    d.depth = job.depth; d.look = job.lookahead;
    d.sp = soft + (size_t)f * soft_stride;
    d.op = out + (size_t)f * out_stride + raw_off;
    d.out_cap = (uint32_t)(out_stride - raw_off < 0xFFFFFFFFull ? out_stride - raw_off : 0xFFFFFFFFull);
#pragma unroll
    for (int t = 0; t < 6; t++) {                        // no lane part in the slot address: the selectors are constants
        const int K = vr_kcls(t);
        d.LC.sel[t][0] = vq_sel(0, 0 ^ K); d.LC.sel[t][1] = vq_sel(1, 1 ^ K);
    }
    d.LC.bA[0] = d.LC.bA[1] = 0u; d.LC.bB[0] = d.LC.bB[1] = 0u;
    {   // constants that must stay register operands (z is always 0, which the compiler cannot know): see vr_step
        const uint32_t z = (uint32_t)(soft_stride >> 63);
        d.kc[0] = 0x1C001C00u + z; d.kc[1] = 0x0E000E00u + z;
#pragma unroll
        for (int j = 0; j < 5; j++) d.mk[j] = (0x00010001u << j) + z;
        d.mkH = 0x00200000u + z; d.mkL = 0x00000020u + z;
    }
    // initial metrics (viterbilut.h:22-32): state 0 -> 0x00, others 0x30; at t = 0 state == address; byte value v sits at v << 8
#pragma unroll
    for (int r = 0; r < 32; r++) d.R[r] = 0x30003000u;
    d.R[0] = 0x30000000u;
    d.end = L * 8u + 16u + 6u; d.ob = 0; d.nraw = 0; d.wslot = 0; d.done = !valid; d.wk_todo = 0u;
    d.next_tb = min(d.end, d.depth + d.look + 6u);      // first time a traceback can fire (viterbi.hpp:182-203)
    uint4* const ring0 = gring + (size_t)blockIdx.x * (D::NB * SB_VL_ENTRY);
    d.ring_q = ring0 + lane; d.ring_b = (const uint8_t*)(ring0 + lane);
    d.pol_ring = vl_policy((flags & 1u) ? 1 : 0); d.pol_soft = vl_policy((flags & 2u) ? 2 : 0);

    // lockstep part: the 32 code blocks of the warp advance together, one 6-step chunk per iteration; the soft values of the next two
    // chunks are always in registers
    uint32_t tb = 0, pos = 0;                           // time and soft position at the start of the next chunk (uniform)
    // Soft values: w0 is the chunk being decoded, w1 the next one, w2 is loaded at the top of the iteration.  (Keeping a load in flight for
    // two chunks in alternating registers, so that not even the rotating move touches it early, was measured: the move's stall samples went
    // away and the kernel got 3 % slower — it is bound by the ALU pipe, and the parity branches cost more than the wait they removed.)
    uint32_t w0[3], w1[3];
    d.fetch(pos, w0); d.fetch(pos + D::CHUNK_BYTES, w1);
    // tail: the whole puncture groups of a code block that do not fill a 6-step chunk, per lane, phases at run time (tb, pos: the start of
    // the chunk the lane could not fill).  A lane runs it once, as soon as it has no whole chunk left, also while other lanes of the warp still
    // have chunks to step (802.11n symbols of 52, 104, 208 and 416 trellis steps leave a partial chunk at the end of a frame,
    // and the flush point may lie in it).  After it the lane is done; it keeps step on zeros without triggers, like a lane that ended in the loop.
    auto tail = [&](uint32_t tb, uint32_t pos) {
        uint32_t k = 0;                                 // steps into the chunk at tb
        auto step_rt = [&](const uint32_t cb, const uint32_t KC) {
            const uint32_t mark = 0x00010001u << (HB == 6 ? k : ((tb + k) & 7u));
            switch (k) { case 0: vr_step_rt<0, false, 0>(d.R, cb, d.LC, KC, mark, FULL); break; case 1: vr_step_rt<1, false, 0>(d.R, cb, d.LC, KC, mark, FULL); break;
                         case 2: vr_step_rt<2, false, 0>(d.R, cb, d.LC, KC, mark, FULL); break; case 3: vr_step_rt<3, false, 0>(d.R, cb, d.LC, KC, mark, FULL); break;
                         case 4: vr_step_rt<4, false, 0>(d.R, cb, d.LC, KC, mark, FULL); break; default: vr_step_rt<5, false, 0>(d.R, cb, d.LC, KC, mark, FULL); }
            k++;
            if ((tb + k) % (uint32_t)HB == 0u) d.store_hist(d.wslot);
        };
        auto block_end = [&]() { if ((tb + k) % (uint32_t)HB == 0u) { d.clear_hist(); d.next_slot(); } };
        while (!d.done && pos + D::GROUP <= d.nsoft) {
            uint32_t g = __ldg(d.sp + pos) | ((uint32_t)__ldg(d.sp + pos + 1) << 8);
            if (D::GROUP > 2) g |= (uint32_t)__ldg(d.sp + pos + 2) << 16;
            if (D::GROUP > 3) g |= (uint32_t)__ldg(d.sp + pos + 3) << 24;
            pos += D::GROUP;
            step_rt(vq_bm_ab<0>(g), d.kc[0]);
            if (D::GSTEPS >= 2) { block_end(); step_rt(vq_bm_a<2>(g), d.kc[1]); }
            if (D::GSTEPS >= 3) { block_end(); step_rt(vq_bm_b<3>(g), d.kc[1]); }
            const uint32_t t = tb + k;
            if ((t & 7u) == 0u) d.normalize();
            d.trigger(t, k == 6u ? 0u : k);
            block_end();
            if (k == 6u) { k = 0; tb += 6u; }
        }
        d.done = true;
    };
#pragma unroll 1
    for (;;) {
        const bool more = !d.done && pos + D::CHUNK_BYTES <= d.nsoft;
        if (!__any_sync(FULL, more)) break;
        uint32_t w2[3];
        d.fetch(pos + 2u * D::CHUNK_BYTES, w2);
        if constexpr (DEFER) d.walk_tick();                 // one look-up of the window in flight (its load was issued a chunk ago)
        const bool quiet = d.done || (more && tb + 6u < d.next_tb);
        if (__all_sync(FULL, quiet)) d.template chunk<0, false>(w0, tb, more);
        else {                                          // a lane out of whole chunks is never quiet: its tail runs here, once per code block
            if (!more && !d.done) tail(tb, pos);
            d.template chunk<0, true>(w0, tb, more);
        }
#pragma unroll
        for (int i = 0; i < 3; i++) { w0[i] = w1[i]; w1[i] = w2[i]; }
        tb += 6u; pos += D::CHUNK_BYTES;
    }
    if (!d.done) tail(tb, pos);                         // the warp ran out together
    if constexpr (DEFER) d.walk_drain();                    // the last window's walk
    if (valid) nraw_out[f] = d.nraw;
}

} // namespace sb
