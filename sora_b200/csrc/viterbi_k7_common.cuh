// sora_b200 — what the K=7 (133,171) Viterbi kernels share: the frame record handed from kernel to kernel, the branch-metric construction
// and the history-carrying add-compare-select step (vr_step) with its helpers.  Device functions only — no kernel, no table, no CUDA runtime
// call — so that tests/cpp/lane_emu.cpp and tests/cpp/re_emu.cpp can compile the one-lane and the four-lane kernels for the HOST (every
// intrinsic they need is a few lines of C++ in tests/cpp/warp_emu.h) and run the very code the GPU runs against the CPU oracle without a GPU.
// Arithmetic contract and machine mapping: see viterbi_k7_re.cuh (history-carrying metrics, in-place trellis).
#pragma once
#include <stdint.h>
#include "tx_frames.cuh"                     // CR_12 / CR_23 / CR_34

namespace sb {

enum : uint32_t {
    E_SUCCESS = 0, E_FRAME_OK = 1, E_FAILED = 0x8000FFFFu, E_PLCP_HEADER_FAIL = 0x80000005u,
    E_CRC32_FAIL = 0x80000006u, E_CS_TIMEOUT = 0x80000007u, E_NO_FRAME = 0x8000F001u,
};

struct FrameInfo {            // per-slot state handed from kernel to kernel (device memory)
    uint32_t status;          // E_SUCCESS while decoding proceeds, else terminal code
    uint32_t detect_vec;      // index of the first 20 Msps 4-sample vector routed to the demod branch
    uint32_t rate_kbps, length, nsym_total, code_rate, ncbps;
    uint32_t soft_bytes;      // deinterleaved soft values written for this frame
    int32_t cfo_est; uint32_t peak_index;
    int32_t dc_re, dc_im;     // CF_VecDC when the carrier sense ended (it persists across frames of one stream)
};

struct VitJob {               // uniform-parameter mode (standalone API); per-frame mode reads FrameInfo instead
    uint32_t code_rate, frame_len, nsoft; uint32_t depth, lookahead; uint32_t raw; // raw=1: emit SERVICE+PSDU bytes undescrambled
};


__host__ __device__ constexpr int vq_rol6(int a, int t) { return ((a << t) | (a >> (6 - t))) & 63; }
__host__ __device__ constexpr int vq_cls(int p) {            // (cA << 1) | cB of predecessor index p (bit 5 ignored)
    return ((((p >> 1) ^ (p >> 2) ^ (p >> 4)) & 1) << 1) | ((p ^ (p >> 1) ^ (p >> 2)) & 1);
}
// PRMT selector building [m0, byte i0, m2, byte i1] from (Cb, m): the branch metric lands in the high byte of each half, the low byte of each
// half comes from byte 0 / byte 2 of m — zero for m = 0, the history mark of the half for m = a mark (0x00010001 << j or one half of it)
__host__ __device__ constexpr unsigned vq_sel(int i0, int i1) { return (unsigned)(4 | (i0 << 4) | (6 << 8) | (i1 << 12)); }

// branch-metric byte vectors (byte index = cA<<1 | cB) from soft values in bytes B0 (A) and B0+1 (B) of the packed word w
#ifndef SB_HOST_EMU
__device__ __forceinline__ int vq_dp4a_us(uint32_t a, int b, int c) { int d; asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
#else        // host emulation: unsigned bytes of a times signed bytes of b, accumulated
inline int vq_dp4a_us(uint32_t a, int b, int c) { for (int i = 0; i < 4; i++) c += (int)((a >> (8 * i)) & 0xFFu) * (int)(int8_t)((uint32_t)b >> (8 * i)); return c; }
#endif
template <int B0> __device__ __forceinline__ uint32_t vq_bm_ab(uint32_t w) {
    // x = tA + tB, y = tA - tB + 14;  bytes [x, y, 28 - y, 28 - x] = c00, c01, c10, c11
    const int x = vq_dp4a_us(w, (int)(0x0202u << (8 * B0)), 0);
    const int y = vq_dp4a_us(w, (int)(0xFE02u << (8 * B0)), 14);
    return 0x1C1C0000u + (uint32_t)x * 0xFF000001u + (uint32_t)y * 0xFFFF0100u;
}
template <int B0> __device__ __forceinline__ uint32_t vq_bm_a(uint32_t w) {      // only A present: bytes [c0, c0, c1, c1]
    const int s = vq_dp4a_us(w, (int)(0x01u << (8 * B0)), 0);
    return 0x0E0E0000u + (uint32_t)s * (0x00000202u - 0x02020000u);
}
template <int B0> __device__ __forceinline__ uint32_t vq_bm_b(uint32_t w) {      // only B present: bytes [c0, c1, c0, c1]
    const int s = vq_dp4a_us(w, (int)(0x01u << (8 * B0)), 0);
    return 0x0E000E00u + (uint32_t)s * (0x00020002u - 0x02000200u);
}

// low four address bits of (register r, half h): r << 1 | h — the order in which the PRMT gather of store_hist lays a lane's 16 history bytes down
__host__ __device__ constexpr int vr_low4(int r, int h) { return (r << 1) | h; }
__host__ __device__ constexpr int vr_scls(int T, int r, int h) { return vq_cls(vq_rol6(vr_low4(r, h), T) & 31); }
__host__ __device__ constexpr int vr_kcls(int T) { return vq_cls(vq_rol6(1, T) & 31); }     // class difference between the two halves of a register

// adds that must run on the FMA pipe (IMAD), not the ALU pipe the add-min and the PRMTs already fill: ptxas picks the pipe of a plain `+` itself
#ifndef SB_HOST_EMU
__device__ __forceinline__ uint32_t vr_fadd(uint32_t a, uint32_t b) { uint32_t d; asm("mad.lo.u32 %0, %1, 1, %2;" : "=r"(d) : "r"(a), "r"(b)); return d; }
__device__ __forceinline__ uint32_t vr_frsub(uint32_t v, uint32_t k) { uint32_t d; asm("mad.lo.u32 %0, %1, 0xFFFFFFFF, %2;" : "=r"(d) : "r"(v), "r"(k)); return d; }   // k - v
#else        // host emulation (tests/cpp/lane_emu.cpp): the same values without PTX
inline uint32_t vr_fadd(uint32_t a, uint32_t b) { return a + b; }
inline uint32_t vr_frsub(uint32_t v, uint32_t k) { return k - v; }
#endif

struct VrLane {
    unsigned sel[6][4];    // per phase: PRMT selectors building [0, Cb[c], 0, Cb[c ^ K]] straight from the class-indexed branch-metric bytes, this
                           // lane's class contribution folded in (Cb[i] = Cbase[i ^ lane class]); c = 0, 1 (lane kernel), c = 0..3 (four-lane kernel)
    uint32_t bA[2], bB[2]; // lane-pair phases: 1 if the history mark of the step goes to my own value / to my partner's (exactly one is set)
};

// The add-compare-select of one trellis step at compile-time phase T (= (t - 1) mod 6 for the step that produces column t), from the
// constants of its two candidates: P[c] is added to the candidate that keeps its slot and Q[c] to the one that comes from the partner slot,
// c = the class of the even candidate's predecessor (see vr_step).
// WARP: the whole warp executes the step together (full-mask shuffle).
// LB = lane bits of the slot address: 2 = four lanes per code block, 8 registers per lane (slot = lane << 4 | reg << 1 | half; k_viterbi_re);
//                                      0 = one lane per code block, 32 registers (slot = reg << 1 | half; k_viterbi_lane).
// The address bit replaced at phase T is bit 5 - T: a lane bit for T < LB (exchange with lane xor 1 << (LB - 1 - T)), a register bit for
// LB <= T <= 4 (pair r, r + (1 << (4 - T))), the half for T = 5.
template <int T, bool WARP, int LB>
__device__ __forceinline__ void vr_acs(uint32_t (&R)[8 << (2 - LB)], const uint32_t (&P)[4], const uint32_t (&Q)[4], const unsigned qmask) {
    constexpr int NR = 8 << (2 - LB);
    if constexpr (T < LB) {                             // pair = partner lane: the path-metric exchange
#pragma unroll
        for (int r = 0; r < NR; r++) {
            const int c0 = vr_scls(T, r, 0);
            const uint32_t Z = __shfl_xor_sync(WARP ? 0xFFFFFFFFu : qmask, R[r], 1 << (LB - 1 - T));
            R[r] = __viaddmin_u16x2(R[r], P[c0], __vadd2(Z, Q[c0 ^ 3]));
        }
    } else if constexpr (T <= 4) {                      // pair = register r ^ d inside the lane
        constexpr int d = 1 << (4 - T);
#pragma unroll
        for (int r = 0; r < NR; r++) {
            if (r & d) continue;
            const int c0 = vr_scls(T, r, 0);
            const uint32_t X = R[r], Y = R[r + d];      // X = states p (even role), Y = states p + 32 (odd role)
            R[r]     = __viaddmin_u16x2(X, P[c0], __vadd2(Y, Q[c0 ^ 3]));
            R[r + d] = __viaddmin_u16x2(Y, Q[c0], __vadd2(X, P[c0 ^ 3]));
        }
    } else {                                            // pair = the two halves of each register: low = p, high = p + 32
#pragma unroll
        for (int r = 0; r < NR; r++) {
            const int c = vr_scls(5, r, 0);
            const uint32_t y = __byte_perm(R[r], 0, 0x1032);          // [p + 32, p]
            R[r] = __viaddmin_u16x2(R[r], P[c], __vadd2(y, Q[c ^ 3]));     // [min(p + a, p32 + b), min(p32 + a, p + b)] = new states 2p, 2p + 1
        }
    }
}
// One trellis step of the lane kernel (LB = 0).  Cbase byte (cA<<1|cB) = metric of the even candidate for a predecessor of that class; the
// complement class (3 - index) is the odd candidate's and equals KC - it per half (KC = 28 << 8 per half when both coded bits are present,
// 14 << 8 when one is punctured; a register like the marks).  The odd candidate (state p+32) carries the history mark of the step,
// 0x00010001 << ((t-1) mod 8):  T <= 4 : mA = mark;   T = 5 : mA = mark << 16 part, mB = low part.
// The marks come in as registers so that every constant add stays one register add (scalar VIADD or IMAD.IADD, both FMA pipe).
template <int T, bool WARP, int LB>
__device__ __forceinline__ void vr_step(uint32_t (&R)[8 << (2 - LB)], const uint32_t Cbase, const VrLane& L, const uint32_t KC, const uint32_t mA, const uint32_t mB, const unsigned qmask) {
    static_assert(LB == 0, "the four-lane kernel steps through vr_step_pk");
    uint32_t V[4], P[4], Q[4];                          // V = [0, Cb[c], 0, Cb[c ^ K]]: branch metrics of class c (low half) and its high-half companion
    V[0] = __byte_perm(Cbase, 0, L.sel[T][0]); V[1] = __byte_perm(Cbase, 0, L.sel[T][1]);
    V[3] = vr_frsub(V[0], KC); V[2] = vr_frsub(V[1], KC);                 // complement classes; no borrow: every half of V is <= its half of KC
#pragma unroll
    for (int c = 0; c < 4; c++) {
        if constexpr (T <= 4) { P[c] = V[c]; Q[c] = vr_fadd(V[c], mA); }
        else { P[c] = vr_fadd(V[c], mA); Q[c] = vr_fadd(V[c], mB); }
    }
    vr_acs<T, WARP, LB>(R, P, Q, qmask);
}
// One trellis step of the four-lane kernel (LB = 2).  Issue pipes on sm_90 (tools/microbench/pipes2.cu, DESIGN §4): VIADDMNMX, PRMT, LOP3 and
// IADD3 take the ALU pipe; VIADD.16x2, IMAD, IDP.4A and the scalar VIADD the FMA pipe, and VIADDMNMX takes half an FMA slot as well.  So the
// ACS alone loads the FMA pipe more than the ALU pipe, and the constants of a step are built mostly on the ALU pipe: every one is a PRMT of
// the branch-metric word, whose byte for class 3 - i is the complement of the byte for class i (ksum - Cb[i], vr_bmbyte), so the selectors L.sel[T][c] name all four
// classes and no subtract is needed, and the selectors take the low byte of each half from the mark operand (vq_sel), so a marked constant
// costs no add.  Where an add to a constant already built is one instruction too (T = 2..5), the second candidate's constants are FMA-pipe
// adds, which balances the two pipes:
//   T <= 1 : P = PRMT(Cb, mP), Q = PRMT(Cb, mQ); mP = mark if this lane holds the odd role else 0, mQ = mark - mP;
//   T = 2..4 : P = PRMT(Cb, 0), Q = P + mQ; mQ = mark;   T = 5 : P = PRMT(Cb, mP), Q = P + mQ; mP = high half of the mark, mQ = low half - mP.
template <int T, bool WARP>
__device__ __forceinline__ void vr_step_pk(uint32_t (&R)[8], const uint32_t Cbase, const VrLane& L, const uint32_t mP, const uint32_t mQ, const unsigned qmask) {
    uint32_t P[4], Q[4];
#pragma unroll
    for (int c = 0; c < 4; c++) {
        P[c] = __byte_perm(Cbase, mP, L.sel[T][c]);
        Q[c] = T < 2 ? __byte_perm(Cbase, mQ, L.sel[T][c]) : vr_fadd(P[c], mQ);
    }
    vr_acs<T, WARP, 2>(R, P, Q, qmask);
}
// the same with the mark of the step given as a plain value (6-step path and tail: the time is only known at run time)
template <int T, bool WARP, int LB>
__device__ __forceinline__ void vr_step_rt(uint32_t (&R)[8 << (2 - LB)], const uint32_t Cbase, const VrLane& L, const uint32_t KC, const uint32_t mark, const unsigned qmask) {
    if constexpr (LB == 2) {
        if constexpr (T < 2) vr_step_pk<T, WARP>(R, Cbase, L, L.bA[T] * mark, L.bB[T] * mark, qmask);
        else if constexpr (T <= 4) vr_step_pk<T, WARP>(R, Cbase, L, 0u, mark, qmask);
        else vr_step_pk<T, WARP>(R, Cbase, L, mark & 0xFFFF0000u, (mark & 0x0000FFFFu) - (mark & 0xFFFF0000u), qmask);
    }
    else if constexpr (T <= 4) vr_step<T, WARP, LB>(R, Cbase, L, KC, mark, 0u, qmask);
    else vr_step<T, WARP, LB>(R, Cbase, L, KC, mark & 0xFFFF0000u, mark & 0x0000FFFFu, qmask);
}

// rate 3/4, four-lane kernel: the A-only and the B-only step of a puncture group (soft bytes 2 and 3 of w, values 0..7) from one multiply:
// bytes [2 tA, 2 tB, 14 - 2 tA, 14 - 2 tB] (no byte borrows from another); vr_bmbyte names the byte that holds a class's metric
__host__ __device__ __forceinline__ uint32_t vq_bm_a2b3(uint32_t w) { return 0x0E0E0000u + (w >> 16) * 0xFFFE0002u; }
// byte of the four-lane kernel's branch-metric word of phase t that holds the metric of class i = cA << 1 | cB; byte 3 - i of vq_bm_ab,
// vq_bm_a and vq_bm_b (and byte vr_bmbyte(3 - i) of vq_bm_a2b3) is the complement of the byte of class i
__host__ __device__ constexpr int vr_bmbyte(int code_rate, int t, int i) {
    return code_rate != CR_34 || t % 3 == 0 ? i : t % 3 == 1 ? 2 * (i >> 1) : 1 + 2 * (i & 1);
}
// branch-metric vector of step s (0..5) of a 6-step chunk held in w[] (vq_bm_* above)
template <int CODE_RATE, int s> __device__ __forceinline__ uint32_t vr_bm(const uint32_t (&w)[3]) {
    if constexpr (CODE_RATE == CR_12) return (s & 1) ? vq_bm_ab<2>(w[s >> 1]) : vq_bm_ab<0>(w[s >> 1]);
    else if constexpr (CODE_RATE == CR_34) return s % 3 == 0 ? vq_bm_ab<0>(w[s / 3]) : s % 3 == 1 ? vq_bm_a<2>(w[s / 3]) : vq_bm_b<3>(w[s / 3]);
    else return (s & 1) ? vq_bm_a<2>(w[s >> 1]) : vq_bm_ab<0>(w[s >> 1]);
}

// best state at time t (phase tm): smallest (byte = m7 << 1 | newest mark, state index) over the 64 slots of a code block (viterbicore.h:468-520);
// returns the slot address of that state.  Out of line for the same reason as vr_traceback.
template <int LB>
__device__ __forceinline__ uint32_t vr_best_core(const uint32_t (&R)[8 << (2 - LB)], const uint32_t q, const uint32_t tm, const uint32_t tn, const unsigned QM) {
    uint32_t best = 0xFFFFFFFFu;
#pragma unroll
    for (int r = 0; r < (8 << (2 - LB)); r++) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const uint32_t v = h ? (R[r] >> 16) : (R[r] & 0xFFFFu);
            const uint32_t A = (q << (6 - LB)) | (uint32_t)vr_low4(r, h);
            const uint32_t ns = ((A << tm) | (A >> (6u - tm))) & 63u;         // state index of this slot at time t
            best = min(best, ((((v >> 9) << 1) | ((v >> tn) & 1u)) << 8) | ns);
        }
    }
    if (LB >= 1) best = min(best, __shfl_xor_sync(QM, best, 1));
    if (LB == 2) best = min(best, __shfl_xor_sync(QM, best, 2));
    const uint32_t n = best & 63u;
    return ((n >> tm) | (n << (6u - tm))) & 63u;
}
// the same for the four-lane kernel, whose selectors index the word through vr_bmbyte
template <int CODE_RATE, int s> __device__ __forceinline__ uint32_t vr_bm_pk(const uint32_t (&w)[3]) {
    if constexpr (CODE_RATE == CR_34 && s % 3 != 0) return vq_bm_a2b3(w[s / 3]);
    else return vr_bm<CODE_RATE, s>(w);
}
// sum of the two complementary branch metrics of step s: 28 with both coded bits, 14 with one
template <int CODE_RATE, int s> __host__ __device__ constexpr uint32_t vr_ksum() {
    return CODE_RATE == CR_12 ? 28u : CODE_RATE == CR_34 ? (s % 3 == 0 ? 28u : 14u) : ((s & 1) ? 14u : 28u);
}

} // namespace sb
