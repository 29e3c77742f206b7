// sora_b200 — batched K=7 (133,171) soft Viterbi, v2 "quad" mapping for sm_90a.
//
// Arithmetic contract: bit-exact with kernel/bb/Brick11/src/viterbicore.h:269-556 driven like
// kernel/bb/Brick11/src/viterbi.hpp:104-237), different machine mapping:
//
//   * 4 lanes decode one code block; each lane keeps 16 of the 64 path metrics in 8 registers, two per register as
//     16-bit halves, so compare-select is the native 16x2 SIMD of sm_90 (VIMNMX.U16x2).
//   * Metrics sit in the HIGH byte of each half: the reference's uint8 wrap is the natural carry-out of the half (a plain
//     32-bit IMAD.IADD on the FMA pipe is a 16x2 add; the carry of the low half only lands in a dead byte), and the
//     survivor mark costs one LOP3 per *input* register (even role: & 0xFE00FE00, odd role: (& 0xFF00FF00) | 0x01000100).
//     The dead bytes are cleared by those masks every step and cannot decide a compare: the candidates' marks differ.
//   * The trellis is processed IN PLACE: butterfly (p, p+32) -> (2p, 2p+1) writes its results into the slots it read.
//     A slot's physical address is A = lane[2] | four bits made of half[1] and reg[3] (their order depends on the style, see
//     vq_low4); its state index at time t is rol6(A, t mod 6), so the pairing dimension walks through the address bits with
//     period 6: two steps pair with a partner lane (one SHFL.BFLY per register: the path-metric exchange), one step pairs the
//     two halves of each register, three steps pair two registers of the same lane (pure SIMD, no data movement).
//   * Branch metrics: the 4 possible values of a step are bytes of one register (two IDP4A + two IMAD straight from the
//     packed soft bytes); each 2-state operand is one PRMT with a compile-time selector.
//   * Survivor bits: the LSB of every new metric, 16 per lane per step -> one 16-bit word in a [column][block] shared
//     memory ring; bit index == physical address, so the traceback never leaves address space: the predecessor of slot A
//     at column c is A with bit (6 - c%6)%6 replaced by the survivor bit.
//   * One lane of the quad runs the windowed traceback (six columns per iteration with compile-time bit positions: after six
//     columns the address register is the six decoded bits), the x^7+x^4+1 descrambler and the CRC-32 / verdict.
//   * Two renderings of the mark handling (vq_step_a / vq_step_b below), chosen per code rate by measurement.
#pragma once
#include "rx11a_kernels.cuh"

namespace sb {


#define SB_VQ_WARPS 1                      // warps per CTA
#define SB_VQ_FR (8 * SB_VQ_WARPS)         // code blocks per CTA
#define SB_VQ_RING_MAX 294                     // columns kept per code block: depth + lookahead + 7 (287 for 256/24) + up to 5 written before a
                                           // recorded traceback is served; multiple of 6

// static class of (reg r, half h) at phase T, lane part excluded (GF(2)-linear, so the lane part is XORed in later)
// low four address bits of (register r, half h): reg bit 0 | half | reg bit 2 | reg bit 1 — the order in which the PRMT gather of the
// survivor marks (vq_commit_marks) lays the 16 decisions of a lane down, so that ring bit index == address
// (style B); style A keeps half | reg.
template <int S> __host__ __device__ constexpr int vq_low4(int r, int h) { return S ? ((r & 1) << 3) | (h << 2) | (r >> 1) : (h << 3) | r; }
template <int S> __host__ __device__ constexpr int vq_scls(int T, int r, int h) { return vq_cls(vq_rol6(vq_low4<S>(r, h), T) & 31); }
__host__ __device__ constexpr int vq_lcls(int T, int q) { return vq_cls(vq_rol6(q << 4, T) & 31); }

struct VqLane {
    unsigned swz[6];       // per-phase byte swizzle applying this lane's class contribution
    unsigned lm[2], lo[2]; // lane-phase role mask of this lane's own registers (even: & EV, odd: (& FF) | ONE)
};

// one trellis step at compile-time phase T.  Cbase byte (cA<<1|cB) = metric of the even candidate for a predecessor of
// that class; the complement class (3 - index) is the odd candidate's.
// Two renderings of the same arithmetic; which one is faster depends on how often the per-group bookkeeping runs, i.e. on the
// code rate: style A keeps the ALU pipe lighter (R = 1/2), style B issues fewer instructions (R = 2/3, 3/4).
//   style A: the survivor marks are taken out of the fresh metrics once per step (LOP3 + IMAD-side subtract / shifted accumulate), the
//            even / odd roles of the next step are plain adds; address = lane | half | reg.
//   style B: the role masks of the next step replace the stale marks (one LOP3 per input register), the 16 marks of a lane are gathered
//            with four PRMTs; address = lane | reg bit 0 | half | reg bits 2,1 so that the gathered word is already in address order.
template <int T>
__device__ __forceinline__ void vq_step_a(uint32_t (&R)[8], uint32_t Cbase, const VqLane& L, unsigned qmask) {
    // R comes in with the survivor marks already removed (vq_commit); the odd role is then a plain add of the mark.
    const uint32_t Cb = __byte_perm(Cbase, 0, L.swz[T]);
    const uint32_t ONE = 0x01000100u;
    if (T <= 1) {                                       // pair = partner lane (xor 2 at T=0, xor 1 at T=1)
#pragma unroll
        for (int r = 0; r < 8; r++) {
            const int c0 = vq_scls<0>(T, r, 0), c1 = vq_scls<0>(T, r, 1);
            uint32_t av = __byte_perm(Cb, 0, vq_sel(c0, c1)), bv = __byte_perm(Cb, 0, vq_sel(3 - c0, 3 - c1));
            uint32_t own = R[r] + L.lo[T];              // marked according to this lane's role; the partner did the same
            uint32_t Z = __shfl_xor_sync(qmask, own, T == 0 ? 2 : 1);
            R[r] = __vminu2(own + av, Z + bv);
        }
    } else if (T == 2) {                                // pair = the two halves of each register
#pragma unroll
        for (int r = 0; r < 8; r++) {
            const int c = vq_scls<0>(2, r, 0);             // class of p (low half); the high half is p+32: complement
            uint32_t ab = __byte_perm(Cb, 0, vq_sel(c, 3 - c)), ba = __byte_perm(Cb, 0, vq_sel(3 - c, c));
            uint32_t m = R[r] + 0x01000000u;            // low half = even role, high half = odd role
            uint32_t t1 = m + ab, t2 = m + ba;          // t1 = [p+a, p32+b], t2 = [p+b, p32+a]
            R[r] = __vminu2(__byte_perm(t1, t2, 0x5410), __byte_perm(t1, t2, 0x7632));   // [t1.lo, t2.lo] vs [t1.hi, t2.hi]
        }
    } else {                                            // pair = register r ^ d inside the lane
        const int d = T == 3 ? 4 : T == 4 ? 2 : 1;
#pragma unroll
        for (int r = 0; r < 8; r++) {
            if (r & d) continue;
            const int c0 = vq_scls<0>(T, r, 0), c1 = vq_scls<0>(T, r, 1);
            uint32_t av = __byte_perm(Cb, 0, vq_sel(c0, c1)), bv = __byte_perm(Cb, 0, vq_sel(3 - c0, 3 - c1));
            uint32_t X = R[r], Y = R[r + d] + ONE;
            R[r]     = __vminu2(X + av, Y + bv);
            R[r + d] = __vminu2(X + bv, Y + av);
        }
    }
}
// Take the survivor marks (bit 8 of each half) out of the fresh metrics and return them as the 16 decision bits of this
// lane: bit 8h + r.  One LOP3 per register; the subtraction and the gather (m << r accumulated) are IMADs on the FMA pipe.
// The bytes below the metrics ("dead" bytes) collect the wrap carries of the low halves; they never decide a compare
// (the candidates' marks differ) and are wiped at every normalisation, long before they could overflow.
__device__ __forceinline__ uint32_t vq_commit_marks_a(uint32_t (&R)[8]) {
    uint32_t acc = 0;
#pragma unroll
    for (int r = 0; r < 8; r++) { const uint32_t m = R[r] & 0x01000100u; R[r] -= m; acc = m * (1u << r) + acc; }
    return __byte_perm(acc, 0, 0x4431);                 // [byte 1, byte 3, 0, 0]
}
template <int T>
__device__ __forceinline__ void vq_step_b(uint32_t (&R)[8], uint32_t Cbase, const VqLane& L, unsigned qmask) {
    // Metrics carry the survivor mark of the previous step in bit 8 of each half; the role masks below replace it (and wipe the
    // byte under the metric, where the uint8 wrap carries land) in the same LOP3.
    const uint32_t Cb = __byte_perm(Cbase, 0, L.swz[T]);
    const uint32_t EV = 0xFE00FE00u, FF = 0xFF00FF00u, ONE = 0x01000100u;
    if (T <= 1) {                                       // pair = partner lane (xor 2 at T=0, xor 1 at T=1)
#pragma unroll
        for (int r = 0; r < 8; r++) {
            const int c0 = vq_scls<1>(T, r, 0), c1 = vq_scls<1>(T, r, 1);
            uint32_t av = __byte_perm(Cb, 0, vq_sel(c0, c1)), bv = __byte_perm(Cb, 0, vq_sel(3 - c0, 3 - c1));
            uint32_t own = (R[r] & L.lm[T]) | L.lo[T];  // marked according to this lane's role; the partner did the same
            uint32_t Z = __shfl_xor_sync(qmask, own, T == 0 ? 2 : 1);
            R[r] = __vminu2(own + av, Z + bv);
        }
    } else if (T == 3) {                                // pair = the two halves of each register (address bit 2)
#pragma unroll
        for (int r = 0; r < 8; r++) {
            const int c = vq_scls<1>(3, r, 0);             // class of p (low half); the high half is p+32: complement
            uint32_t aa = __byte_perm(Cb, 0, vq_sel(c, c)), bb = __byte_perm(Cb, 0, vq_sel(3 - c, 3 - c));
            uint32_t m = (R[r] & 0xFF00FE00u) | 0x01000000u;              // [p even role, p32 odd role]
            uint32_t y = __byte_perm(m, 0, 0x1032);     // [p32, p]
            R[r] = __vminu2(m + aa, y + bb);            // [min(p+a, p32+b), min(p32+a, p+b)] = new states 2p, 2p+1
        }
    } else {                                            // pair = register r ^ d inside the lane (address bits 3, 1, 0)
        const int d = T == 2 ? 1 : T == 4 ? 4 : 2;
#pragma unroll
        for (int r = 0; r < 8; r++) {
            if (r & d) continue;
            const int c0 = vq_scls<1>(T, r, 0), c1 = vq_scls<1>(T, r, 1);
            uint32_t av = __byte_perm(Cb, 0, vq_sel(c0, c1)), bv = __byte_perm(Cb, 0, vq_sel(3 - c0, 3 - c1));
            uint32_t X = R[r] & EV, Y = (R[r + d] & FF) | ONE;
            R[r]     = __vminu2(X + av, Y + bv);
            R[r + d] = __vminu2(X + bv, Y + av);
        }
    }
}
// The 16 survivor marks of this lane (bit 8 of each half of the fresh metrics) as one word, bit index = vq_low4(r, h).
// Four PRMTs line the eight metric bytes of two registers up ([R.b1, R.b3, R'.b1, R'.b3]); bit 0 of every byte is a mark, pair p
// goes to bit p of its byte by three shift + bit-select steps, and the four nibbles are squeezed into 16 bits.
__device__ __forceinline__ uint32_t vq_commit_marks_b(const uint32_t (&R)[8]) {
    const uint32_t p0 = __byte_perm(R[0], R[1], 0x7531), p1 = __byte_perm(R[2], R[3], 0x7531);
    const uint32_t p2 = __byte_perm(R[4], R[5], 0x7531), p3 = __byte_perm(R[6], R[7], 0x7531);
    uint32_t t = (p0 & 0x01010101u) | ((p1 << 1) & ~0x01010101u);
    t = (t & 0x03030303u) | ((p2 << 2) & ~0x03030303u);
    t = (t & 0x07070707u) | ((p3 << 3) & ~0x07070707u);
    t &= 0x0F0F0F0Fu;
    t |= t >> 4;                                        // bytes 0 and 2 now hold two nibbles each
    return __byte_perm(t, 0, 0x4420);                   // [byte 0, byte 2, 0, 0]
}
template <int T, int S>
__device__ __forceinline__ void vq_step(uint32_t (&R)[8], uint32_t Cbase, const VqLane& L, unsigned qmask) {
    if (S) vq_step_b<T>(R, Cbase, L, qmask); else vq_step_a<T>(R, Cbase, L, qmask);
}

template <int CODE_RATE>
__global__ void __launch_bounds__(32 * SB_VQ_WARPS) k_viterbi_quad(const uint8_t* __restrict__ soft, uint64_t soft_stride,
        uint32_t nframes, const FrameInfo* __restrict__ info, VitJob job, DevTables T,
        uint8_t* __restrict__ out, uint64_t out_stride, uint32_t* __restrict__ status_out, uint32_t* __restrict__ crc_out) {
    constexpr uint32_t SB_VQ_RING = CODE_RATE == CR_12 ? 294u : 288u;   // 6 columns of slack only where tracebacks are deferred (see DEFER)
    __shared__ unsigned long long s_ring[SB_VQ_RING][SB_VQ_FR];    // column c lives in slot (c - 1) mod SB_VQ_RING
    __shared__ uint32_t s_crc[256];                    // CRC-32 (reflected 0xEDB88320, core/inc/CRC32.h:76)
    __shared__ uint8_t s_scr[128];
    __shared__ uint8_t s_win[SB_VQ_FR][48];
    const int lane = threadIdx.x & 31, q = lane & 3;
    const unsigned QM = 0xFu << (lane & 28);           // the 4 lanes of this code block: quads run as independent sub-warps
    const int fb = (threadIdx.x >> 2);                 // code block within the CTA
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_crc[i] = __ldg(T.crc32 + i);
    for (int i = threadIdx.x; i < 128; i += blockDim.x) s_scr[i] = __ldg(T.scramble + i);
    __syncthreads();
    const uint32_t f = blockIdx.x * SB_VQ_FR + fb;
    // per-frame parameters; frames of other rates (or finished/invalid) are skipped by this instantiation
    uint32_t L = job.frame_len, nsoft = job.nsoft; bool active = f < nframes;
    if (active && info) {
        FrameInfo fi = info[f];
        active = fi.status == E_SUCCESS && fi.code_rate == (uint32_t)CODE_RATE;
        L = fi.length; nsoft = fi.soft_bytes;
    } else if (active) active = job.code_rate == (uint32_t)CODE_RATE;
    if (!active) return;                                // whole quad leaves together (no block-wide sync below)
    constexpr int S = CODE_RATE == CR_12 ? 0 : 1;       // arithmetic style (see vq_step)
    constexpr uint32_t GROUP = CODE_RATE == CR_12 ? 2u : CODE_RATE == CR_34 ? 4u : 3u;   // soft bytes per puncture group
    constexpr uint32_t GSTEPS = CODE_RATE == CR_12 ? 1u : CODE_RATE == CR_34 ? 3u : 2u;  // trellis steps per group
    const uint32_t depth = job.depth, look = job.lookahead;
    const uint8_t* sp = soft + (size_t)f * soft_stride;
    uint8_t* op = out + (size_t)f * out_stride;
    const uint32_t out_cap = (uint32_t)(out_stride < 0xFFFFFFFFull ? out_stride : 0xFFFFFFFFull);
    VqLane LC;
#pragma unroll
    for (int t = 0; t < 6; t++) {
        int lc = q == 0 ? vq_lcls(t, 0) : q == 1 ? vq_lcls(t, 1) : q == 2 ? vq_lcls(t, 2) : vq_lcls(t, 3);
        LC.swz[t] = (unsigned)((0 ^ lc) | ((1 ^ lc) << 4) | ((2 ^ lc) << 8) | ((3 ^ lc) << 12));
    }
    {
        const uint32_t EV = 0xFE00FE00u, FF = 0xFF00FF00u, ONE = 0x01000100u;
        int b0 = (q >> 1) & 1, b1 = q & 1;              // pair bit at T=0 is address bit 5 (lane bit 1), at T=1 address bit 4
        LC.lm[0] = b0 ? FF : EV; LC.lo[0] = b0 ? ONE : 0u;
        LC.lm[1] = b1 ? FF : EV; LC.lo[1] = b1 ? ONE : 0u;
    }
    // initial metrics (viterbilut.h:22-32): state 0 -> 0x00, others 0x30; at t=0 state == address
    uint32_t R[8];
#pragma unroll
    for (int r = 0; r < 8; r++) R[r] = 0x30003000u;
    if (q == 0) R[0] = 0x30000000u;
    const uint32_t end = L * 8u + 16u + 6u;
    uint32_t tb = 0, ob = 0;                            // tb = trellis time at the start of the current 6-step chunk
    uint32_t wcol = 0;                                  // ring slot of column tb + 1 (multiple of 6)
    uint32_t next_tb = min(end, depth + look + 6u);     // first time a traceback can fire (viterbi.hpp:182-203)
    uint32_t desc_count = 0, desc_reg = 0, byte_count = 0, crc = 0xFFFFFFFFu, fcs = 0, verdict = E_SUCCESS, nraw = 0;
    uint32_t lastdec = 0;                               // style A: this lane's 16 survivor marks of the newest column
    bool done = false;
    uint16_t* ring16 = (uint16_t*)&s_ring[0][0] + fb * 4 + q;      // + slot * (4 * SB_VQ_FR)
    uint32_t pos_soft = 0;

    // normalisation + traceback triggers, evaluated after every puncture group at time t (column t sits in ring slot cslot);
    // tm = t % 6 is a compile-time constant in the main loop
    // With DEFER, traceback requests are only recorded when they fire (best state, column, window) and carried out once per 6-step chunk: the
    // pointer chase + descrambler + CRC code then exists once instead of once per group position, which keeps the loop inside the
    // instruction cache.  The ring has 6 columns of slack for the steps that run before the request is served.
    constexpr bool DEFER = CODE_RATE == CR_12;          // measured: pays at R = 1/2 (a group after every step), not at 2/3 and 3/4
    uint32_t pA[2], pcol[2], pcm[2], pla[2], pnout[2], npend = 0;
    // windowed traceback from slot A0 of the column in ring slot col0 (column phase cm0), then descrambler / CRC-32 / verdict
    auto do_traceback = [&](const uint32_t A0, const uint32_t col0, const uint32_t cm0, const uint32_t la, const uint32_t nout) {
        __syncwarp(QM);
            if (q == 0) {
                // traceback in address space: survivor bit d of slot A at column c = bit A of that column's word;
                // the predecessor slot is A with bit (6 - c%6)%6 replaced by d; d is also the decoded bit of column c.
                uint32_t A = A0, col = col0, cm = cm0, todo = la + nout;
                uint32_t fifo = 0; int cnt = -(int)la;                      // the first `la` bits are only looked through; at most 13 bits wait
                uint8_t* win = s_win[fb]; uint32_t wpos = nout >> 3;        // bytes come out last-first; the sink needs them first-first
                auto emit = [&]() { while (cnt >= 8) { win[--wpos] = (uint8_t)(fifo >> (cnt - 8)); cnt -= 8; } };
                while (cm != 0 && todo) {               // up to 5 columns until the column phase is 0
                    const unsigned long long w = s_ring[col][fb];
                    const uint32_t d = (uint32_t)(w >> A) & 1u, j = 6u - cm;
                    A = (A & ~(1u << j)) | (d << j);
                    col = col ? col - 1 : SB_VQ_RING - 1; cm--; todo--;
                    fifo = (fifo << 1) | d; cnt++;
                }
                emit();
                while (todo >= 6) {                     // six columns with phases 0,5,4,3,2,1: bit k of A is replaced at the k-th of them,
                    const unsigned long long* wp = &s_ring[col][fb];       // and slots col..col-5 never wrap (col % 6 == 5)
#pragma unroll
                    for (int k = 0; k < 6; k++) {
                        const unsigned long long w = wp[-k * SB_VQ_FR];
                        const uint32_t d = (uint32_t)(w >> A) & 1u;
                        A = (A & ~(1u << k)) | (d << k);
                    }
                    col = col >= 6 ? col - 6 : col + SB_VQ_RING - 6; todo -= 6;
                    fifo = (fifo << 6) | (__brev(A) >> 26); cnt += 6;       // decoded bits, newest column first
                    emit();
                }
                while (todo) {                          // cm == 0 on entry
                    const unsigned long long w = s_ring[col][fb];
                    const uint32_t d = (uint32_t)(w >> A) & 1u, j = cm ? 6u - cm : 0u;
                    A = (A & ~(1u << j)) | (d << j);
                    col = col ? col - 1 : SB_VQ_RING - 1; cm = cm ? cm - 1 : 5; todo--;
                    fifo = (fifo << 1) | d; cnt++;
                }
                emit();
                const uint32_t nbytes = nout >> 3;      // <= 35 (final flush)
                if (job.raw) {
                    for (uint32_t b = 0; b < nbytes; b++) op[(size_t)nraw + b] = win[b];
                } else {
                    for (uint32_t b = 0; b < nbytes; b++) {       // scramble.hpp:323-351, PHY_11a.hpp:655-700
                        uint32_t by = win[b];
                        desc_count++;
                        if (desc_count == 1) continue;
                        if (desc_count == 2) { desc_reg = by >> 1; continue; }
                        desc_reg = s_scr[desc_reg];
                        uint32_t o = by ^ desc_reg; desc_reg >>= 1;
                        if (byte_count < (uint32_t)((int)L - 4)) {
                            if (byte_count < out_cap) op[byte_count] = (uint8_t)o;
                            byte_count++;
                            crc = (crc >> 8) ^ s_crc[(crc ^ o) & 0xFFu];
                        } else if (byte_count < L) {
                            if (byte_count < out_cap) op[byte_count] = (uint8_t)o;
                            byte_count++;
                            fcs |= o << (8u * (byte_count - 1u - (L - 4u)));
                            if (byte_count == L) verdict = (~crc == fcs) ? (uint32_t)E_FRAME_OK : (uint32_t)E_CRC32_FAIL;
                        }
                    }
                }
                nraw += nbytes;
            }
        __syncwarp(QM);
    };
    auto after_group = [&](const uint32_t t, const uint32_t tm, const uint32_t cslot) {
        if ((t & 7u) == 0) {                            // viterbi.hpp:177-180 -> viterbicore.h:445-465
            uint32_t m = __vminu2(__vminu2(__vminu2(R[0], R[1]), __vminu2(R[2], R[3])), __vminu2(__vminu2(R[4], R[5]), __vminu2(R[6], R[7])));
            m = min(m & 0xFFFFu, m >> 16) >> 8;         // smallest metric byte of this lane
            m = min(m, __shfl_xor_sync(QM, m, 1)); m = min(m, __shfl_xor_sync(QM, m, 2));
            const uint32_t mv = (m & 0xFEu) * 0x01000100u;
#pragma unroll
            for (int r = 0; r < 8; r++) R[r] = S ? R[r] - mv : (R[r] - mv) & 0xFF00FF00u;   // every metric byte >= m: no borrow; style A wipes its carry bytes here
        }
        if (t < next_tb) return;
        uint32_t nout, la;                              // viterbi.hpp:182-203
        if (t >= end) { nout = end - ob - 6u; la = t - end; }
        else { nout = depth; la = look + (t - (ob + depth + look + 6u)) % 8u; }
        if (nout) {                                     // uniform inside the quad
            // best state: smallest (metric incl. mark, state index) over the 64 slots (viterbicore.h:468-520).  Each half becomes the
            // 16-bit key (metric | mark) << 8 | state index (the part of the index that comes from reg / half is a constant at this
            // phase); a SIMD min tree, then the lane part of the index, then the quad.
            uint32_t n;
            if constexpr (DEFER) {
                uint32_t k2 = 0xFFFFFFFFu;
    #pragma unroll
                for (int r = 0; r < 8; r++) {
                    constexpr uint32_t dummy = 0; (void)dummy;
                    const uint32_t n0 = (uint32_t)(((vq_low4<S>(r, 0) << tm) | (vq_low4<S>(r, 0) >> (6u - tm))) & 63u);
                    const uint32_t n1 = (uint32_t)(((vq_low4<S>(r, 1) << tm) | (vq_low4<S>(r, 1) >> (6u - tm))) & 63u);
                    uint32_t key = (R[r] & 0xFF00FF00u) | (n1 << 16) | n0;
                    if (!S) key |= (((lastdec >> r) & 1u) << 8) | (((lastdec >> (8 + r)) & 1u) << 24);   // style A keeps the marks in the decision word
                    k2 = __vminu2(k2, key);
                }
                uint32_t best = min(k2 & 0xFFFFu, k2 >> 16);
                const uint32_t nl = (((uint32_t)q << 4 << tm) | ((uint32_t)q << 4 >> (6u - tm))) & 63u;
                best |= nl;
                best = min(best, __shfl_xor_sync(QM, best, 1)); best = min(best, __shfl_xor_sync(QM, best, 2));
                n = best & 63u;
            } else {
                uint32_t best = 0xFFFFFFFFu;            // (metric | mark) << 16 | state index << 8 | address
#pragma unroll
                for (int r = 0; r < 8; r++) {
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const uint32_t v = h ? (R[r] >> 24) : ((R[r] >> 8) & 0xFFu);      // metric byte, survivor mark included (style B)
                        const uint32_t A = ((uint32_t)q << 4) | (uint32_t)vq_low4<S>(r, h);
                        const uint32_t ns = ((A << tm) | (A >> (6u - tm))) & 63u;         // state index of this slot at time t
                        best = min(best, (v << 16) | (ns << 8) | A);
                    }
                }
                best = min(best, __shfl_xor_sync(QM, best, 1)); best = min(best, __shfl_xor_sync(QM, best, 2));
                n = (best >> 8) & 63u;
            }
            const uint32_t A0 = ((n >> tm) | (n << (6u - tm))) & 63u;
            if (DEFER) { if (npend < 2u) { pA[npend] = A0; pcol[npend] = cslot; pcm[npend] = tm; pla[npend] = la; pnout[npend] = nout; } npend++; }
            else do_traceback(A0, cslot, tm, la, nout);
            ob += nout;
        }
        if (ob + 6u >= end && t >= end) done = true;
        next_tb = min(end, ob + depth + look + 6u);
        if (next_tb <= t) next_tb = t + 1u;              // a frame shorter than the prefix: re-evaluate at every group
    };
    auto serve_tracebacks = [&]() {
        if constexpr (DEFER) {
            if (npend == 0) return;                     // uniform inside the quad
            for (uint32_t pi = 0; pi < npend && pi < 2u; pi++) do_traceback(pA[pi], pcol[pi], pcm[pi], pla[pi], pnout[pi]);
            npend = 0;
        }
    };
    // store the survivor bits of column tb + k + 1 (slot wcol + k)
    auto commit = [&](const uint32_t k) {
        if (S) lastdec = vq_commit_marks_b(R); else lastdec = vq_commit_marks_a(R);
        ring16[(wcol + k) * (4 * SB_VQ_FR)] = (uint16_t)lastdec;
    };

    // main loop: 6 trellis steps (one phase cycle) per iteration; the next chunk's soft values are prefetched
    constexpr uint32_t CHUNK_BYTES = 6u / GSTEPS * GROUP;        // 12 (R=1/2), 9 (2/3), 8 (3/4)
    uint32_t w0 = 0, w1 = 0, w2 = 0;                    // current chunk, little-endian bytes
    auto fetch = [&](uint32_t pos, uint32_t& a0, uint32_t& a1, uint32_t& a2) {
        if (pos + CHUNK_BYTES > nsoft) { a0 = a1 = a2 = 0; return; }
        if (CODE_RATE == CR_34) { uint2 v = __ldg((const uint2*)(sp + pos)); a0 = v.x; a1 = v.y; a2 = 0; }
        else if (CODE_RATE == CR_12) { a0 = __ldg((const uint32_t*)(sp + pos)); a1 = __ldg((const uint32_t*)(sp + pos + 4)); a2 = __ldg((const uint32_t*)(sp + pos + 8)); }
        else { uint32_t b[9];
#pragma unroll
               for (int i = 0; i < 9; i++) b[i] = __ldg(sp + pos + i);
               // keep every puncture group inside one word: w0 = b0 b1 b2 -, w1 = b3 b4 b5 -, w2 = b6 b7 b8 -
               a0 = b[0] | (b[1] << 8) | (b[2] << 16); a1 = b[3] | (b[4] << 8) | (b[5] << 16); a2 = b[6] | (b[7] << 8) | (b[8] << 16); }
    };
    fetch(0, w0, w1, w2);
    while (!done && pos_soft + CHUNK_BYTES <= nsoft) {
        uint32_t n0, n1, n2; fetch(pos_soft + CHUNK_BYTES, n0, n1, n2);
        pos_soft += CHUNK_BYTES;
        if (CODE_RATE == CR_12) {
            vq_step<0, S>(R, vq_bm_ab<0>(w0), LC, QM); commit(0); after_group(tb + 1, 1, wcol);
            vq_step<1, S>(R, vq_bm_ab<2>(w0), LC, QM); commit(1); after_group(tb + 2, 2, wcol + 1);
            vq_step<2, S>(R, vq_bm_ab<0>(w1), LC, QM); commit(2); after_group(tb + 3, 3, wcol + 2);
            vq_step<3, S>(R, vq_bm_ab<2>(w1), LC, QM); commit(3); after_group(tb + 4, 4, wcol + 3);
            vq_step<4, S>(R, vq_bm_ab<0>(w2), LC, QM); commit(4); after_group(tb + 5, 5, wcol + 4);
            vq_step<5, S>(R, vq_bm_ab<2>(w2), LC, QM); commit(5); after_group(tb + 6, 0, wcol + 5);
        } else if (CODE_RATE == CR_34) {
            vq_step<0, S>(R, vq_bm_ab<0>(w0), LC, QM); commit(0);
            vq_step<1, S>(R, vq_bm_a<2>(w0), LC, QM);  commit(1);
            vq_step<2, S>(R, vq_bm_b<3>(w0), LC, QM);  commit(2); after_group(tb + 3, 3, wcol + 2);
            vq_step<3, S>(R, vq_bm_ab<0>(w1), LC, QM); commit(3);
            vq_step<4, S>(R, vq_bm_a<2>(w1), LC, QM);  commit(4);
            vq_step<5, S>(R, vq_bm_b<3>(w1), LC, QM);  commit(5); after_group(tb + 6, 0, wcol + 5);
        } else {
            vq_step<0, S>(R, vq_bm_ab<0>(w0), LC, QM); commit(0);
            vq_step<1, S>(R, vq_bm_a<2>(w0), LC, QM);  commit(1); after_group(tb + 2, 2, wcol + 1);
            vq_step<2, S>(R, vq_bm_ab<0>(w1), LC, QM); commit(2);
            vq_step<3, S>(R, vq_bm_a<2>(w1), LC, QM);  commit(3); after_group(tb + 4, 4, wcol + 3);
            vq_step<4, S>(R, vq_bm_ab<0>(w2), LC, QM); commit(4);
            vq_step<5, S>(R, vq_bm_a<2>(w2), LC, QM);  commit(5); after_group(tb + 6, 0, wcol + 5);
        }
        serve_tracebacks();
        tb += 6; wcol += 6; if (wcol >= SB_VQ_RING) wcol -= SB_VQ_RING;
        w0 = n0; w1 = n1; w2 = n2;
    }
    // tail: whole puncture groups that do not fill a 6-step chunk (standalone API with arbitrary nsoft).
    // Rare and short, so phases are dispatched at run time.
    {
        uint32_t tm = 0, k = 0;                         // t % 6 (the main loop always leaves it at 0), steps into the chunk at tb
        auto step_rt = [&](uint32_t Cbase) {
            switch (tm) { case 0: vq_step<0, S>(R, Cbase, LC, QM); break; case 1: vq_step<1, S>(R, Cbase, LC, QM); break;
                          case 2: vq_step<2, S>(R, Cbase, LC, QM); break; case 3: vq_step<3, S>(R, Cbase, LC, QM); break;
                          case 4: vq_step<4, S>(R, Cbase, LC, QM); break; default: vq_step<5, S>(R, Cbase, LC, QM); }
            commit(k); k++;
            tm = tm == 5 ? 0 : tm + 1;
        };
        while (!done && pos_soft + GROUP <= nsoft) {
            uint32_t w = __ldg(sp + pos_soft) | ((uint32_t)__ldg(sp + pos_soft + 1) << 8);
            if (GROUP > 2) w |= (uint32_t)__ldg(sp + pos_soft + 2) << 16;
            if (GROUP > 3) w |= (uint32_t)__ldg(sp + pos_soft + 3) << 24;
            pos_soft += GROUP;
            step_rt(vq_bm_ab<0>(w));
            if (GSTEPS >= 2) step_rt(vq_bm_a<2>(w));
            if (GSTEPS >= 3) step_rt(vq_bm_b<3>(w));
            after_group(tb + k, tm, wcol + k - 1);
            serve_tracebacks();
            if (k == 6) { k = 0; tb += 6; wcol += 6; if (wcol >= SB_VQ_RING) wcol -= SB_VQ_RING; }
        }
    }
    if (q == 0) {
        if (!job.raw) { if (verdict == E_SUCCESS) verdict = E_FAILED; status_out[f] = verdict; crc_out[f] = fcs; }
        else { status_out[f] = nraw; crc_out[f] = 0; }
    }
}

} // namespace sb
