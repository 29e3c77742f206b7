// sora_b200 — 802.11b (DSSS / CCK) receive kernel for sm_90a.
//
// One thread decodes one capture slot (44 Msps COMPLEX16, 4 samples per chip) from a fresh context up to its first
// frame event, like MAC11b_Receive drives CreateDemodGraph (kernel/bb/demod11/fb11b_demod.cpp:26-79,
// fb11bdemod_config.hpp:123-180).  Every stage of the reference is a short sequential state machine per sample / chip /
// symbol (energy detect, early-late timing, Barker peak search, SFD hunt, differential demap, CCK arg-max, self-
// synchronising descrambler), so the data-parallel axis is the slot: 32 slots advance in lock-step per warp.
// Stages and their reference bricks:
//   TDCRemove / TDCEstimator            kernel/brick/inc/dc.hpp:8-43,101-166
//   TEnergyDetect                       kernel/bb/Brick11/src/cca.hpp:13-98
//   TSymTiming, TBarkerSync             kernel/bb/Brick11/src/symtiming.hpp:12-169,177-308
//   TBB11bDespread, TDBPSKDemap, TDQPSKDemap   kernel/bb/Brick11/src/barkerspread.hpp:229-451
//   TSFDSync                            kernel/bb/Brick11/src/sfd_sync.hpp:12-133
//   TCCK5P5Decoder, TCCK11Decoder       kernel/bb/Brick11/src/cck.hpp:11-780
//   TDesc741                            kernel/bb/Brick11/src/scramble.hpp:95-162
//   TBB11bPlcpParser, TBB11bFrameSink   kernel/bb/Brick11/src/PHY_11b.hpp:504-747
#pragma once
#include "rx11a_kernels.cuh"

namespace sb {

enum : uint32_t { E_SFD_FAIL = 0x80000004u, E_SFD_TIMEOUT = 0x80000008u, E_SYNC_TIMEOUT = 0x80000009u };

struct Result11b { uint32_t status, rate_kbps, length, crc32, sample_index, detect_vec; };

struct S16 { short re, im; };
__device__ __forceinline__ S16 s_sub(S16 a, S16 b) { S16 r; r.re = (short)(a.re - b.re); r.im = (short)(a.im - b.im); return r; }
__device__ __forceinline__ S16 s_add(S16 a, S16 b) { S16 r; r.re = (short)(a.re + b.re); r.im = (short)(a.im + b.im); return r; }
__device__ __forceinline__ S16 s_sra(S16 a, int n) { S16 r; r.re = (short)(a.re >> n); r.im = (short)(a.im >> n); return r; }
__device__ __forceinline__ S16 s_w(uint32_t w) { S16 r; r.re = (short)(w & 0xFFFF); r.im = (short)(w >> 16); return r; }
__device__ __forceinline__ S16 s_ld(const uint32_t* p) { uint32_t w = __ldg(p); S16 r; r.re = (short)(w & 0xFFFF); r.im = (short)(w >> 16); return r; }
__device__ __forceinline__ int imul(int a, int b) { return (int)((unsigned)a * (unsigned)b); }

struct CckPick { int mx; unsigned val; };
// arg-max over the four (phi3, phi4) hypotheses of one phi2 module (cck.hpp:283-372)
__device__ __forceinline__ CckPick cck11_module(int a1r, int a1i, int a2r, int a2i, int a3r, int a3i, int a4r, int a4i) {
    const int b00r = (a2r + a1r) >> 2, b00i = (a2i + a1i) >> 2, b10r = (a2r - a1r) >> 2, b10i = (a2i - a1i) >> 2;
    const int b01r = (a2r - a1i) >> 2, b01i = (a2i + a1r) >> 2, b11r = (a2r + a1i) >> 2, b11i = (a2i - a1r) >> 2;
    const int b20r = (a4r + a3r) >> 2, b20i = (a4i + a3i) >> 2, b30r = (a4r - a3r) >> 2, b30i = (a4i - a3i) >> 2;
    const int b21r = (a4r - a3i) >> 2, b21i = (a4i + a3r) >> 2, b31r = (a4r + a3i) >> 2, b31i = (a4i - a3r) >> 2;
    int Lr[4], Li[4];
    Lr[0] = imul(b00r, b20r) + imul(b00i, b20i); Li[0] = imul(b00r, b20i) - imul(b00i, b20r);
    Lr[1] = imul(b01r, b21r) + imul(b01i, b21i); Li[1] = imul(b01r, b21i) - imul(b01i, b21r);
    Lr[2] = imul(b10r, b30r) + imul(b10i, b30i); Li[2] = imul(b10r, b30i) - imul(b10i, b30r);
    Lr[3] = imul(b11r, b31r) + imul(b11i, b31i); Li[3] = imul(b11r, b31i) - imul(b11i, b31r);
    int mx[4]; unsigned vl[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const unsigned base = k == 0 ? 0x00u : k == 1 ? 0x30u : k == 2 ? 0x10u : 0x20u;
        const int ar = Lr[k] < 0 ? -Lr[k] : Lr[k], ai = Li[k] < 0 ? -Li[k] : Li[k];
        if (ar > ai) { if (Lr[k] > 0) { mx[k] = Lr[k]; vl[k] = base; } else { mx[k] = -Lr[k]; vl[k] = base | 0x40u; } }
        else         { if (Li[k] > 0) { mx[k] = Li[k]; vl[k] = base | 0xC0u; } else { mx[k] = -Li[k]; vl[k] = base | 0x80u; } }
    }
    CckPick p;
    if (mx[0] > mx[1]) { p.mx = mx[0]; p.val = vl[0]; } else { p.mx = mx[1]; p.val = vl[1]; }
    if (mx[2] > mx[3]) { if (mx[2] > p.mx) { p.mx = mx[2]; p.val = vl[2]; } }
    else               { if (mx[3] > p.mx) { p.mx = mx[3]; p.val = vl[3]; } }
    return p;
}
__device__ __forceinline__ unsigned dqpsk_bits(S16 ref, S16 s) {              // barkerspread.hpp:430-437; bit0 | bit1<<1
    const int re = ref.re * s.re + ref.im * s.im, im = ref.re * s.im - ref.im * s.re;
    return ((unsigned)(re + im) >> 31) | (((unsigned)(re - im) >> 31) << 1);
}

struct Rx11bState {
    // context
    uint32_t error_code; int cca_state, rate_state, plcp_state;
    S16 DC, last_symbol; unsigned byte_reg, frame_length, data_rate_kbps, frame_crc32, detect_vec, vec_count;
    // bricks
    uint32_t avg_energy, win0, win1, win2, win3, win4, win5, win6, win7, ed_count;   // TEnergyDetect's 8-vector window as a shift register (newest in win0)
    uint32_t dc_cnt; S16 dc_sum;
    int m_index, m_frag, st_n;
    int bs_state, bs_last_peak, bs_max, bs_search; S16 bs_partial[10];
    int q_n, cck_even;                            // chips of the running symbol: Barker despread accumulates (q_sr, q_si), CCK chips wait in shared memory
    int q_sr, q_si;
    unsigned sym_bits; int sym_n;                 // DBPSK / DQPSK bits of the running byte
    bool sfd_one; unsigned sfd_word; int sfd_err; unsigned sfd_cnt;
    unsigned hdr_lo, hdr_hi; int hdr_n;           // PLCP header bytes 0..3 / 4..5
    uint32_t byte_count, crc;
};

__global__ void __launch_bounds__(64) k_rx11b(const uint32_t* __restrict__ iq, const uint64_t* __restrict__ off, const uint32_t* __restrict__ len,
                                              uint32_t nframes, uint32_t cca_thr, uint8_t* __restrict__ out, uint64_t out_stride,
                                              Result11b* __restrict__ res, uint32_t max_frames, uint32_t* __restrict__ counts) {
    __shared__ uint32_t s_crc[16];
    __shared__ unsigned short s_crc16[16];
    __shared__ uint32_t s_q[64][17];                   // CCK chip queue of every thread (16 chips; 17 words per row: no bank conflicts between threads)
    if (threadIdx.x < 16) {
        uint32_t c = threadIdx.x; for (int k = 0; k < 4; k++) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1; s_crc[threadIdx.x] = c;
        uint32_t d = threadIdx.x; for (int k = 0; k < 4; k++) d = (d & 1) ? 0x8408u ^ (d >> 1) : d >> 1; s_crc16[threadIdx.x] = (unsigned short)d;
    }
    __syncthreads();
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nframes) return;
    const uint32_t* x = iq + off[f];                   // start of the part of the slot not consumed yet (continuous-capture mode moves it)
    const bool al16 = (((uintptr_t)x) & 15u) == 0;     // block starts are multiples of 4 samples from the slot start
    auto ld4 = [&](const uint32_t* p, uint32_t (&w)[4]) {
        if (al16) { const uint4 v = __ldg((const uint4*)p); w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w; }
        else { w[0] = __ldg(p); w[1] = __ldg(p + 1); w[2] = __ldg(p + 2); w[3] = __ldg(p + 3); }
    };
    const uint32_t slot_len = len[f]; uint32_t nblk = slot_len / 28u, consumed = 0, found = 0;
    uint8_t* op = out + (size_t)f * max_frames * out_stride;
    const uint32_t out_cap = (uint32_t)(out_stride < 0xFFFFFFFFull ? out_stride : 0xFFFFFFFFull);
    Rx11bState s;
    auto bricks_reset = [&]() {
        s.avg_energy = 0; s.win0 = s.win1 = s.win2 = s.win3 = s.win4 = s.win5 = s.win6 = s.win7 = 0; s.ed_count = 0;
        s.dc_cnt = 8; s.dc_sum.re = s.dc_sum.im = 0;
        s.m_index = 2; s.m_frag = 0; s.st_n = 0;
        s.bs_state = 0; s.bs_last_peak = -1; s.bs_max = 0; s.bs_search = 0; for (int i = 0; i < 10; i++) { s.bs_partial[i].re = 0; s.bs_partial[i].im = 0; }
        s.q_n = 0; s.q_sr = s.q_si = 0; s.sym_n = 0; s.sym_bits = 0; s.cck_even = 0;
        s.sfd_one = false; s.sfd_word = 0; s.sfd_err = 0; s.sfd_cnt = 0; s.hdr_n = 0; s.hdr_lo = s.hdr_hi = 0;
        s.byte_count = 0; s.crc = 0xFFFFFFFFu;
    };
    auto ctx_reset = [&]() { s.error_code = E_SUCCESS; s.cca_state = 0; s.rate_state = 0; s.plcp_state = 0; };
    s.DC.re = s.DC.im = 0; s.last_symbol.re = s.last_symbol.im = 0; s.byte_reg = 0; s.frame_length = 0; s.data_rate_kbps = 0; s.frame_crc32 = 0;
    s.detect_vec = 0; s.vec_count = 0;
    ctx_reset(); bricks_reset();

    // ---- byte path: TDesc741 -> PLCP parser | frame sink ----
    auto on_byte = [&](unsigned b) {
        unsigned xx = b, sr = s.byte_reg, o = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) { unsigned o1 = (xx ^ sr ^ (sr >> 3)) & 1u; sr = ((sr >> 1) | ((xx & 1u) << 6)) & 0xFFu; o = (o >> 1) | (o1 << 7); xx >>= 1; }
        s.byte_reg = b >> 1;
        if (s.plcp_state == 0) {
            if (s.hdr_n < 4) s.hdr_lo |= (o & 0xFFu) << (8 * s.hdr_n); else s.hdr_hi |= (o & 0xFFu) << (8 * (s.hdr_n - 4));
            s.hdr_n++;
            if (s.hdr_n < 6) return;
            s.hdr_n = 0;
            unsigned c = 0xFFFFu;
#pragma unroll
            for (int i = 0; i < 4; i++) { c ^= (s.hdr_lo >> (8 * i)) & 0xFFu; c = (c >> 4) ^ s_crc16[c & 15]; c = (c >> 4) ^ s_crc16[c & 15]; }
            c = (~c) & 0xFFFFu;
            const unsigned got = s.hdr_hi & 0xFFFFu;
            const unsigned hl = s.hdr_lo; s.hdr_lo = s.hdr_hi = 0;
            if (c != got) { s.error_code = E_PLCP_HEADER_FAIL; return; }
            const unsigned signal = hl & 0xFFu, service = (hl >> 8) & 0xFFu, l = hl >> 16;
            if (signal == 0x0A) { s.data_rate_kbps = 1000; s.frame_length = (l >> 3) & 0xFFFFu; s.rate_state = 1; }
            else if (signal == 0x14) { s.data_rate_kbps = 2000; s.frame_length = (l >> 2) & 0xFFFFu; s.rate_state = 2; }
            else if (signal == 0x37) { s.data_rate_kbps = 5500; s.frame_length = (((l * 11u) >> 4) - (service >> 7) - ((service >> 3) & 1u)) & 0xFFFFu; s.rate_state = 3; }
            else if (signal == 0x6E) { s.data_rate_kbps = 11000; s.frame_length = (((l * 11u) >> 3) - (service >> 7) - ((service >> 3) & 1u)) & 0xFFFFu; s.rate_state = 4; }
            else { s.data_rate_kbps = 0; s.frame_length = 0; }
            s.plcp_state = 1;
            return;
        }
        if (s.error_code != E_SUCCESS) return;
        const uint32_t L = s.frame_length;
        if (s.byte_count < (uint32_t)((int)L - 4)) {
            if (s.byte_count < out_cap) op[s.byte_count] = (uint8_t)o;
            s.byte_count++;
            s.crc ^= o; s.crc = (s.crc >> 4) ^ s_crc[s.crc & 15]; s.crc = (s.crc >> 4) ^ s_crc[s.crc & 15];
        } else if (s.byte_count < L) {
            if (s.byte_count < out_cap) op[s.byte_count] = (uint8_t)o;
            s.frame_crc32 = (s.frame_crc32 >> 8) | (o << 16);               // rolling window of the last three bytes
            s.byte_count++;
            if (s.byte_count == L - 1u) s.error_code = ((~s.crc & 0x00FFFFFFu) == (s.frame_crc32 & 0x00FFFFFFu)) ? (uint32_t)E_FRAME_OK : (uint32_t)E_CRC32_FAIL;
        }
    };
    // ---- chip path behind TBB11bRxRateSel ----
    auto on_chip = [&](S16 c) {
        if (s.error_code != E_SUCCESS && s.error_code != E_CS_TIMEOUT) return;
        if (s.rate_state <= 2) {
            {   // QuickBarkerDespread (barkerspread.hpp:276-304), one chip at a time: chips 1 and 4 are negated before the shift, chips 8..10 after it
                const int i = s.q_n; short re, im;
                if (i == 1 || i == 4) { re = (short)((short)(-c.re) >> 4); im = (short)((short)(-c.im) >> 4); }
                else if (i >= 8) { re = (short)(-(c.re >> 4)); im = (short)(-(c.im >> 4)); }
                else { re = (short)(c.re >> 4); im = (short)(c.im >> 4); }
                s.q_sr += re; s.q_si += im;
            }
            if (++s.q_n < 11) return;
            S16 sym; sym.re = (short)s.q_sr; sym.im = (short)s.q_si;
            s.q_n = 0; s.q_sr = s.q_si = 0;
            if (s.rate_state == 0) {                                        // TSFDSync
                const unsigned bit = (unsigned)(s.last_symbol.re * sym.re + s.last_symbol.im * sym.im) >> 31;
                s.last_symbol = sym;
                s.byte_reg &= 0x7fu;
                const unsigned sbit = (bit ^ s.byte_reg ^ (s.byte_reg >> 3)) & 1u;
                s.byte_reg = (s.byte_reg >> 1) | (bit << 6);
                s.sfd_word = ((s.sfd_word >> 1) | (sbit << 15)) & 0xFFFFu;
                s.sfd_cnt++;
                if (!s.sfd_one) { if (s.sfd_word == 0xFFFFu) s.sfd_one = true; }
                else {
                    if (s.sfd_word == 0xF3A0u) s.rate_state = 1;
                    else if (s.sfd_word != 0xFFFFu) { if (s.sfd_err++ > 32) { s.error_code = E_SFD_FAIL; return; } }
                }
                if (s.sfd_cnt > 144u) s.error_code = E_SFD_TIMEOUT;
                return;
            }
            if (s.rate_state == 1) {                                        // TDBPSKDemap: 8 symbols -> one byte, each against its predecessor
                s.sym_bits |= ((unsigned)(s.last_symbol.re * sym.re + s.last_symbol.im * sym.im) >> 31) << s.sym_n;
                s.last_symbol = sym;
                if (++s.sym_n == 8) { const unsigned r = s.sym_bits; s.sym_n = 0; s.sym_bits = 0; on_byte(r); }
            } else {                                                        // TDQPSKDemap: 4 symbols -> one byte
                s.sym_bits |= dqpsk_bits(s.last_symbol, sym) << (2 * s.sym_n);
                s.last_symbol = sym;
                if (++s.sym_n == 4) { const unsigned r = s.sym_bits; s.sym_n = 0; s.sym_bits = 0; on_byte(r); }
            }
            return;
        }
        uint32_t* qrow = s_q[threadIdx.x];
        qrow[s.q_n++] = ((uint32_t)(unsigned short)c.re) | ((uint32_t)(unsigned short)c.im << 16);
        if (s.rate_state == 4) {
            if (s.q_n < 8) return;
            s.q_n = 0;
            int R[8], I[8];
#pragma unroll
            for (int i = 0; i < 8; i++) { const S16 ch = s_w(qrow[i]); R[i] = ch.re; I[i] = ch.im; }
            const S16 q7 = s_w(qrow[7]);
            CckPick m1 = cck11_module(R[0] + R[1], I[0] + I[1], R[2] - R[3], I[2] - I[3], R[4] + R[5], I[4] + I[5], R[7] - R[6], I[7] - I[6]);
            CckPick m2 = cck11_module(I[0] + R[1], I[1] - R[0], I[2] - R[3], -(R[2] + I[3]), I[4] + R[5], I[5] - R[4], R[7] - I[6], R[6] + I[7]);
            m2.val |= 0x08u;
            unsigned o;
            if (m1.mx > m2.mx) {
                CckPick m4 = cck11_module(R[1] - I[0], R[0] + I[1], -(I[2] + R[3]), R[2] - I[3], R[5] - I[4], R[4] + I[5], I[6] + R[7], I[7] - R[6]);
                m4.val |= 0x0Cu; o = m1.mx > m4.mx ? m1.val : m4.val;
            } else {
                CckPick m3 = cck11_module(R[1] - R[0], I[1] - I[0], -(R[2] + R[3]), -(I[2] + I[3]), R[5] - R[4], I[5] - I[4], R[6] + R[7], I[6] + I[7]);
                m3.val |= 0x04u; o = m2.mx > m3.mx ? m2.val : m3.val;
            }
            o |= dqpsk_bits(s.last_symbol, q7);
            o ^= (unsigned)((s.cck_even << 1) | s.cck_even);
            s.cck_even ^= 1; s.last_symbol = q7;
            on_byte(o & 0xFFu);
            return;
        }
        if (s.q_n < 16) return;                                             // TCCK5P5Decoder: two half bytes per 16 chips
        s.q_n = 0;
        unsigned b = 0;
#pragma unroll
        for (int hb = 0; hb < 2; hb++) {
            int R[8], I[8];
#pragma unroll
            for (int i = 0; i < 8; i++) { const S16 ch = s_w(qrow[8 * hb + i]); R[i] = ch.re; I[i] = ch.im; }
            const S16 q7 = s_w(qrow[8 * hb + 7]);
            auto corr = [&](int a00r, int a00i, int a01r, int a01i, int a10r, int a10i, int a11r, int a11i) -> int {
                int b0r = a00r + a01r, b0i = -(a00i + a01i), b1r = a10r + a11r, b1i = a10i + a11i;
                b0r >>= 2; b0i >>= 2; b1r >>= 2; b1i >>= 2;
                return imul(b0r, b1r) - imul(b0i, b1i);
            };
            const int l1 = corr(I[0] + R[1], I[1] - R[0], I[2] - R[3], -(R[2] + I[3]), I[4] + R[5], I[5] - R[4], R[7] - I[6], R[6] + I[7]);
            const int l2 = corr(R[1] - I[0], R[0] + I[1], -(I[2] + R[3]), R[2] - I[3], R[5] - I[4], R[4] + I[5], I[6] + R[7], I[7] - R[6]);
            const unsigned b3 = hb ? 0x80u : 0x08u, b2 = hb ? 0x40u : 0x04u;
            int max1, max2; unsigned v1, v2;
            if (l1 > 0) { max1 = l1; v1 = 0; } else { max1 = -l1; v1 = b3; }
            if (l2 > 0) { max2 = l2; v2 = b2; } else { max2 = -l2; v2 = b2 | b3; }
            b |= max1 > max2 ? v1 : v2;
            b |= dqpsk_bits(s.last_symbol, q7) << (4 * hb);
            if (hb) b ^= 0x30u;
            s.last_symbol = q7;
        }
        on_byte(b & 0xFFu);
    };
    // ---- TBarkerSync ----
    auto barker_sync = [&](S16 in) {
        if (s.bs_state == 4) { on_chip(in); return; }
        s.bs_search++;
        if (s.bs_search >= 44) { s.error_code = E_SYNC_TIMEOUT; return; }
        const S16 ss = s_sra(in, 4);
        const S16 o = s_sub(s.bs_partial[0], ss);
        s.bs_partial[0] = s_sub(s.bs_partial[1], ss); s.bs_partial[1] = s_sub(s.bs_partial[2], ss); s.bs_partial[2] = s_add(s.bs_partial[3], ss);
        s.bs_partial[3] = s_add(s.bs_partial[4], ss); s.bs_partial[4] = s_add(s.bs_partial[5], ss); s.bs_partial[5] = s_sub(s.bs_partial[6], ss);
        s.bs_partial[6] = s_add(s.bs_partial[7], ss); s.bs_partial[7] = s_add(s.bs_partial[8], ss); s.bs_partial[8] = s_sub(s.bs_partial[9], ss);
        s.bs_partial[9] = ss;
        const int corr = o.re * o.re + o.im * o.im;
        if (s.bs_state == 0) {
            if (corr > s.bs_max) { s.bs_max = corr; s.bs_last_peak = 1; }
            else { s.bs_last_peak++; if (s.bs_last_peak == 11) s.bs_state = 1; }
        } else if (s.bs_state == 1) { s.bs_max = corr / 2; s.bs_last_peak = 1; s.bs_state = 2; }
        else if (s.bs_state == 2) {
            if (corr > s.bs_max) { s.bs_max = corr; s.bs_last_peak = 0; s.bs_state = 0; }
            else { s.bs_last_peak++; if (s.bs_last_peak == 11) s.bs_state = 3; }
        } else s.bs_state = 4;
    };

    // One pass of this loop = one event of the reference's driver (fb11b_demod.cpp:26-75).  max_frames == 1 is the slot-per-frame mode;
    // larger values walk a continuous capture: after FRAME_OK / CRC32_FAIL the source seeks past the last FCS byte, every event ends with
    // Flush(); ctx.reset(); Reset() and the DC estimate, the descrambler register and the differential reference carry over.
    for (;;) {
    Result11b r; r.status = E_NO_FRAME; r.rate_kbps = 0; r.length = 0; r.crc32 = 0; r.sample_index = 0; r.detect_vec = 0;
    uint32_t st_base = 0;                               // sample index (from x) of the first sample of the symbol-timing block being filled
    uint32_t blk = 0; bool event = false;
    for (; blk < nblk; blk++) {
        for (int v = 0; v < 7; v++) {
            const uint32_t p0 = blk * 28u + 4u * v;
            if (s.cca_state == 0) {
                if (s.error_code != E_CS_TIMEOUT) {     // TEnergyDetect stops consuming after the timeout (`ipin.clear(); return 0`)
                    S16 xv[4]; uint32_t pw = 0;
                    uint32_t w4[4]; ld4(x + p0, w4);
#pragma unroll
                    for (int k = 0; k < 4; k++) { xv[k] = s_sub(s_w(w4[k]), s.DC); pw += (uint32_t)((xv[k].re * xv[k].re + xv[k].im * xv[k].im) >> 5); }
                    s.avg_energy = s.avg_energy - s.win7 + pw;
                    s.win7 = s.win6; s.win6 = s.win5; s.win5 = s.win4; s.win4 = s.win3; s.win3 = s.win2; s.win2 = s.win1; s.win1 = s.win0; s.win0 = pw;
                    s.ed_count++;
                    if (s.ed_count >= 32) {
                        if (s.ed_count >= 100) s.error_code = E_CS_TIMEOUT;
                        else if (s.avg_energy >= cca_thr) { s.cca_state = 1; s.detect_vec = s.vec_count + 1; s.st_n = 0; st_base = p0 + 4u; }
                    }
                    if (s.cca_state != 1 && s.error_code != E_CS_TIMEOUT) {                       // TDCEstimator behind the energy gate
                        int hr = 0, hi = 0;
#pragma unroll
                        for (int k = 0; k < 4; k++) { hr += xv[k].re >> 5; hi += xv[k].im >> 5; }
                        s.dc_sum.re = (short)(s.dc_sum.re + (short)hr); s.dc_sum.im = (short)(s.dc_sum.im + (short)hi);
                        if (s.dc_cnt == 0) { s.DC.re = (short)(s.DC.re + (s.dc_sum.re >> 2)); s.DC.im = (short)(s.DC.im + (s.dc_sum.im >> 2)); s.dc_cnt = 8; s.dc_sum.re = s.dc_sum.im = 0; }
                        s.dc_cnt--;
                    }
                }
            } else {
                s.st_n += 4;
                if (s.st_n == 28) {                     // TSymTiming on the 28 samples x[st_base .. st_base+28) minus DC
                    uint32_t wv[7][4];                  // the whole 28-sample block: seven 128-bit loads when the slot is 16-byte aligned
#pragma unroll
                    for (int j = 0; j < 7; j++) ld4(x + st_base + 4u * j, wv[j]);
                    int idx = s.m_index;
                    if (idx < 0) {                      // symtiming.hpp: a negative phase re-reads the first sample of the block
                        const S16 o = s_sub(s_w(wv[0][0]), s.DC); s.m_index += 4; idx += 4;
                        if (s.error_code == E_SUCCESS) barker_sync(o);
                    }
                    {   // the picked samples are idx, idx+4, ...: always the same component of consecutive vectors
                        const int c = idx & 3, j0 = idx >> 2;
                        uint32_t pk[7];
#pragma unroll
                        for (int j = 0; j < 7; j++) pk[j] = c == 0 ? wv[j][0] : c == 1 ? wv[j][1] : c == 2 ? wv[j][2] : wv[j][3];
#pragma unroll 1
                        for (int j = j0; j < 7; j++) {
                            const uint32_t w = j == 0 ? pk[0] : j == 1 ? pk[1] : j == 2 ? pk[2] : j == 3 ? pk[3] : j == 4 ? pk[4] : j == 5 ? pk[5] : pk[6];   // register select, no local array
                            const S16 o = s_sub(s_w(w), s.DC); if (s.error_code == E_SUCCESS) barker_sync(o);
                        }
                    }
                    if (s.m_index >= 4) s.m_index = 0;
                    int sum[4] = {0, 0, 0, 0};
#pragma unroll
                    for (int i = 0; i < 28; i++) { S16 vv = s_sra(s_sub(s_w(wv[i >> 2][i & 3]), s.DC), 3); sum[i & 3] += vv.re * vv.re + vv.im * vv.im; }
                    const int mi = s.m_index, early = mi == 0 ? 3 : mi - 1, late = mi == 3 ? 0 : mi + 1;
                    auto pick4 = [&](int i) { return i == 0 ? sum[0] : i == 1 ? sum[1] : i == 2 ? sum[2] : sum[3]; };
                    const int se = pick4(early), sl = pick4(late), sm = pick4(mi);
                    if (se < sl) { if (sm < se) { s.m_index++; s.m_frag = 0; } else if (sm < sl) s.m_frag++; }
                    else { if (sm < sl) { s.m_index--; s.m_frag = 0; } else if (sm < se) s.m_frag--; }
                    if (s.m_frag >= 4) { s.m_index++; s.m_frag = -3; } else if (s.m_frag <= -4) { s.m_index--; s.m_frag = 3; }
                    s.st_n = 0; st_base += 28u;
                }
            }
            s.vec_count++;
        }
        const uint32_t err = s.error_code;              // the driver polls once per source block (fb11b_demod.cpp:29-31)
        if (err == E_SUCCESS) continue;
        if (err != E_CS_TIMEOUT) {
            r.status = err; r.rate_kbps = s.data_rate_kbps; r.length = s.frame_length; r.crc32 = s.frame_crc32 & 0x00FFFFFFu;
            r.sample_index = consumed + (blk + 1u) * 28u; r.detect_vec = s.detect_vec;
            event = true; break;
        }
        ctx_reset(); bricks_reset();
    }
    if (!event) { if (max_frames == 1u) res[f] = r; break; }
    res[(size_t)f * max_frames + found] = r; found++;
    if (found == max_frames) break;
    uint32_t adv = (blk + 1u) * 28u;
    if (r.status == E_FRAME_OK || r.status == E_CRC32_FAIL)      // "jump advance of the last CRC byte" (fb11b_demod.cpp:43-61)
        adv += s.data_rate_kbps == 1000 ? 352u : s.data_rate_kbps == 2000 ? 176u : s.data_rate_kbps == 5500 ? 64u : 32u;
    consumed += adv;
    if (consumed + 28u > slot_len) break;
    x += adv; nblk = (slot_len - consumed) / 28u; op += out_stride;
    ctx_reset(); bricks_reset();
    }
    if (counts) counts[f] = found;
}

} // namespace sb
