// sora_b200 — the transmitters: 802.11a, 802.11b, 802.11n and the legacy 802.11a / 802.11b ones, and the legacy 802.11b transmit filter.
#include "handle.cuh"
#include "tx11a_kernels.cuh"
#include "tx11b_kernels.cuh"
#include "tx11b_legacy_kernels.cuh"
#include "tx11a_legacy_kernels.cuh"
#include "tx11n_kernels.cuh"

// ---- 802.11a transmit (SURVEY.md §8(f) rank 2) -------------------------------------------------------------------------------
static int upload_tables_tx(sb200_handle* h) {
    if (h->tabtx.p) return SB200_OK;
    uint32_t tw128[3][32], tw32[3][8]; uint8_t seq[127], phase[128];
    for (int m = 1; m <= 3; m++) {
        for (int j = 0; j < 32; j++) tw128[m - 1][j] = pack(mk((int)trunc(32767.0 * cos(2 * M_PI * j * m / 128)), (int)trunc(-32767.0 * sin(2 * M_PI * j * m / 128))));
        for (int j = 0; j < 8; j++) tw32[m - 1][j] = pack(mk((int)trunc(32767.0 * cos(2 * M_PI * j * m / 32)), (int)trunc(-32767.0 * sin(2 * M_PI * j * m / 32))));
    }
    {   // scrambler x^7 + x^4 + 1 as a 127-periodic sequence: c[t] = c[t-7] ^ c[t-4] from the all-ones state; phase[s] = t such that
        // the seven outputs before t equal state s (bit 0 = oldest), which is how T11aSc's byte register reads (scramble.hpp:186-203)
        int hist[7] = {1, 1, 1, 1, 1, 1, 1}; uint8_t c[127 + 7];
        for (int t = 0; t < 127; t++) { int o = hist[0] ^ hist[3]; c[t] = (uint8_t)o; for (int q = 0; q < 6; q++) hist[q] = hist[q + 1]; hist[6] = o; }
        memcpy(seq, c, 127);
        for (int s7 = 0; s7 < 128; s7++) {
            phase[s7] = 255;
            for (int t = 0; t < 127; t++) { bool ok = true; for (int q = 0; q < 7 && ok; q++) ok = c[(t + 127 - 7 + q) % 127] == ((s7 >> q) & 1); if (ok) { phase[s7] = (uint8_t)t; break; } }
        }
    }
    TableArena ar;
    const size_t o_a = ar.add(tw128, sizeof tw128), o_b = ar.add(tw32, sizeof tw32), o_s = ar.add(seq, 127), o_p = ar.add(phase, 128), o_pre = ar.add(nullptr, 640 * 4);
    const int rc = ar.upload(h, h->tabtx, "cudaMalloc tx tables", "tx table upload");
    if (rc != SB200_OK) return rc;
    char* base = (char*)h->tabtx.p;
    DevTablesTx& X = h->X;
    X.tw128 = (const uint32_t*)(base + o_a); X.tw32 = (const uint32_t*)(base + o_b); X.scr_seq = (const uint8_t*)(base + o_s); X.scr_phase = (const uint8_t*)(base + o_p);
    X.preamble = (uint32_t*)(base + o_pre);
    k_tx11a_preamble<<<1, 32>>>(X);
    const cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { h->tabtx.release(); return h->fail(SB200_E_CUDA, "k_tx11a_preamble", e); }
    h->launches += 1;
    return SB200_OK;
}

// 802.11a rates: SIGNAL rate code, coded bits per subcarrier, code rate, data bits per symbol (ieee80211a_cmn.h:66-157; bba.h:179-186, atx.h:20-57)
struct Rate11a { uint32_t kbps, code, nbpsc, cr, ndbps; };
static const Rate11a kRates11a[8] = {{6000, 0xB, 1, CR_12, 24}, {9000, 0xF, 1, CR_34, 36}, {12000, 0xA, 2, CR_12, 48}, {18000, 0xE, 2, CR_34, 72},
    {24000, 0x9, 4, CR_12, 96}, {36000, 0xD, 4, CR_34, 144}, {48000, 0x8, 6, CR_23, 192}, {54000, 0xC, 6, CR_34, 216}};
// 802.11b rates: SIGNAL rate code, chips per PSDU byte (bb/bbb.h:47-50, DataRate.h:40-43)
struct Rate11b { uint32_t kbps, code, chips_per_byte; };
static const Rate11b kRates11b[4] = {{1000, 0x0A, 88}, {2000, 0x14, 44}, {5500, 0x37, 16}, {11000, 0x6E, 8}};
template <class R, size_t N> static const R* find_rate(const R (&rates)[N], uint32_t kbps) {
    for (const R& r : rates) if (r.kbps == kbps) return &r;
    return nullptr;
}

// The FCS of every payload (k_tx11a_crc) into the crc workspace, for the transmitters that append it
static int crc_pass(sb200_handle* h, cudaStream_t st, const uint8_t* d_pay, const uint64_t* d_off, const uint32_t* d_len, uint32_t nframes, const uint32_t** d_crc) {
    CK(h->crc.need(nframes * 4ull));
    k_tx11a_crc<<<(nframes + 127) / 128, 128, 0, st>>>(d_pay, d_off, d_len, nframes, h->T, (uint32_t*)h->crc.p);
    *d_crc = (const uint32_t*)h->crc.p; h->launches += 1;
    return SB200_OK;
}

extern "C" int sb200_tx11a_batch(sb200_handle* h, const uint8_t* payload, uint64_t payload_total, const uint64_t* pay_off, const uint32_t* pay_len, const uint8_t* seeds,
                                 uint32_t nframes, uint32_t rate_kbps, uint32_t lead_samples, uint32_t sample_bits, void* out, uint64_t out_stride_samples,
                                 uint32_t* nsamples, void* cuda_stream) {
    if (!h || !payload || !pay_off || !pay_len || !out) return h ? h->fail(SB200_E_INVALID, "null argument") : SB200_E_INVALID;
    if (sample_bits != 8 && sample_bits != 16) return h->fail(SB200_E_INVALID, "sample_bits must be 8 (COMPLEX8) or 16 (COMPLEX16 = COMPLEX8 << 8)");
    if (nframes == 0) return SB200_OK;
    const Rate11a* R = find_rate(kRates11a, rate_kbps);
    if (!R) return h->fail(SB200_E_INVALID, "rate_kbps is not an 802.11a rate");
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin()); call.reads(payload); call.reads(seeds);
    int rc = upload_tables_tx(h); if (rc != SB200_OK) return rc;
    // frame table on the host (sizes the grid and checks the slots)
    FrameTable ft(pay_off, pay_len, nframes);
    TxJob job{}; job.rate_code = R->code; job.nbpsc = R->nbpsc; job.code_rate = R->cr; job.ndbps = R->ndbps; job.ndbps_pad = rate_kbps == 9000 ? 72 : R->ndbps;
    job.lead = lead_samples; job.fmt16 = sample_bits == 16;
    uint32_t max_nsym = 0;
    rc = ft.load(h, st, payload_total, [&](uint32_t i, bool inside) {
        if (ft.lenh[i] > 4091u || !inside) return h->fail(SB200_E_INVALID, "payload slot out of range (LENGTH is 12 bits incl. FCS)");
        const uint32_t ns = tx11a_nsym(ft.lenh[i], job.ndbps, job.ndbps_pad);
        if ((uint64_t)lead_samples + 640u + 160ull * (1u + ns) > out_stride_samples) return h->fail(SB200_E_INVALID, "out_stride_samples too small for the frame");
        if (ns > max_nsym) max_nsym = ns;
        return SB200_OK;
    });
    if (rc != SB200_OK) return rc;
    job.max_sym = 1u + max_nsym;
    const uint8_t* d_pay; const uint64_t* d_off; const uint32_t* d_len; const uint8_t* d_seed = nullptr;
    CK(to_device(h->txpay, payload, is_device_ptr(payload), payload_total, st, &d_pay));
    CK(ft.upload(h->txoff, h->txlen, st, &d_off, &d_len));
    if (seeds) CK(to_device(h->txseed, seeds, is_device_ptr(seeds), nframes, st, &d_seed));
    const size_t bps = sample_bits == 16 ? 4 : 2, out_bytes = (size_t)nframes * out_stride_samples * bps;
    Returns ret; void* d_out; uint32_t* d_ns;
    CK(ret.bind(h->txout, out, out_bytes, &d_out));
    CK(ret.bind(h->txns, nsamples, nframes * 4ull, &d_ns));
    const unsigned helpers = 8;                          // warps per frame for the preamble and the zero fill
    dim3 grid(nframes, (job.max_sym + helpers + SB_TX_WARPS - 1) / SB_TX_WARPS);
    CK(cudaEventRecord(h->ev0, st));
    const uint32_t* d_crc; rc = crc_pass(h, st, d_pay, d_off, d_len, nframes, &d_crc); if (rc != SB200_OK) return rc;
    k_tx11a<<<grid, 32 * SB_TX_WARPS, 0, st>>>(d_pay, d_off, d_len, d_seed, nframes, job, h->T, h->X, h->inv_deint, d_crc, d_out, out_stride_samples, d_ns);
    return finish_call(h, st, ret, 0, 1);
}

// 802.11b transmit (tx11b_kernels.cuh)
extern "C" int sb200_tx11b_batch(sb200_handle* h, const uint8_t* payload, uint64_t payload_total, const uint64_t* pay_off, const uint32_t* pay_len,
                                 uint32_t nframes, uint32_t rate_kbps, uint32_t init_phase, uint32_t lead_samples, uint32_t sample_bits, void* out,
                                 uint64_t out_stride_samples, uint32_t* nsamples, uint32_t* final_phase, void* cuda_stream) {
    if (!h || !payload || !pay_off || !pay_len || !out) return h ? h->fail(SB200_E_INVALID, "null argument") : SB200_E_INVALID;
    if (sample_bits != 8 && sample_bits != 16) return h->fail(SB200_E_INVALID, "sample_bits must be 8 (COMPLEX8) or 16 (COMPLEX16 = COMPLEX8 << 8)");
    if (out_stride_samples % 8u || ((uintptr_t)out & 15u)) return h->fail(SB200_E_INVALID, "out must be 16-byte aligned and out_stride_samples a multiple of 8");
    if (nframes == 0) return SB200_OK;
    Tx11bJob job{};
    job.rate_kbps = rate_kbps; job.lead = lead_samples; job.fmt16 = sample_bits == 16; job.init_phase = init_phase & 3u;
    const Rate11b* R = find_rate(kRates11b, rate_kbps);
    if (!R) return h->fail(SB200_E_INVALID, "rate_kbps is not an 802.11b rate");
    job.rate_code = R->code; job.chips_per_byte = R->chips_per_byte;
    for (int k = 0; k < 20; k++) {                                                      // pulse.hpp:292-300, with that file's own PI
        const int i = 8 - k; const double PI_ = 3.141593;
        const double x = (i == 1 || i == -1) ? 1.0 : 4 * cos(PI_ * i / 2) / PI_ / (1 - i * i);
        job.taps[k] = (short)(x * 80 + .5);
    }
    {   const int H[20] = SB_TX11B_TAPS;                                                    // the aligned kernel's compile-time copy
        for (int k = 0; k < 20; k++) if (job.taps[k] != H[k]) return h->fail(SB200_E_INVALID, "shaper taps differ from the compiled constants"); }
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin()); call.reads(payload);
    FrameTable ft(pay_off, pay_len, nframes);
    uint32_t max_len = 0;
    int rc = ft.load(h, st, payload_total, [&](uint32_t i, bool inside) {
        const uint32_t len = ft.lenh[i];
        if (len > 4091u || !inside) return h->fail(SB200_E_INVALID, "payload slot out of range (frame_length 1..4095 incl. FCS)");
        if ((uint64_t)lead_samples + tx11b_nsamples(tx11b_nchips(len, job.chips_per_byte)) > out_stride_samples) return h->fail(SB200_E_INVALID, "out_stride_samples too small for the frame");
        if (len > max_len) max_len = len;
        return SB200_OK;
    });
    if (rc != SB200_OK) return rc;
    job.desc_stride = (24u + max_len + 4u + 7u) & ~7u;
    const uint8_t* d_pay; const uint64_t* d_off; const uint32_t* d_len;
    CK(to_device(h->txpay, payload, is_device_ptr(payload), payload_total, st, &d_pay));
    CK(ft.upload(h->txoff, h->txlen, st, &d_off, &d_len));
    const size_t bps = sample_bits == 16 ? 4 : 2, out_bytes = (size_t)nframes * out_stride_samples * bps;
    Returns ret; void* d_out; uint32_t* d_ns; uint32_t* d_fp;
    CK(ret.bind(h->txout, out, out_bytes, &d_out));
    CK(ret.bind(h->txns, nsamples, nframes * 4ull, &d_ns));
    CK(ret.bind(h->txseed, final_phase, nframes * 4ull, &d_fp));
    CK(h->crc.need(nframes * 4ull)); CK(h->txdesc.need((size_t)nframes * job.desc_stride * 2ull));   // sized before ev0: crc_pass then finds it large enough
    const uint64_t per_cta = (uint64_t)SB_TX11B_THREADS * SB_TX11B_SPT, ny = (out_stride_samples + per_cta - 1) / per_cta;
    if (ny > 65535u || (uint64_t)lead_samples + out_stride_samples >= (1ull << 27)) return h->fail(SB200_E_INVALID, "out_stride_samples too large");
    CK(cudaEventRecord(h->ev0, st));
    const uint32_t* d_crc; rc = crc_pass(h, st, d_pay, d_off, d_len, nframes, &d_crc); if (rc != SB200_OK) return rc;
    k_tx11b_code<<<(nframes + 127) / 128, 128, 0, st>>>(d_pay, d_off, d_len, nframes, job, d_crc, (uint16_t*)h->txdesc.p, d_fp);
    {   const dim3 grid(nframes, (unsigned)ny); const uint16_t* dd = (const uint16_t*)h->txdesc.p; const bool al = lead_samples % 4u == 0;
#define SB_TX11B_LAUNCH(R) do { if (al) k_tx11b_shape<true, R><<<grid, SB_TX11B_THREADS, 0, st>>>(d_len, job, dd, d_out, out_stride_samples, d_ns); \
                                else k_tx11b_shape<false, R><<<grid, SB_TX11B_THREADS, 0, st>>>(d_len, job, dd, d_out, out_stride_samples, d_ns); } while (0)
        switch (rate_kbps) { case 1000: SB_TX11B_LAUNCH(1000); break; case 2000: SB_TX11B_LAUNCH(2000); break; case 5500: SB_TX11B_LAUNCH(5500); break; default: SB_TX11B_LAUNCH(11000); break; }
#undef SB_TX11B_LAUNCH
    }
    return finish_call(h, st, ret, 0, 2);
}

// Legacy 802.11b transmit filter (tx11b_legacy_kernels.cuh): BB11BPMDSpreadFIR4SSE (variant 0) / BB11BPMDSpreadFIR4ASM (variant 1), batched.
extern "C" int sb200_tx11b_fir37(sb200_handle* h, const int8_t* chips, uint64_t chips_total, const uint64_t* frame_off, const uint32_t* frame_len,
                                 uint32_t nframes, uint32_t variant, int8_t* out, void* cuda_stream) {
    if (!h || !chips || !frame_off || !frame_len || !out) return h ? h->fail(SB200_E_INVALID, "null argument") : SB200_E_INVALID;
    if (variant > 1) return h->fail(SB200_E_INVALID, "variant must be 0 (BB11BPMDSpreadFIR4SSE) or 1 (BB11BPMDSpreadFIR4ASM)");
    if (nframes == 0) return SB200_OK;
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin()); call.reads(chips);
    FrameTable ft(frame_off, frame_len, nframes);
    const bool in_dev = is_device_ptr(chips), out_dev = is_device_ptr(out);
    uint32_t max_len = 0;
    const int rc = ft.load(h, st, chips_total, [&](uint32_t i, bool inside) {
        if ((ft.lenh[i] & 7u) || (ft.offh[i] & 7u)) return h->fail(SB200_E_INVALID, "frame_off and frame_len must be multiples of 8 samples (the reference fails on uiInputSize & 7 and needs 16-byte aligned buffers)");
        if (!inside) return h->fail(SB200_E_INVALID, "frame exceeds chips_total");
        if (ft.lenh[i] > max_len) max_len = ft.lenh[i];
        return SB200_OK;
    });
    if (rc != SB200_OK) return rc;
    if ((in_dev && ((uintptr_t)chips & 15u)) || (out_dev && ((uintptr_t)out & 15u))) return h->fail(SB200_E_INVALID, "device buffers must be 16-byte aligned");
    const int8_t* d_in; int8_t* d_out = out; const uint64_t* d_off; const uint32_t* d_len;
    CK(to_device(h->txpay, chips, in_dev, chips_total * 2ull, st, &d_in, 16));
    if (!out_dev) { CK(h->txout.need(chips_total * 2ull + 16)); d_out = (int8_t*)h->txout.p; }
    CK(ft.upload(h->txoff, h->txlen, st, &d_off, &d_len));
    const uint64_t groups = (uint64_t)(max_len >> 3) * 2u; uint64_t ny = (groups + SB_FIR37_THREADS - 1) / SB_FIR37_THREADS; if (ny > 4096) ny = 4096; if (ny == 0) ny = 1;
    CK(cudaEventRecord(h->ev0, st));
    const dim3 grid(nframes, (unsigned)ny);
    if (variant == 0) k_fir37_legacy<0><<<grid, SB_FIR37_THREADS, 0, st>>>(d_in, d_off, d_len, nframes, d_out);
    else k_fir37_legacy<1><<<grid, SB_FIR37_THREADS, 0, st>>>(d_in, d_off, d_len, nframes, d_out);
    Returns none;                                       // only the frames' own ranges are defined: copied back one by one below (they may be sparse in the buffer)
    const int frc = finish_call(h, st, none, 0, 1);
    if (frc != SB200_OK || out_dev) return frc;
    for (uint32_t i = 0; i < nframes; i++) if (ft.lenh[i]) CK(cudaMemcpyAsync(out + 2ull * ft.offh[i], d_out + 2ull * ft.offh[i], 2ull * ft.lenh[i], cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return SB200_OK;
}

// Legacy 802.11b transmitter (tx11b_legacy_kernels.cuh): BB11BPMDBufferTx4XWith{Long,Short}Header, optionally followed by the 37-tap filter.
extern "C" int sb200_tx11b_legacy_batch(sb200_handle* h, const uint8_t* payload, uint64_t payload_total, const uint64_t* pay_off, const uint32_t* pay_len,
                                        uint32_t nframes, uint32_t rate_kbps, uint32_t short_preamble, uint32_t flags, uint32_t filter, int8_t* out,
                                        uint64_t out_stride_samples, uint32_t* nsamples, void* cuda_stream) {
    if (!h || !payload || !pay_off || !pay_len || !out) return h ? h->fail(SB200_E_INVALID, "null argument") : SB200_E_INVALID;
    if (flags & SB200_TX11B_LEGACY_PBCC) return h->fail(SB200_E_INVALID, "PBCC is not supported: the reference only lengthens PLCPGetLength for it and still sends CCK");
    if (flags & ~SB200_TX11B_LEGACY_FCS_IN_PAYLOAD) return h->fail(SB200_E_INVALID, "unknown flags");
    if (filter > 2) return h->fail(SB200_E_INVALID, "filter must be 0 (encoder output), 1 (BB11BPMDSpreadFIR4SSE) or 2 (BB11BPMDSpreadFIR4ASM)");
    if (short_preamble > 1) return h->fail(SB200_E_INVALID, "short_preamble must be 0 or 1");
    if (out_stride_samples % 8u || ((uintptr_t)out & 15u)) return h->fail(SB200_E_INVALID, "out must be 16-byte aligned and out_stride_samples a multiple of 8");
    if (nframes == 0) return SB200_OK;
    Tx11bLegacyJob job{};
    job.rate_kbps = rate_kbps; job.short_preamble = short_preamble; job.fcs_in_payload = (flags & SB200_TX11B_LEGACY_FCS_IN_PAYLOAD) ? 1u : 0u; job.filter = filter;
    const Rate11b* R = find_rate(kRates11b, rate_kbps);
    if (!R) return h->fail(SB200_E_INVALID, "rate_kbps is not an 802.11b rate");
    job.rate_code = R->code; job.data_chips_per_byte = short_preamble && rate_kbps == 1000 ? 0u : R->chips_per_byte;   // the short preamble's 1 Mbps case sends no data chips
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin()); call.reads(payload);
    FrameTable ft(pay_off, pay_len, nframes);
    uint32_t max_size = 0;
    int rc = ft.load(h, st, payload_total, [&](uint32_t i, bool inside) {
        const uint32_t len = ft.lenh[i], size = job.fcs_in_payload ? len : len + 4u;    // PSDU bytes, FCS included
        if (job.fcs_in_payload && len < 4u) return h->fail(SB200_E_INVALID, "with SB200_TX11B_LEGACY_FCS_IN_PAYLOAD every payload carries its 4 FCS bytes");
        if (len > 4095u || size > 4095u || !inside) return h->fail(SB200_E_INVALID, "payload slot out of range (PSDU 4 .. 4095 bytes incl. FCS)");
        if (tx11b_legacy_nsamples(size, short_preamble, job.data_chips_per_byte) > out_stride_samples) return h->fail(SB200_E_INVALID, "out_stride_samples too small for the frame");
        if (size > max_size) max_size = size;
        return SB200_OK;
    });
    if (rc != SB200_OK) return rc;
    job.desc_stride = (24u + max_size + 7u) & ~7u;
    const uint8_t* d_pay; const uint64_t* d_off; const uint32_t* d_len;
    CK(to_device(h->txpay, payload, is_device_ptr(payload), payload_total, st, &d_pay));
    CK(ft.upload(h->txoff, h->txlen, st, &d_off, &d_len));
    const size_t out_bytes = (size_t)nframes * out_stride_samples * 2;
    Returns ret; int8_t* d_out; uint32_t* d_ns;
    CK(ret.bind(h->txout, out, out_bytes, &d_out));
    CK(ret.bind(h->txns, nsamples, nframes * 4ull, &d_ns));
    CK(h->txdesc.need((size_t)nframes * job.desc_stride * 2ull));
    const uint64_t per_cta = SB_TX11B_LEGACY_THREADS * 8, ny = (out_stride_samples + per_cta - 1) / per_cta;
    if (ny > 65535u) return h->fail(SB200_E_INVALID, "out_stride_samples too large");
    CK(cudaEventRecord(h->ev0, st));
    const uint32_t* d_crc = nullptr;
    if (!job.fcs_in_payload) { rc = crc_pass(h, st, d_pay, d_off, d_len, nframes, &d_crc); if (rc != SB200_OK) return rc; }
    k_tx11b_legacy_code<<<(nframes + 127) / 128, 128, 0, st>>>(d_pay, d_off, d_len, nframes, job, d_crc, (uint16_t*)h->txdesc.p);
    const dim3 grid(nframes, (unsigned)ny); const uint16_t* dd = (const uint16_t*)h->txdesc.p;
    if (filter == 0) k_tx11b_legacy_spread<0><<<grid, SB_TX11B_LEGACY_THREADS, 0, st>>>(d_len, job, dd, d_out, out_stride_samples, d_ns);
    else if (filter == 1) k_tx11b_legacy_spread<1><<<grid, SB_TX11B_LEGACY_THREADS, 0, st>>>(d_len, job, dd, d_out, out_stride_samples, d_ns);
    else k_tx11b_legacy_spread<2><<<grid, SB_TX11B_LEGACY_THREADS, 0, st>>>(d_len, job, dd, d_out, out_stride_samples, d_ns);
    return finish_call(h, st, ret, 0, 2);
}

// Legacy 802.11a transmitter (tx11a_legacy_kernels.cuh): BB11ATxFrameMod / BB11ATxBufferMod6M at SampleRate 40 or 44.
extern "C" int sb200_tx11a_legacy_batch(sb200_handle* h, const uint8_t* payload, uint64_t payload_total, const uint64_t* pay_off, const uint32_t* pay_len,
                                        uint32_t nframes, uint32_t rate_kbps, uint32_t sample_rate_mhz, uint32_t flags, const int16_t* preamble, int8_t* out,
                                        uint64_t out_stride_samples, uint32_t* nsamples, void* cuda_stream) {
    if (!h || !payload || !pay_off || !pay_len || !out || !preamble) return h ? h->fail(SB200_E_INVALID, "null argument") : SB200_E_INVALID;
    if (flags & ~SB200_TX11A_LEGACY_FCS_IN_PAYLOAD) return h->fail(SB200_E_INVALID, "unknown flags");
    if (sample_rate_mhz != 40 && sample_rate_mhz != 44) return h->fail(SB200_E_INVALID, "sample_rate_mhz must be 40 or 44");
    if (out_stride_samples % 8u || ((uintptr_t)out & 15u)) return h->fail(SB200_E_INVALID, "out must be 16-byte aligned and out_stride_samples a multiple of 8");
    if (nframes == 0) return SB200_OK;
    const Rate11a* R = find_rate(kRates11a, rate_kbps);
    if (!R) return h->fail(SB200_E_INVALID, "rate_kbps is not an 802.11a rate");
    Tx11aLegacyJob job{};
    job.rate_code = R->code; job.nbpsc = R->nbpsc; job.code_rate = R->cr; job.ndbps = R->ndbps;
    job.sr44 = sample_rate_mhz == 44; job.fcs_in_payload = (flags & SB200_TX11A_LEGACY_FCS_IN_PAYLOAD) ? 1u : 0u;
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin()); call.reads(payload); call.reads(preamble);
    int rc = upload_tables_tx(h); if (rc != SB200_OK) return rc;
    FrameTable ft(pay_off, pay_len, nframes);
    const bool pre_dev = is_device_ptr(preamble);
    uint32_t max_nsym = 0;
    rc = ft.load(h, st, payload_total, [&](uint32_t i, bool inside) {
        const uint32_t len = ft.lenh[i], size = job.fcs_in_payload ? len : len + 4u;    // PSDU bytes, FCS included
        if (job.fcs_in_payload && len < 4u) return h->fail(SB200_E_INVALID, "with SB200_TX11A_LEGACY_FCS_IN_PAYLOAD every payload carries its 4 FCS bytes");
        if (len > 4096u || size > 4096u || !inside) return h->fail(SB200_E_INVALID, "payload slot out of range (MPDU + FCS at most 4096 bytes)");
        const uint32_t ns = tx11a_legacy_nsym(size, job.ndbps);
        if (tx11a_legacy_padded(ns, job.sr44) > out_stride_samples) return h->fail(SB200_E_INVALID, "out_stride_samples too small for the frame");
        if (ns > max_nsym) max_nsym = ns;
        return SB200_OK;
    });
    if (rc != SB200_OK) return rc;
    job.runs = (1u + max_nsym + SB_TXL_RUN - 1u) / SB_TXL_RUN;
    const uint8_t* d_pay; const uint64_t* d_off; const uint32_t* d_len; const uint32_t* d_pre;
    CK(to_device(h->txpay, payload, is_device_ptr(payload), payload_total, st, &d_pay, 1));
    CK(ft.upload(h->txoff, h->txlen, st, &d_off, &d_len));
    if (pre_dev && ((uintptr_t)preamble & 3u) == 0) d_pre = (const uint32_t*)preamble;
    else { CK(h->txpre.need(640 * 4)); CK(cudaMemcpyAsync(h->txpre.p, preamble, 640 * 4, pre_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st)); d_pre = (const uint32_t*)h->txpre.p; }
    const size_t out_bytes = (size_t)nframes * out_stride_samples * 2;
    Returns ret; int8_t* d_out; uint32_t* d_ns;
    CK(ret.bind(h->txout, out, out_bytes, &d_out));
    CK(ret.bind(h->txns, nsamples, nframes * 4ull, &d_ns));
    const unsigned helpers = 4;                          // warps per frame for the preamble and the zero fill
    const uint64_t ny = (job.runs + helpers + SB_TXL_WARPS - 1) / SB_TXL_WARPS;
    if (ny > 65535u) return h->fail(SB200_E_INVALID, "too many symbols per frame");
    CK(cudaEventRecord(h->ev0, st));
    const uint32_t* d_crc = nullptr;
    if (!job.fcs_in_payload) { rc = crc_pass(h, st, d_pay, d_off, d_len, nframes, &d_crc); if (rc != SB200_OK) return rc; }
    k_tx11a_legacy<<<dim3(nframes, (unsigned)ny), 32 * SB_TXL_WARPS, 0, st>>>(d_pay, d_off, d_len, nframes, job, h->T, h->X, h->inv_deint, d_crc, d_pre, d_out, out_stride_samples, d_ns);
    return finish_call(h, st, ret, 0, 1);
}

// 802.11n transmit (tx11n_kernels.cuh)
static int upload_tables_tx11n(sb200_handle* h) {
    if (h->tabtx11n.p) return SB200_OK;
    // the four preamble tables (Brick11/src/_b_lstf.h, _b_lltf.h, _b_htstf.h, _b_htltf.h) from their defining formula: 128-point inverse DFTs of
    // the L-STF / L-LTF / HT-LTF tone sets, equal power, one common amplitude (fitted: the literal tables fix it to 362.0592 +- 0.0001)
    const double A = 362.0592, PI_ = 3.14159265358979323846;
    static const int8_t L[53] = {1,1,-1,-1,1,1,-1,1,-1,1,1,1,1,1,1,-1,-1,1,1,-1,1,-1,1,1,1,1,0,
                                 1,-1,-1,1,1,-1,1,-1,1,-1,-1,-1,-1,-1,1,1,-1,-1,1,-1,1,-1,1,1,1,1};
    std::vector<double> Sre(3 * 128, 0.0), Sim(3 * 128, 0.0);
    static const int stf_k[12] = {-24, -20, -16, -12, -8, -4, 4, 8, 12, 16, 20, 24}; static const int stf_s[12] = {1, -1, 1, -1, -1, 1, -1, -1, 1, 1, 1, 1};
    for (int i = 0; i < 12; i++) { Sre[(stf_k[i] + 128) % 128] = stf_s[i]; Sim[(stf_k[i] + 128) % 128] = stf_s[i]; }
    for (int k = -26; k <= 26; k++) Sre[128 + (k + 128) % 128] = L[k + 26];
    for (int k = -28; k <= 28; k++) Sre[256 + (k + 128) % 128] = k == -28 || k == -27 ? 1 : k == 27 || k == 28 ? -1 : L[k + 26];
    auto gen = [&](int set, double scale, int n0, int count, uint32_t* out) {
        for (int i = 0; i < count; i++) {
            const int n = n0 + i; double re = 0, im = 0;
            for (int k = 0; k < 128; k++) {
                const double sr = Sre[set * 128 + k], si = Sim[set * 128 + k];
                if (sr == 0 && si == 0) continue;
                const double ph = 2 * PI_ * (double)((((long long)k * n) % 128 + 128) % 128) / 128, c = cos(ph), sn = sin(ph);
                re += sr * c - si * sn; im += sr * sn + si * c;
            }
            out[i] = pack(mk((int)lround(re * scale), (int)lround(im * scale)));
        }
    };
    std::vector<uint32_t> lstf(320), lltf(320), htstf(160), htltf(160), pre(2 * 1120);
    gen(0, A, 0, 320, lstf.data()); gen(1, A * sqrt(24.0 / 52.0), -64, 320, lltf.data()); gen(0, A, -32, 160, htstf.data()); gen(2, A * sqrt(24.0 / 56.0), -32, 160, htltf.data());
    auto negw = [](uint32_t w) { const cs16 c = unpack(w); return pack(mk(-c.re, -c.im)); };
    // stream 1 (preamble11n.hpp:22-37,56-76): tables as they are, second HT-LTF negated; stream 2: 200 ns / 400 ns cyclic delays
    for (int i = 0; i < 320; i++) { pre[i] = lstf[i]; pre[320 + i] = lltf[i]; pre[1120 + (i + 8) % 320] = lstf[i]; }
    for (int i = 0; i < 256; i++) pre[1120 + 320 + 64 + i] = lltf[64 + i - 8];
    for (int i = 0; i < 64; i++) pre[1120 + 320 + i] = pre[1120 + 320 + 256 + i];
    for (int i = 0; i < 160; i++) { pre[640 + i] = htstf[i]; pre[800 + i] = htltf[i]; pre[960 + i] = negw(htltf[i]); pre[1120 + 640 + (i + 16) % 160] = htstf[i]; }
    for (int r = 0; r < 2; r++) { uint32_t* o = pre.data() + 1120 + 800 + 160 * r; for (int i = 0; i < 128; i++) o[32 + i] = htltf[32 + i - 16]; for (int i = 0; i < 32; i++) o[i] = o[128 + i]; }
    // inverse of T11Interleave<52 N_BPSC, N_BPSC, 13, 11, I_SS> (interleave.hpp:33-60): air position -> stream bit
    std::vector<uint8_t> inv(4 * 104, 0);
    for (int bi = 0; bi < 2; bi++) for (int iss = 1; iss <= 2; iss++) {
        const int nbpsc = bi + 1, ncbps = 52 * nbpsc, ncol = 13, nrot = 11, ns = 1;
        for (int k = 0; k < ncbps; k++) {
            const int i = ncbps / ncol * (k % ncol) + k / ncol, j = ns * (i / ns) + (i + ncbps - ncol * i / ncbps) % ns;
            const int r = (ncbps + j - (((iss - 1) * 2) % 3 + 3 * ((iss - 1) / 3)) * nrot * nbpsc) % ncbps;
            inv[(bi * 2 + iss - 1) * 104 + r] = (uint8_t)k;
        }
    }
    std::vector<uint16_t> inv16(4 * 312, 0);                                                  // the same for 16-QAM (s = 2) and 64-QAM (s = 3): T11nInterleaveQAM16/64_S1/_S2
    for (int bi = 0; bi < 2; bi++) for (int iss = 1; iss <= 2; iss++) {
        const int nbpsc = bi ? 6 : 4, ncbps = 52 * nbpsc, ncol = 13, nrot = 11, ns = nbpsc / 2;
        for (int k = 0; k < ncbps; k++) {
            const int i = ncbps / ncol * (k % ncol) + k / ncol, j = ns * (i / ns) + (i + ncbps - ncol * i / ncbps) % ns;
            const int r = (ncbps + j - (((iss - 1) * 2) % 3 + 3 * ((iss - 1) / 3)) * nrot * nbpsc) % ncbps;
            inv16[(bi * 2 + iss - 1) * 312 + r] = (uint16_t)k;
        }
    }
    TableArena ar;
    const size_t o_pre = ar.add(pre.data(), pre.size() * 4), o_inv = ar.add(inv.data(), inv.size()), o_inv16 = ar.add(inv16.data(), inv16.size() * 2);
    const int rc = ar.upload(h, h->tabtx11n, "cudaMalloc tx11n tables", "tx11n table upload");
    if (rc != SB200_OK) return rc;
    const char* base = (const char*)h->tabtx11n.p;
    h->XN.pre = (const uint32_t*)(base + o_pre); h->XN.inv = (const uint8_t*)(base + o_inv); h->XN.inv16 = (const uint16_t*)(base + o_inv16);
    return SB200_OK;
}

extern "C" int sb200_tx11n_batch(sb200_handle* h, const uint8_t* payload, uint64_t payload_total, const uint64_t* pay_off, const uint32_t* pay_len, const uint8_t* seeds,
                                 uint32_t nframes, uint32_t mcs, uint32_t lead_samples, int16_t* out0, int16_t* out1, uint64_t out_stride_samples,
                                 uint32_t* nsamples, void* cuda_stream) {
    if (!h || !payload || !pay_off || !pay_len || !out0 || !out1) return h ? h->fail(SB200_E_INVALID, "null argument") : SB200_E_INVALID;
    if (nframes == 0) return SB200_OK;
    Tx11nJob job{}; job.mcs = mcs; job.lead = lead_samples;
    switch (mcs) {                                      // ieee80211const.h:35-55; the range the receiver accepts (PHY_11n.hpp:496-501)
        case 8:  job.nbpsc = 1; job.code_rate = CR_12; job.ndbps = 52;  job.enc_in = 1; job.parse_in = 13; break;
        case 9:  job.nbpsc = 2; job.code_rate = CR_12; job.ndbps = 104; job.enc_in = 1; job.parse_in = 26; break;
        case 10: job.nbpsc = 2; job.code_rate = CR_34; job.ndbps = 156; job.enc_in = 3; job.parse_in = 26; break;
        case 11: job.nbpsc = 4; job.code_rate = CR_12; job.ndbps = 208; job.enc_in = 1; job.parse_in = 52; break;      // the 16-QAM / 64-QAM branches of the modulator graph
        case 12: job.nbpsc = 4; job.code_rate = CR_34; job.ndbps = 312; job.enc_in = 3; job.parse_in = 52; break;      // (fb11nmod_config.hpp:133-155: enc11 .. enc14)
        case 13: job.nbpsc = 6; job.code_rate = CR_23; job.ndbps = 416; job.enc_in = 2; job.parse_in = 78; break;
        case 14: job.nbpsc = 6; job.code_rate = CR_34; job.ndbps = 468; job.enc_in = 3; job.parse_in = 78; break;
        default: return h->fail(SB200_E_INVALID, "mcs must be 8 .. 14");
    }
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin()); call.reads(payload); call.reads(seeds);
    int rc = upload_tables_tx(h); if (rc != SB200_OK) return rc;
    rc = upload_tables_tx11n(h); if (rc != SB200_OK) return rc;
    FrameTable ft(pay_off, pay_len, nframes);
    if (is_device_ptr(out0) != is_device_ptr(out1)) return h->fail(SB200_E_INVALID, "both output buffers must live on the same side");
    uint32_t max_nsym = 0;
    rc = ft.load(h, st, payload_total, [&](uint32_t i, bool inside) {
        if (ft.lenh[i] > 4091u || !inside) return h->fail(SB200_E_INVALID, "payload slot out of range");
        const uint32_t ns = tx11n_nsym_emitted(ft.lenh[i], job, nullptr, nullptr);
        if ((uint64_t)lead_samples + 1600u + 160ull * ns > out_stride_samples) return h->fail(SB200_E_INVALID, "out_stride_samples too small for the frame");
        if (ns > max_nsym) max_nsym = ns;
        return SB200_OK;
    });
    if (rc != SB200_OK) return rc;
    job.max_sym = 3u + max_nsym;
    const uint8_t* d_pay; const uint64_t* d_off; const uint32_t* d_len; const uint8_t* d_seed = nullptr;
    CK(to_device(h->txpay, payload, is_device_ptr(payload), payload_total, st, &d_pay));
    CK(ft.upload(h->txoff, h->txlen, st, &d_off, &d_len));
    if (seeds) CK(to_device(h->txseed, seeds, is_device_ptr(seeds), nframes, st, &d_seed));
    const size_t out_bytes = (size_t)nframes * out_stride_samples * 4;
    Returns ret; int16_t* d_o0; int16_t* d_o1; uint32_t* d_ns;
    CK(ret.bind(h->txout, out0, out_bytes, &d_o0));
    CK(ret.bind(h->txout1, out1, out_bytes, &d_o1));
    CK(ret.bind(h->txns, nsamples, nframes * 4ull, &d_ns));
    const unsigned helpers = 8;
    dim3 grid(nframes, (2u * job.max_sym + helpers + SB_TX11N_WARPS - 1) / SB_TX11N_WARPS);
    CK(cudaEventRecord(h->ev0, st));
    const uint32_t* d_crc; rc = crc_pass(h, st, d_pay, d_off, d_len, nframes, &d_crc); if (rc != SB200_OK) return rc;
    k_tx11n<<<grid, 32 * SB_TX11N_WARPS, 0, st>>>(d_pay, d_off, d_len, d_seed, nframes, job, h->T, h->X, h->XN, h->inv_deint, d_crc, (uint32_t*)d_o0, (uint32_t*)d_o1, out_stride_samples, d_ns);
    return finish_call(h, st, ret, 0, 1);
}
