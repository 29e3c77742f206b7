// sora_b200 — the transmitters: 802.11a, 802.11b, 802.11n and the legacy 802.11a / 802.11b ones, and the legacy 802.11b transmit filter.
#include "handle.cuh"
#include "tx_frames.cuh"
#include "tx11a_kernels.cuh"
#include "tx11b_kernels.cuh"
#include "tx11b_legacy_kernels.cuh"
#include "tx11a_legacy_kernels.cuh"
#include "tx11n_kernels.cuh"
#include <type_traits>

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

// ---- what the batch transmitters share ----------------------------------------------------------------------------------------------
// The argument checks before a transmitter looks at its rate: no null handle or pointer among `p`; then, after the chain's own checks,
// check_out(): the sample format (8 | 16) and, where `aligned_out` is given, 16-byte aligned output rows a multiple of 8 samples apart.
template <class... P> static int check_null(sb200_handle* h, const P*... p) {
    if (!h) return SB200_E_INVALID;
    return (p && ...) ? SB200_OK : h->fail(SB200_E_INVALID, "null argument");
}
static int check_out(sb200_handle* h, uint32_t sample_bits, const void* aligned_out, uint64_t out_stride_samples) {
    if (sample_bits != 8 && sample_bits != 16) return h->fail(SB200_E_INVALID, "sample_bits must be 8 (COMPLEX8) or 16 (COMPLEX16 = COMPLEX8 << 8)");
    if (aligned_out && (out_stride_samples % 8u || ((uintptr_t)aligned_out & 15u))) return h->fail(SB200_E_INVALID, "out must be 16-byte aligned and out_stride_samples a multiple of 8");
    return SB200_OK;
}

// f(std::integral_constant<int, i>()) for a runtime i of 0 .. N - 1 (checked by the caller): the transmit kernels take their rate, output
// alignment, filter or variant as a template parameter.
template <int N, class F> static void with_index(uint32_t i, F f) {
    if constexpr (N > 1) { if (i == N - 1) return f(std::integral_constant<int, N - 1>()); with_index<N - 1>(i, f); }
    else f(std::integral_constant<int, 0>());
}

// One call of a batch transmitter after its argument checks, in this order: begin() sets the device and opens the call (the payload and
// `in` are read on the stream); load() reads the frame table with the chain's own per-slot check (FrameTable::load); stage() places the
// payload and its off / len tables on the device; bind() binds `out` and nsamples; start() sizes the remaining workspaces, records ev0 and,
// for the chains that append the FCS, runs k_tx11a_crc into the crc workspace (d_crc, else null); finish() ends the call with the chain's
// own launches.  No workspace grows between ev0 and ev1.
struct TxCall {
    sb200_handle* h; cudaStream_t st; cudaError_t dev; CallScope scope; FrameTable ft; Returns ret;
    const uint8_t* d_pay = nullptr; const uint64_t* d_off = nullptr; const uint32_t* d_len = nullptr; uint32_t* d_ns = nullptr; const uint32_t* d_crc = nullptr;
    TxCall(sb200_handle* h_, void* stream, const uint64_t* off, const uint32_t* len, uint32_t n)
        : h(h_), st((cudaStream_t)stream), dev(cudaSetDevice(h_->device)), scope(h_, st), ft(off, len, n) {}
    int begin(const void* payload, const void* in = nullptr) {
        if (dev != cudaSuccess) return h->fail(SB200_E_CUDA, "cudaSetDevice(h->device)", dev);
        CK(scope.begin()); scope.reads(payload); scope.reads(in);
        return SB200_OK;
    }
    template <class Slot> int load(uint64_t total, Slot slot) { return ft.load(h, st, total, slot); }
    cudaError_t stage(const uint8_t* payload, uint64_t total, size_t slack = 0) {
        const cudaError_t e = to_device(h->txpay, payload, is_device_ptr(payload), total, st, &d_pay, slack);
        return e != cudaSuccess ? e : ft.upload(h->txoff, h->txlen, st, &d_off, &d_len);
    }
    template <class T> cudaError_t bind(T* out, size_t out_bytes, T** d_out, uint32_t* nsamples) {
        const cudaError_t e = ret.bind(h->txout, out, out_bytes, d_out);
        return e != cudaSuccess ? e : ret.bind(h->txns, nsamples, ft.n * 4ull, &d_ns);
    }
    cudaError_t start(bool fcs, size_t desc_bytes = 0) {
        cudaError_t e = fcs ? h->crc.need(ft.n * 4ull) : cudaSuccess;
        if (e == cudaSuccess && desc_bytes) e = h->txdesc.need(desc_bytes);
        if (e == cudaSuccess) e = cudaEventRecord(h->ev0, st);
        if (e != cudaSuccess || !fcs) return e;
        k_tx11a_crc<<<(ft.n + 127) / 128, 128, 0, st>>>(d_pay, d_off, d_len, ft.n, h->T, (uint32_t*)h->crc.p);
        d_crc = (const uint32_t*)h->crc.p; h->launches += 1;
        return cudaSuccess;
    }
    int finish(uint64_t launches) { return finish_call(h, st, ret, 0, launches); }
};

extern "C" int sb200_tx11a_batch(sb200_handle* h, const uint8_t* payload, uint64_t payload_total, const uint64_t* pay_off, const uint32_t* pay_len, const uint8_t* seeds,
                                 uint32_t nframes, uint32_t rate_kbps, uint32_t lead_samples, uint32_t sample_bits, void* out, uint64_t out_stride_samples,
                                 uint32_t* nsamples, void* cuda_stream) {
    int rc = check_null(h, payload, pay_off, pay_len, out);
    if (rc == SB200_OK) rc = check_out(h, sample_bits, nullptr, 0);
    if (rc != SB200_OK || nframes == 0) return rc;
    const Rate11a* R = find_rate(kRates11a, rate_kbps);
    if (!R) return h->fail(SB200_E_INVALID, "rate_kbps is not an 802.11a rate");
    TxJob job{}; job.rate_code = R->code; job.nbpsc = R->nbpsc; job.code_rate = R->cr; job.ndbps = R->ndbps; job.ndbps_pad = R->ndbps_pad;
    job.lead = lead_samples; job.fmt16 = sample_bits == 16;
    TxCall c(h, cuda_stream, pay_off, pay_len, nframes);
    uint32_t max_nsym = 0;
    if ((rc = c.begin(payload, seeds)) != SB200_OK || (rc = upload_tables_tx(h)) != SB200_OK) return rc;
    rc = c.load(payload_total, [&](uint32_t i, bool inside) {
        if (c.ft.lenh[i] > 4091u || !inside) return h->fail(SB200_E_INVALID, "payload slot out of range (LENGTH is 12 bits incl. FCS)");
        const uint32_t ns = tx11a_nsym(c.ft.lenh[i], job.ndbps, job.ndbps_pad);
        if (lead_samples + tx11a_samples(ns) > out_stride_samples) return h->fail(SB200_E_INVALID, "out_stride_samples too small for the frame");
        if (ns > max_nsym) max_nsym = ns;
        return SB200_OK;
    });
    if (rc != SB200_OK) return rc;
    job.max_sym = 1u + max_nsym;
    const uint8_t* d_seed = nullptr; void* d_out;
    CK(c.stage(payload, payload_total));
    if (seeds) CK(to_device(h->txseed, seeds, is_device_ptr(seeds), nframes, c.st, &d_seed));
    CK(c.bind(out, (size_t)nframes * out_stride_samples * (sample_bits / 4u), &d_out, nsamples));
    const unsigned helpers = 8;                          // warps per frame for the preamble and the zero fill
    const dim3 grid(nframes, (job.max_sym + helpers + SB_TX_WARPS - 1) / SB_TX_WARPS);
    CK(c.start(true));
    k_tx11a<<<grid, 32 * SB_TX_WARPS, 0, c.st>>>(c.d_pay, c.d_off, c.d_len, d_seed, nframes, job, h->T, h->X, h->inv_deint, c.d_crc, d_out, out_stride_samples, c.d_ns);
    return c.finish(1);
}

// 802.11b transmit (tx11b_kernels.cuh)
extern "C" int sb200_tx11b_batch(sb200_handle* h, const uint8_t* payload, uint64_t payload_total, const uint64_t* pay_off, const uint32_t* pay_len,
                                 uint32_t nframes, uint32_t rate_kbps, uint32_t init_phase, uint32_t lead_samples, uint32_t sample_bits, void* out,
                                 uint64_t out_stride_samples, uint32_t* nsamples, uint32_t* final_phase, void* cuda_stream) {
    int rc = check_null(h, payload, pay_off, pay_len, out);
    if (rc == SB200_OK) rc = check_out(h, sample_bits, out, out_stride_samples);
    if (rc != SB200_OK || nframes == 0) return rc;
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
    TxCall c(h, cuda_stream, pay_off, pay_len, nframes);
    uint32_t max_len = 0;
    if ((rc = c.begin(payload)) != SB200_OK) return rc;
    rc = c.load(payload_total, [&](uint32_t i, bool inside) {
        const uint32_t len = c.ft.lenh[i];
        if (len > 4091u || !inside) return h->fail(SB200_E_INVALID, "payload slot out of range (frame_length 1..4095 incl. FCS)");
        if ((uint64_t)lead_samples + tx11b_nsamples(tx11b_nchips(len, job.chips_per_byte)) > out_stride_samples) return h->fail(SB200_E_INVALID, "out_stride_samples too small for the frame");
        if (len > max_len) max_len = len;
        return SB200_OK;
    });
    if (rc != SB200_OK) return rc;
    job.desc_stride = (24u + max_len + 4u + 7u) & ~7u;
    void* d_out; uint32_t* d_fp;
    CK(c.stage(payload, payload_total));
    CK(c.bind(out, (size_t)nframes * out_stride_samples * (sample_bits / 4u), &d_out, nsamples));
    CK(c.ret.bind(h->txseed, final_phase, nframes * 4ull, &d_fp));
    const uint64_t per_cta = (uint64_t)SB_TX11B_THREADS * SB_TX11B_SPT, ny = (out_stride_samples + per_cta - 1) / per_cta;
    if (ny > 65535u || (uint64_t)lead_samples + out_stride_samples >= (1ull << 27)) return h->fail(SB200_E_INVALID, "out_stride_samples too large");
    CK(c.start(true, (size_t)nframes * job.desc_stride * 2ull));
    const uint16_t* dd = (const uint16_t*)h->txdesc.p; const dim3 grid(nframes, (unsigned)ny);
    k_tx11b_code<<<(nframes + 127) / 128, 128, 0, c.st>>>(c.d_pay, c.d_off, c.d_len, nframes, job, c.d_crc, (uint16_t*)h->txdesc.p, d_fp);
    with_index<4>((uint32_t)(R - kRates11b), [&](auto r) { with_index<2>(lead_samples % 4u == 0, [&](auto al) {
        k_tx11b_shape<decltype(al)::value == 1, kRates11b[decltype(r)::value].kbps><<<grid, SB_TX11B_THREADS, 0, c.st>>>(c.d_len, job, dd, d_out, out_stride_samples, c.d_ns);
    }); });
    return c.finish(2);
}

// Legacy 802.11b transmit filter (tx11b_legacy_kernels.cuh): BB11BPMDSpreadFIR4SSE (variant 0) / BB11BPMDSpreadFIR4ASM (variant 1), batched.
extern "C" int sb200_tx11b_fir37(sb200_handle* h, const int8_t* chips, uint64_t chips_total, const uint64_t* frame_off, const uint32_t* frame_len,
                                 uint32_t nframes, uint32_t variant, int8_t* out, void* cuda_stream) {
    int rc = check_null(h, chips, frame_off, frame_len, out);
    if (rc == SB200_OK && variant > 1) rc = h->fail(SB200_E_INVALID, "variant must be 0 (BB11BPMDSpreadFIR4SSE) or 1 (BB11BPMDSpreadFIR4ASM)");
    if (rc != SB200_OK || nframes == 0) return rc;
    TxCall c(h, cuda_stream, frame_off, frame_len, nframes);
    uint32_t max_len = 0;
    if ((rc = c.begin(chips)) != SB200_OK) return rc;
    const bool in_dev = is_device_ptr(chips), out_dev = is_device_ptr(out);
    rc = c.load(chips_total, [&](uint32_t i, bool inside) {
        if ((c.ft.lenh[i] & 7u) || (c.ft.offh[i] & 7u)) return h->fail(SB200_E_INVALID, "frame_off and frame_len must be multiples of 8 samples (the reference fails on uiInputSize & 7 and needs 16-byte aligned buffers)");
        if (!inside) return h->fail(SB200_E_INVALID, "frame exceeds chips_total");
        if (c.ft.lenh[i] > max_len) max_len = c.ft.lenh[i];
        return SB200_OK;
    });
    if (rc != SB200_OK) return rc;
    if ((in_dev && ((uintptr_t)chips & 15u)) || (out_dev && ((uintptr_t)out & 15u))) return h->fail(SB200_E_INVALID, "device buffers must be 16-byte aligned");
    const int8_t* d_in; int8_t* d_out = out;
    CK(to_device(h->txpay, chips, in_dev, chips_total * 2ull, c.st, &d_in, 16));
    if (!out_dev) { CK(h->txout.need(chips_total * 2ull + 16)); d_out = (int8_t*)h->txout.p; }
    CK(c.ft.upload(h->txoff, h->txlen, c.st, &c.d_off, &c.d_len));
    const uint64_t groups = (uint64_t)(max_len >> 3) * 2u; uint64_t ny = (groups + SB_FIR37_THREADS - 1) / SB_FIR37_THREADS; if (ny > 4096) ny = 4096; if (ny == 0) ny = 1;
    CK(c.start(false));
    with_index<2>(variant, [&](auto v) { k_fir37_legacy<decltype(v)::value><<<dim3(nframes, (unsigned)ny), SB_FIR37_THREADS, 0, c.st>>>(d_in, c.d_off, c.d_len, nframes, d_out); });
    const int frc = c.finish(1);                        // nothing bound: only the frames' own ranges are defined, copied back one by one below (they may be sparse in the buffer)
    if (frc != SB200_OK || out_dev) return frc;
    for (uint32_t i = 0; i < nframes; i++) if (c.ft.lenh[i]) CK(cudaMemcpyAsync(out + 2ull * c.ft.offh[i], d_out + 2ull * c.ft.offh[i], 2ull * c.ft.lenh[i], cudaMemcpyDeviceToHost, c.st));
    CK(cudaStreamSynchronize(c.st));
    return SB200_OK;
}

// Legacy 802.11b transmitter (tx11b_legacy_kernels.cuh): BB11BPMDBufferTx4XWith{Long,Short}Header, optionally followed by the 37-tap filter.
extern "C" int sb200_tx11b_legacy_batch(sb200_handle* h, const uint8_t* payload, uint64_t payload_total, const uint64_t* pay_off, const uint32_t* pay_len,
                                        uint32_t nframes, uint32_t rate_kbps, uint32_t short_preamble, uint32_t flags, uint32_t filter, int8_t* out,
                                        uint64_t out_stride_samples, uint32_t* nsamples, void* cuda_stream) {
    int rc = check_null(h, payload, pay_off, pay_len, out);
    if (rc != SB200_OK) return rc;
    if (flags & SB200_TX11B_LEGACY_PBCC) return h->fail(SB200_E_INVALID, "PBCC is not supported: the reference only lengthens PLCPGetLength for it and still sends CCK");
    if (flags & ~SB200_TX11B_LEGACY_FCS_IN_PAYLOAD) return h->fail(SB200_E_INVALID, "unknown flags");
    if (filter > 2) return h->fail(SB200_E_INVALID, "filter must be 0 (encoder output), 1 (BB11BPMDSpreadFIR4SSE) or 2 (BB11BPMDSpreadFIR4ASM)");
    if (short_preamble > 1) return h->fail(SB200_E_INVALID, "short_preamble must be 0 or 1");
    if ((rc = check_out(h, 8, out, out_stride_samples)) != SB200_OK || nframes == 0) return rc;
    Tx11bLegacyJob job{};
    job.rate_kbps = rate_kbps; job.short_preamble = short_preamble; job.fcs_in_payload = (flags & SB200_TX11B_LEGACY_FCS_IN_PAYLOAD) ? 1u : 0u; job.filter = filter;
    const Rate11b* R = find_rate(kRates11b, rate_kbps);
    if (!R) return h->fail(SB200_E_INVALID, "rate_kbps is not an 802.11b rate");
    job.rate_code = R->code; job.data_chips_per_byte = tx11b_legacy_data_chips(*R, short_preamble);
    TxCall c(h, cuda_stream, pay_off, pay_len, nframes);
    uint32_t max_size = 0;
    if ((rc = c.begin(payload)) != SB200_OK) return rc;
    rc = c.load(payload_total, [&](uint32_t i, bool inside) {
        const uint32_t len = c.ft.lenh[i], size = job.fcs_in_payload ? len : len + 4u;    // PSDU bytes, FCS included
        if (job.fcs_in_payload && len < 4u) return h->fail(SB200_E_INVALID, "with SB200_TX11B_LEGACY_FCS_IN_PAYLOAD every payload carries its 4 FCS bytes");
        if (len > 4095u || size > 4095u || !inside) return h->fail(SB200_E_INVALID, "payload slot out of range (PSDU 4 .. 4095 bytes incl. FCS)");
        if (tx11b_legacy_nsamples(size, short_preamble, job.data_chips_per_byte) > out_stride_samples) return h->fail(SB200_E_INVALID, "out_stride_samples too small for the frame");
        if (size > max_size) max_size = size;
        return SB200_OK;
    });
    if (rc != SB200_OK) return rc;
    job.desc_stride = (24u + max_size + 7u) & ~7u;
    int8_t* d_out;
    CK(c.stage(payload, payload_total));
    CK(c.bind(out, (size_t)nframes * out_stride_samples * 2, &d_out, nsamples));
    const uint64_t per_cta = SB_TX11B_LEGACY_THREADS * 8, ny = (out_stride_samples + per_cta - 1) / per_cta;
    if (ny > 65535u) return h->fail(SB200_E_INVALID, "out_stride_samples too large");
    CK(c.start(!job.fcs_in_payload, (size_t)nframes * job.desc_stride * 2ull));
    const uint16_t* dd = (const uint16_t*)h->txdesc.p;
    k_tx11b_legacy_code<<<(nframes + 127) / 128, 128, 0, c.st>>>(c.d_pay, c.d_off, c.d_len, nframes, job, c.d_crc, (uint16_t*)h->txdesc.p);
    with_index<3>(filter, [&](auto f) {
        k_tx11b_legacy_spread<decltype(f)::value><<<dim3(nframes, (unsigned)ny), SB_TX11B_LEGACY_THREADS, 0, c.st>>>(c.d_len, job, dd, d_out, out_stride_samples, c.d_ns);
    });
    return c.finish(2);
}

// Legacy 802.11a transmitter (tx11a_legacy_kernels.cuh): BB11ATxFrameMod / BB11ATxBufferMod6M at SampleRate 40 or 44.
extern "C" int sb200_tx11a_legacy_batch(sb200_handle* h, const uint8_t* payload, uint64_t payload_total, const uint64_t* pay_off, const uint32_t* pay_len,
                                        uint32_t nframes, uint32_t rate_kbps, uint32_t sample_rate_mhz, uint32_t flags, const int16_t* preamble, int8_t* out,
                                        uint64_t out_stride_samples, uint32_t* nsamples, void* cuda_stream) {
    int rc = check_null(h, payload, pay_off, pay_len, out, preamble);
    if (rc != SB200_OK) return rc;
    if (flags & ~SB200_TX11A_LEGACY_FCS_IN_PAYLOAD) return h->fail(SB200_E_INVALID, "unknown flags");
    if (sample_rate_mhz != 40 && sample_rate_mhz != 44) return h->fail(SB200_E_INVALID, "sample_rate_mhz must be 40 or 44");
    if ((rc = check_out(h, 8, out, out_stride_samples)) != SB200_OK || nframes == 0) return rc;
    const Rate11a* R = find_rate(kRates11a, rate_kbps);
    if (!R) return h->fail(SB200_E_INVALID, "rate_kbps is not an 802.11a rate");
    Tx11aLegacyJob job{};
    job.rate_code = R->code; job.nbpsc = R->nbpsc; job.code_rate = R->cr; job.ndbps = R->ndbps;
    job.sr44 = sample_rate_mhz == 44; job.fcs_in_payload = (flags & SB200_TX11A_LEGACY_FCS_IN_PAYLOAD) ? 1u : 0u;
    TxCall c(h, cuda_stream, pay_off, pay_len, nframes);
    uint32_t max_nsym = 0;
    if ((rc = c.begin(payload, preamble)) != SB200_OK || (rc = upload_tables_tx(h)) != SB200_OK) return rc;
    rc = c.load(payload_total, [&](uint32_t i, bool inside) {
        const uint32_t len = c.ft.lenh[i], size = job.fcs_in_payload ? len : len + 4u;    // PSDU bytes, FCS included
        if (job.fcs_in_payload && len < 4u) return h->fail(SB200_E_INVALID, "with SB200_TX11A_LEGACY_FCS_IN_PAYLOAD every payload carries its 4 FCS bytes");
        if (len > 4096u || size > 4096u || !inside) return h->fail(SB200_E_INVALID, "payload slot out of range (MPDU + FCS at most 4096 bytes)");
        const uint32_t ns = tx11a_legacy_nsym(size, job.ndbps);
        if (tx11a_legacy_padded(ns, job.sr44) > out_stride_samples) return h->fail(SB200_E_INVALID, "out_stride_samples too small for the frame");
        if (ns > max_nsym) max_nsym = ns;
        return SB200_OK;
    });
    if (rc != SB200_OK) return rc;
    job.runs = (1u + max_nsym + SB_TXL_RUN - 1u) / SB_TXL_RUN;
    const uint32_t* d_pre; int8_t* d_out; const bool pre_dev = is_device_ptr(preamble);
    CK(c.stage(payload, payload_total, 1));
    if (pre_dev && ((uintptr_t)preamble & 3u) == 0) d_pre = (const uint32_t*)preamble;
    else { CK(h->txpre.need(640 * 4)); CK(cudaMemcpyAsync(h->txpre.p, preamble, 640 * 4, pre_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, c.st)); d_pre = (const uint32_t*)h->txpre.p; }
    CK(c.bind(out, (size_t)nframes * out_stride_samples * 2, &d_out, nsamples));
    const unsigned helpers = 4;                          // warps per frame for the preamble and the zero fill
    const uint64_t ny = (job.runs + helpers + SB_TXL_WARPS - 1) / SB_TXL_WARPS;
    if (ny > 65535u) return h->fail(SB200_E_INVALID, "too many symbols per frame");
    CK(c.start(!job.fcs_in_payload));
    k_tx11a_legacy<<<dim3(nframes, (unsigned)ny), 32 * SB_TXL_WARPS, 0, c.st>>>(c.d_pay, c.d_off, c.d_len, nframes, job, h->T, h->X, h->inv_deint, c.d_crc, d_pre, d_out, out_stride_samples, c.d_ns);
    return c.finish(1);
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
    int rc = check_null(h, payload, pay_off, pay_len, out0, out1);
    if (rc != SB200_OK || nframes == 0) return rc;
    const Mcs11n* M = find_rate(kMcs11n, mcs, &Mcs11n::mcs);
    if (!M) return h->fail(SB200_E_INVALID, "mcs must be 8 .. 14");
    Tx11nJob job = tx11n_job(*M, lead_samples);
    TxCall c(h, cuda_stream, pay_off, pay_len, nframes);
    uint32_t max_nsym = 0;
    if ((rc = c.begin(payload, seeds)) != SB200_OK || (rc = upload_tables_tx(h)) != SB200_OK || (rc = upload_tables_tx11n(h)) != SB200_OK) return rc;
    if (is_device_ptr(out0) != is_device_ptr(out1)) return h->fail(SB200_E_INVALID, "both output buffers must live on the same side");
    rc = c.load(payload_total, [&](uint32_t i, bool inside) {
        if (c.ft.lenh[i] > 4091u || !inside) return h->fail(SB200_E_INVALID, "payload slot out of range");
        const uint32_t ns = tx11n_nsym_emitted(c.ft.lenh[i], job, nullptr, nullptr);
        if (lead_samples + tx11n_samples(ns) > out_stride_samples) return h->fail(SB200_E_INVALID, "out_stride_samples too small for the frame");
        if (ns > max_nsym) max_nsym = ns;
        return SB200_OK;
    });
    if (rc != SB200_OK) return rc;
    job.max_sym = 3u + max_nsym;
    const uint8_t* d_seed = nullptr; int16_t* d_o0; int16_t* d_o1; const size_t out_bytes = (size_t)nframes * out_stride_samples * 4;
    CK(c.stage(payload, payload_total));
    if (seeds) CK(to_device(h->txseed, seeds, is_device_ptr(seeds), nframes, c.st, &d_seed));
    CK(c.bind(out0, out_bytes, &d_o0, nsamples));
    CK(c.ret.bind(h->txout1, out1, out_bytes, &d_o1));
    const unsigned helpers = 8;
    const dim3 grid(nframes, (2u * job.max_sym + helpers + SB_TX11N_WARPS - 1) / SB_TX11N_WARPS);
    CK(c.start(true));
    k_tx11n<<<grid, 32 * SB_TX11N_WARPS, 0, c.st>>>(c.d_pay, c.d_off, c.d_len, d_seed, nframes, job, h->T, h->X, h->XN, h->inv_deint, c.d_crc, (uint32_t*)d_o0, (uint32_t*)d_o1, out_stride_samples, c.d_ns);
    return c.finish(1);
}
