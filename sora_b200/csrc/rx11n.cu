// sora_b200 — 802.11n 2x2 receive (rx11n_kernels.cuh): its tables, the batch pipeline, continuous captures and the stage taps.
#include "handle.cuh"
#include "rx11n_kernels.cuh"
#include <new>
#include <memory>

// ---- 802.11n 2x2 ----------------------------------------------------------------------------------------------------------
static int upload_tables11n(sb200_handle* h) {
    if (h->tab11n.p) return SB200_OK;
    std::unique_ptr<HostTables11n> H(new (std::nothrow) HostTables11n());
    if (!H) return h->fail(SB200_E_NOMEM, "host tables 11n");
    build_host_tables11n(*H);
    TableArena ar;
    const size_t o_sc = ar.add(H->sincos, sizeof H->sincos), o_at = ar.add(H->atan_lut, sizeof H->atan_lut), o_dm = ar.add(H->demap, 256), o_c8 = ar.add(H->crc8, 256),
                 o_pos = ar.add(H->pos, sizeof H->pos), o_l = ar.add(H->lltf_pos, 64), o_ht = ar.add(H->htltf_pos, 64), o_p16 = ar.add(H->pos16, sizeof H->pos16),
                 o_d16 = ar.add(H->demap16, sizeof H->demap16), o_d64 = ar.add(H->demap64, sizeof H->demap64);
    const int rc = ar.upload(h, h->tab11n, "cudaMalloc tables 11n", "table upload 11n");
    if (rc != SB200_OK) return rc;
    const char* base = (const char*)h->tab11n.p;
    DevTables11n& N = h->N;
    N.sincos = (const uint32_t*)(base + o_sc); N.atan_lut = (const int16_t*)(base + o_at); N.demap = (const uint8_t*)(base + o_dm); N.crc8 = (const uint8_t*)(base + o_c8);
    N.pos = (const uint8_t*)(base + o_pos); N.lltf_pos = (const uint8_t*)(base + o_l); N.htltf_pos = (const uint8_t*)(base + o_ht);
    N.pos16 = (const uint16_t*)(base + o_p16); N.demap16 = (const uint8_t*)(base + o_d16); N.demap64 = (const uint8_t*)(base + o_d64);
    return SB200_OK;
}

__global__ void k_pack_results11n(const FrameInfo* __restrict__ info, const uint32_t* __restrict__ status, const uint32_t* __restrict__ crc, uint32_t n,
                                  bool keep_unparsed, sb200_frame_result_11n* __restrict__ res) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    FrameInfo fi = info[i];
    sb200_frame_result_11n r;
    const bool decoded = fi.status == E_SUCCESS;
    r.status = decoded ? status[i] : fi.status; r.mcs = fi.rate_kbps == MCS11N_UNPARSED && !keep_unparsed ? 0u : fi.rate_kbps; r.length = fi.length; r.crc32 = decoded ? crc[i] : 0u; r.nsym = fi.nsym_total;
    r.detect_index = fi.detect_vec == 0xFFFFFFFFu ? 0u : fi.detect_vec * 4u;
    r.cfo_est = (int16_t)fi.cfo_est; r.lsig_length = (uint16_t)fi.peak_index;
    res[i] = r;
}

static int rx11n_run(sb200_handle* h, const int16_t* iq0, const int16_t* iq1, uint64_t iq_total, const uint64_t* frame_off, const uint32_t* frame_len,
                     uint32_t nframes, uint8_t* out_bytes, uint32_t out_stride, sb200_frame_result_11n* res, cudaStream_t st, Taps11n taps,
                     uint8_t* soft_host, uint64_t soft_host_stride, const uint32_t* state_idx = nullptr /* host: carrier-sense state slot per capture (stream mode) */) {
    if (!h || !iq0 || !iq1 || !frame_off || !frame_len || !res) return h ? h->fail(SB200_E_INVALID, "null argument") : SB200_E_INVALID;
    if (nframes == 0) return SB200_OK;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin()); call.reads(iq0); call.reads(iq1);
    int rc = upload_tables11n(h); if (rc != SB200_OK) return rc;
    const bool iq_dev = is_device_ptr(iq0);
    if (iq_dev != is_device_ptr(iq1)) return h->fail(SB200_E_INVALID, "both antenna buffers must live on the same side");
    const uint64_t* d_off; const uint32_t* d_len; uint32_t max_len = 0; bool tab_on_host = false;
    { int rc = slot_table(h, frame_off, frame_len, nframes, iq_total, false, st, &d_off, &d_len, &max_len, &tab_on_host); if (rc != SB200_OK) return rc; }
    const uint32_t* d_iq0; const uint32_t* d_iq1;
    CK(to_device(h->iq, (const uint32_t*)iq0, iq_dev, iq_total * 4ull, st, &d_iq0));
    CK(to_device(h->iq1, (const uint32_t*)iq1, iq_dev, iq_total * 4ull, st, &d_iq1));
    const uint64_t max_sym = (max_len / 2u) / 80u + 1u;
    h->N.mcs_limit = h->ht_mcs_limit;
    const uint64_t soft_stride = ((max_sym * (h->ht_mcs_limit > 11u ? 624ull : 208ull)) + 15ull) & ~15ull;   // 2 x 52 x N_BPSC soft values per symbol
    const uint64_t row = 1536;                         // >= 1500 (MTU, PHY_11n.hpp:478,505)
    CK(h->info.need(nframes * sizeof(FrameInfo))); CK(h->soft.need(nframes * soft_stride)); CK(h->out.need(nframes * row));
    CK(h->status.need(nframes * 4ull)); CK(h->crc.need(nframes * 4ull));
    Returns ret; sb200_frame_result_11n* d_res;
    if (out_bytes && out_stride) ret.bind2d(out_bytes, out_stride, h->out.p, row, out_stride < row ? out_stride : row, nframes);
    CK(ret.bind(h->res, res, nframes * sizeof(sb200_frame_result_11n), &d_res));
    if (soft_host) ret.bind2d(soft_host, soft_host_stride, h->soft.p, soft_stride, soft_host_stride < soft_stride ? soft_host_stride : soft_stride, nframes);
    FrameInfo* d_info = (FrameInfo*)h->info.p;
    CK(cudaEventRecord(h->ev0, st)); CK(cudaEventRecord(h->evk[0], st));
    if (state_idx) {
        const uint32_t* d_idx; CK(to_device(h->ccaidx, state_idx, false, nframes * 4ull, st, &d_idx));
        k_sync11n_stream<<<(nframes + 63) / 64, 64, 0, st>>>(d_iq0, d_iq1, d_off, d_len, nframes, d_idx, (Cca11nState*)h->cca11n.p, d_info);
    } else
    k_sync11n<<<(nframes + 127) / 128, 128, 0, st>>>(d_iq0, d_iq1, d_off, d_len, nframes, d_info);
    CK(cudaEventRecord(h->evk[1], st));
    k_front11n<<<(nframes + SB_FRONT11N_WARPS - 1) / SB_FRONT11N_WARPS, 32 * SB_FRONT11N_WARPS, 0, st>>>(d_iq0, d_iq1, d_off, d_len, nframes, h->T, h->N, h->inv_deint,
            d_info, (uint8_t*)h->soft.p, soft_stride, taps);
    CK(cudaEventRecord(h->evk[2], st));
    VitJob job{}; job.depth = 192; job.lookahead = 36; job.raw = 0;                    // T11aViterbi<5000*8, 312, 192, 36> (fb11ndemod_config.hpp:189)
    static const int rates[3] = {CR_12, CR_34, CR_23};  // CR_23: MCS 13, refused unless ht_mcs_limit > 13
    const bool cr23 = h->ht_mcs_limit > 13u;
    rc = viterbi_stage(h, nframes, st, (const uint8_t*)h->soft.p, soft_stride, d_info, job, (uint8_t*)h->out.p, row, (uint32_t*)h->status.p, (uint32_t*)h->crc.p, rates, cr23 ? 3 : 2);
    if (rc != SB200_OK) return rc;
    CK(cudaEventRecord(h->evk[3], st));
    k_pack_results11n<<<(nframes + 255) / 256, 256, 0, st>>>(d_info, (const uint32_t*)h->status.p, (const uint32_t*)h->crc.p, nframes, state_idx != nullptr, d_res);
    CK(cudaEventRecord(h->evk[4], st));
    return finish_call(h, st, ret, 4, 3);
}

// Continuous two-antenna captures: every pass decodes the next frame of all captures that still have samples (the batch pipeline over the
// rest of each capture), with TCCA11n / MimoAutoCorr's never-reset state kept per capture on the device (k_sync11n_stream).
extern "C" int sb200_rx11n_streams(sb200_handle* h, const int16_t* iq0, const int16_t* iq1, uint64_t iq_total, const uint64_t* stream_off, const uint32_t* stream_len,
                                   uint32_t nstreams, uint32_t max_frames, uint8_t* out_bytes, uint32_t out_stride, sb200_frame_result_11n* res,
                                   uint32_t* sample_index, uint32_t* nframes_out, void* cuda_stream) {
    if (!h || !iq0 || !iq1 || !stream_off || !stream_len || !res || !nframes_out) return h ? h->fail(SB200_E_INVALID, "null argument") : SB200_E_INVALID;
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin());          // results in host memory: the call synchronises anyway
    const bool iq_dev = is_device_ptr(iq0);
    {   const int rc = stream_table(h, stream_off, stream_len, nstreams, iq_total, res, out_bytes, nframes_out, iq_dev != is_device_ptr(iq1)); if (rc != SB200_OK) return rc; }
    if (nstreams == 0 || max_frames == 0) return SB200_OK;
    const int16_t* d_iq0; const int16_t* d_iq1;
    CK(to_device(h->iq, iq0, iq_dev, iq_total * 4ull, st, &d_iq0));
    CK(to_device(h->iq1, iq1, iq_dev, iq_total * 4ull, st, &d_iq1));
    CK(h->cca11n.need((size_t)nstreams * sizeof(Cca11nState))); CK(cudaMemsetAsync(h->cca11n.p, 0, (size_t)nstreams * sizeof(Cca11nState), st));   // TCCA11n / MimoAutoCorr constructors
    std::vector<uint64_t> pos(nstreams, 0);
    std::vector<uint32_t> last_mcs(nstreams, 0);      // CF_HTRxVector::ht_frame_mcs of each capture: never reset between events
    std::vector<uint32_t> active(nstreams); for (uint32_t s = 0; s < nstreams; s++) active[s] = s;
    std::vector<uint64_t> off; std::vector<uint32_t> len, idx; std::vector<sb200_frame_result_11n> r; std::vector<uint8_t> bytes;
    const uint32_t row = out_bytes ? (out_stride < 1536u ? out_stride : 1536u) : 0u;
    int rc = SB200_OK;
    while (!active.empty()) {
        std::vector<uint32_t> live;
        for (uint32_t s : active) if (nframes_out[s] < max_frames && pos[s] + 28 <= stream_len[s]) live.push_back(s);
        if (live.empty()) break;
        const uint32_t n = (uint32_t)live.size();
        off.resize(n); len.resize(n); idx.resize(n); r.resize(n); if (row) bytes.resize((size_t)n * row);
        for (uint32_t j = 0; j < n; j++) { const uint32_t s = live[j]; off[j] = stream_off[s] + pos[s]; len[j] = (uint32_t)(stream_len[s] - pos[s]); idx[j] = s; }
        Taps11n taps{}; h->tab_off = nullptr;
        rc = rx11n_run(h, d_iq0, d_iq1, iq_total, off.data(), len.data(), n, row ? bytes.data() : nullptr, row, r.data(), st, taps, nullptr, 0, idx.data());
        if (rc != SB200_OK) break;
        active.clear();
        for (uint32_t j = 0; j < n; j++) {
            const uint32_t s = live[j];
            if (r[j].status == SB200_FRAME_NONE) continue;                               // this capture ran out of samples: RxThread returns
            // symbols that went through the graph behind the 128-sample L-LTF: the three SIG symbols when the header is refused (T11nSigParser
            // runs in the third), else SIG x 3 + HT-STF + HT-LTF x 2 + data = total_symbols + 2 (PHY_11n.hpp:508 counts data + 4)
            const bool whole = r[j].status == SB200_FRAME_OK || r[j].status == SB200_FRAME_CRC32_FAIL || r[j].status == SB200_FRAME_FAILED;
            const uint64_t e20 = (uint64_t)r[j].detect_index + 128ull + 80ull * (whole ? r[j].nsym + 2ull : 3ull);
            const uint64_t v_last = e20 / 4ull - 1ull, blk = (8ull * v_last + 7ull) / 28ull;
            pos[s] += (blk + 1ull) * 28ull;                                                   // the driver sees the event after that source block
            const size_t slot = (size_t)s * max_frames + nframes_out[s];
            if (r[j].mcs == MCS11N_UNPARSED) r[j].mcs = last_mcs[s];
            last_mcs[s] = r[j].mcs;
            res[slot] = r[j];
            if (sample_index) sample_index[slot] = (uint32_t)pos[s];
            if (row) memcpy(out_bytes + slot * out_stride, bytes.data() + (size_t)j * row, row);
            nframes_out[s]++;
            active.push_back(s);
        }
    }
    return rc;
}

extern "C" int sb200_rx11n_batch(sb200_handle* h, const int16_t* iq0, const int16_t* iq1, uint64_t iq_total_samples, const uint64_t* frame_off,
                                 const uint32_t* frame_len, uint32_t nframes, uint8_t* out_bytes, uint32_t out_stride, sb200_frame_result_11n* res, void* cuda_stream) {
    Taps11n taps{};
    return rx11n_run(h, iq0, iq1, iq_total_samples, frame_off, frame_len, nframes, out_bytes, out_stride, res, (cudaStream_t)cuda_stream, taps, nullptr, 0);
}

extern "C" int sb200_rx11n_taps(sb200_handle* h, const int16_t* iq0, const int16_t* iq1, uint64_t iq_total_samples, const uint64_t* frame_off,
                                const uint32_t* frame_len, uint32_t nframes, uint32_t max_sym, sb200_frame_result_11n* res,
                                int16_t* siso, int16_t* hinv, int16_t* eq, int16_t* theta, uint8_t* sig, uint8_t* soft, uint64_t soft_stride) {
    if (!h) return SB200_E_INVALID;
    CK(cudaSetDevice(h->device));
    const size_t b0 = (size_t)nframes * 2 * 64 * 4, b1 = (size_t)nframes * 4 * 64 * 4, b2 = (size_t)nframes * 2 * max_sym * 64 * 4, b3 = (size_t)nframes * max_sym * 2, b4 = (size_t)nframes * 16;
    const size_t size[5] = {b0, b1, b2 + 4, b3 + 4, b4}, back[5] = {b0, b1, b2, b3, b4};
    void* const dst[5] = {siso, hinv, eq, theta, sig};
    return run_with_taps(h, size, dst, back, [&] {
        Taps11n taps{};
        taps.siso = (uint32_t*)h->taps[0].p; taps.hinv = (uint32_t*)h->taps[1].p; taps.eq = (uint32_t*)h->taps[2].p; taps.theta = (int16_t*)h->taps[3].p; taps.sig = (uint8_t*)h->taps[4].p; taps.max_sym = max_sym;
        return rx11n_run(h, iq0, iq1, iq_total_samples, frame_off, frame_len, nframes, nullptr, 0, res, 0, taps, soft, soft_stride);
    });
}
