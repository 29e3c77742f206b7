// sora_b200 — 802.11b receive (rx11b_kernels.cuh): batch slots and continuous captures.
#include "handle.cuh"
#include "rx11b_kernels.cuh"

static int rx11b_run(sb200_handle* h, const int16_t* iq, uint64_t iq_total, const uint64_t* frame_off, const uint32_t* frame_len,
                     uint32_t nframes, uint32_t max_frames, uint8_t* out_bytes, uint32_t out_stride, sb200_frame_result_11b* res, uint32_t* counts, void* cuda_stream) {
    static_assert(sizeof(sb200_frame_result_11b) == sizeof(Result11b), "result layout");
    if (!h || !iq || !frame_off || !frame_len || !res) return h ? h->fail(SB200_E_INVALID, "null argument") : SB200_E_INVALID;
    if (max_frames == 0) return h->fail(SB200_E_INVALID, "max_frames must be at least 1");
    if (nframes == 0) return SB200_OK;
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin()); call.reads(iq);
    const bool iq_dev = is_device_ptr(iq);
    const uint32_t* d_iq; const uint64_t* d_off; const uint32_t* d_len; uint32_t max_len = 0; bool tab_on_host = false;
    { int rc = slot_table(h, frame_off, frame_len, nframes, iq_total, false, st, &d_off, &d_len, &max_len, &tab_on_host); if (rc != SB200_OK) return rc; }
    CK(to_device(h->iq, (const uint32_t*)iq, iq_dev, iq_total * 4ull, st, &d_iq));
    const uint64_t row = 4096; const size_t nres = (size_t)nframes * max_frames;
    CK(h->out.need(nres * row));
    Returns ret; Result11b* d_res; uint32_t* d_cnt;
    if (out_bytes && out_stride) ret.bind2d(out_bytes, out_stride, h->out.p, row, out_stride < row ? out_stride : row, nres);
    CK(ret.bind(h->res, (Result11b*)res, nres * sizeof(Result11b), &d_res));
    CK(ret.bind(h->txns, counts, nframes * 4ull, &d_cnt));
    if (max_frames > 1) CK(cudaMemsetAsync(d_res, 0, nres * sizeof(Result11b), st));          // entries past the count read "no event"
    CK(cudaEventRecord(h->ev0, st));
    k_rx11b<<<(nframes + 63) / 64, 64, 0, st>>>(d_iq, d_off, d_len, nframes, h->cca_thr, (uint8_t*)h->out.p, row, d_res, max_frames, d_cnt);
    return finish_call(h, st, ret, 0, 1);
}

extern "C" int sb200_rx11b_batch(sb200_handle* h, const int16_t* iq, uint64_t iq_total, const uint64_t* frame_off, const uint32_t* frame_len,
                                 uint32_t nframes, uint8_t* out_bytes, uint32_t out_stride, sb200_frame_result_11b* res, void* cuda_stream) {
    return rx11b_run(h, iq, iq_total, frame_off, frame_len, nframes, 1, out_bytes, out_stride, res, nullptr, cuda_stream);
}

extern "C" int sb200_rx11b_streams(sb200_handle* h, const int16_t* iq, uint64_t iq_total, const uint64_t* stream_off, const uint32_t* stream_len,
                                   uint32_t nstreams, uint32_t max_frames, uint8_t* out_bytes, uint32_t out_stride, sb200_frame_result_11b* res,
                                   uint32_t* nframes_out, void* cuda_stream) {
    return rx11b_run(h, iq, iq_total, stream_off, stream_len, nstreams, max_frames, out_bytes, out_stride, res, nframes_out, cuda_stream);
}
