// sora_b200 — the K=7 Viterbi stage of the receive chains and sb200_viterbi_k7: the four-lane kernel (viterbi_k7_re.cuh) or the lane
// kernel (viterbi_k7_lane.cuh) per launch, with the work lists and the frame sink around them.
#include "handle.cuh"
#include "viterbi_k7_re.cuh"
#include "viterbi_k7_lane.cuh"

// One launch of the Viterbi for code rate CR: the lane kernel (viterbi_k7_lane.cuh) for launches of lane_min .. lane_max code blocks, in
// the rendering the options select (8-column history blocks with the deferred walk unless told otherwise); the others the
// four-lanes-per-code-block kernel.  `smem`: dynamic shared memory of the four-lane kernel (padding, the vq_pad_smem knob).  Each code
// block's count of decoded bytes goes to nraw.  vring_need() sizes the lane kernel's history rings for n code blocks first.
static bool use_lane(const sb200_handle* h, uint32_t n) { return n >= h->lane_min && n <= h->lane_max; }
static cudaError_t vring_need(sb200_handle* h, uint32_t n) {
    if (use_lane(h, n)) return h->vring.need((size_t)((n + SB_VL_FR - 1) / SB_VL_FR) * SB_VL_NB8D * SB_VL_ENTRY * 16);   // the largest ring of the lane kernel's renderings
    return cudaSuccess;                                // the four-lane kernel keeps its ring in shared memory
}
// k_viterbi_re<CR> as persistent CTAs: at most as many as the SMs hold at once with `smem` bytes of dynamic shared memory (the
// occupancy calculator's count, taken once per handle and padding), each taking groups of code blocks from the counter `next`.
template <int CR>
static cudaError_t launch_re(sb200_handle* h, uint32_t n, cudaStream_t s, uint32_t smem, const uint8_t* soft, uint64_t soft_stride, const uint32_t* list,
                             const uint32_t* cnt, const FrameInfo* info, const VitJob& job, uint8_t* out, uint64_t out_stride, uint32_t raw_off,
                             uint32_t* nraw, uint32_t* next) {
    sb200_handle::VrOcc& o = h->vr_occ[CR];
    if (o.ctas == 0 || o.smem != smem) {
        if (!h->sms) { const cudaError_t e = cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, h->device); if (e != cudaSuccess) return e; }
        int per_sm = 0;
        const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_viterbi_re<CR>, 32, smem);
        if (e != cudaSuccess) return e;
        o.ctas = (uint32_t)max(per_sm, 1) * (uint32_t)h->sms; o.smem = smem;
    }
    const uint32_t groups = (n + SB_VR_FR - 1) / SB_VR_FR;
    k_viterbi_re<CR><<<min(groups, o.ctas), 32, smem, s>>>(soft, soft_stride, n, list, cnt, info, job, out, out_stride, raw_off, nraw, next);
    return cudaSuccess;
}
template <int CR>
static cudaError_t launch_viterbi(sb200_handle* h, uint32_t n, cudaStream_t s, const uint8_t* soft, uint64_t soft_stride, const uint32_t* list, const uint32_t* cnt,
                                  const FrameInfo* info, const VitJob& job, uint8_t* out, uint64_t out_stride, uint32_t* nraw, uint32_t smem, uint32_t* next) {
    const uint32_t raw_off = info ? 14u : 0u;          // frames are decoded 14 bytes into their row, raw blocks at its start
    uint4* const ring = (uint4*)h->vring.p;             // the lane kernel's history rings
    h->last_vit = use_lane(h, n) ? "k_viterbi_lane" : "k_viterbi_re";
    if (use_lane(h, n) && h->vl_hb == 8 && h->vl_defer) k_viterbi_lane<CR, 8, true><<<(n + SB_VL_FR - 1) / SB_VL_FR, 32, h->vl_pad_smem, s>>>(soft, soft_stride, n, list, cnt, info, job, out, out_stride, raw_off, nraw, ring, h->vl_flags);
    else if (use_lane(h, n) && h->vl_hb == 8) k_viterbi_lane<CR, 8><<<(n + SB_VL_FR - 1) / SB_VL_FR, 32, h->vl_pad_smem, s>>>(soft, soft_stride, n, list, cnt, info, job, out, out_stride, raw_off, nraw, ring, h->vl_flags);
    else if (use_lane(h, n))         k_viterbi_lane<CR, 6><<<(n + SB_VL_FR - 1) / SB_VL_FR, 32, h->vl_pad_smem, s>>>(soft, soft_stride, n, list, cnt, info, job, out, out_stride, raw_off, nraw, ring, h->vl_flags);
    else                             return launch_re<CR>(h, n, s, smem, soft, soft_stride, list, cnt, info, job, out, out_stride, raw_off, nraw, next);
    return cudaSuccess;
}

// The Viterbi stage: one launch per code rate of `rates`, in that order.  Frames (`info` set) get work lists (vlist from frame `first`, vcnt
// block `slot`: the counts, then the group counters of k_viterbi_re's three code rates) and k_sink11a; raw code blocks (`info` null) only
// the counters.  `smem34`: the 802.11a vq_pad_smem knob.
int viterbi_stage(sb200_handle* h, uint32_t n, cudaStream_t s, const uint8_t* soft, uint64_t soft_stride, const FrameInfo* info, const VitJob& job,
                  uint8_t* out, uint64_t out_stride, uint32_t* status, uint32_t* crc, const int* rates, uint32_t nrates,
                  uint32_t first, uint32_t slot, uint32_t smem34) {
    const uint32_t* list = nullptr; const uint32_t* cnt = nullptr;
    CK(vring_need(h, n));
    CK(h->vcnt.need(32ull * (slot + 1u)));
    uint32_t* d_cnt = (uint32_t*)h->vcnt.p + 8 * (size_t)slot;
    CK(cudaMemsetAsync(d_cnt, 0, 32, s));
    uint32_t* const next = d_cnt + 4;
    if (info) {
        CK(h->vlist.need((first + (size_t)n) * 12ull));
        uint32_t* d_list = (uint32_t*)h->vlist.p + 3 * (size_t)first;
        k_vit_lists<<<(n + 255) / 256, 256, 0, s>>>(info, n, d_cnt, d_list);
        list = d_list; cnt = d_cnt; h->launches += 1;
    }
    for (uint32_t r = 0; r < nrates; r++) {
        const int cr = rates[r];
        if (cr == CR_34) CK(launch_viterbi<CR_34>(h, n, s, soft, soft_stride, list, cnt, info, job, out, out_stride, status, smem34, next + CR_34));
        else if (cr == CR_12) CK(launch_viterbi<CR_12>(h, n, s, soft, soft_stride, list, cnt, info, job, out, out_stride, status, 0, next + CR_12));
        else CK(launch_viterbi<CR_23>(h, n, s, soft, soft_stride, list, cnt, info, job, out, out_stride, status, 0, next + CR_23));
    }
    h->launches += nrates;
    if (info) { k_sink11a<<<(n + 127) / 128, 128, 0, s>>>(out, out_stride, n, info, h->T, status, crc); h->launches += 1; }
    return SB200_OK;
}

extern "C" int sb200_viterbi_k7(sb200_handle* h, const uint8_t* soft, uint64_t soft_stride, uint32_t nsoft, uint32_t nblocks,
                                int code_rate, uint32_t frame_len_bytes, uint32_t depth, uint32_t lookahead,
                                uint8_t* out, uint64_t out_stride, void* cuda_stream) {
    if (!h || !soft || !out) return h ? h->fail(SB200_E_INVALID, "null argument") : SB200_E_INVALID;
    if (code_rate < 0 || code_rate > 2 || depth == 0 || (depth & 7) || depth + lookahead + 8 > 288 || depth > 256)
        return h->fail(SB200_E_INVALID, "unsupported code_rate/depth/lookahead");
    if (soft_stride < nsoft || out_stride < frame_len_bytes + 2ull) return h->fail(SB200_E_INVALID, "stride too small");
    if (nblocks == 0) return SB200_OK;
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin()); call.reads(soft);
    const uint8_t* d_soft; uint64_t d_stride = soft_stride;
    const bool aligned = ((uintptr_t)soft & 15) == 0 && (soft_stride & 15) == 0;
    if (is_device_ptr(soft) && aligned) d_soft = soft;
    else {
        d_stride = ((uint64_t)nsoft + 15ull) & ~15ull;
        CK(h->soft.need(nblocks * d_stride + 16));
        CK(cudaMemcpy2DAsync(h->soft.p, d_stride, soft, soft_stride, nsoft, nblocks, is_device_ptr(soft) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
        d_soft = (const uint8_t*)h->soft.p;
    }
    uint8_t* d_out = out; uint64_t d_ostride = out_stride; Returns ret;
    if (!is_device_ptr(out)) {
        d_ostride = (frame_len_bytes + 2ull + 15ull) & ~15ull; CK(h->out.need(nblocks * d_ostride)); d_out = (uint8_t*)h->out.p;
        ret.bind2d(out, out_stride, d_out, d_ostride, frame_len_bytes + 2ull, nblocks);
    }
    CK(h->status.need(nblocks * 4ull)); CK(h->crc.need(nblocks * 4ull));
    VitJob job{}; job.code_rate = (uint32_t)code_rate; job.frame_len = frame_len_bytes; job.nsoft = nsoft; job.depth = depth; job.lookahead = lookahead; job.raw = 1;
    CK(cudaEventRecord(h->ev0, st));
    const int rc = viterbi_stage(h, nblocks, st, d_soft, d_stride, nullptr, job, d_out, d_ostride, (uint32_t*)h->status.p, (uint32_t*)h->crc.p, &code_rate, 1);
    if (rc != SB200_OK) return rc;
    return finish_call(h, st, ret, 0, 0);
}
