// sora_b200 — host side of the C ABI (include/sora_b200.h): the handle (create, destroy, options, the last call's figures), the base tables,
// slot and capture tables, page-locked host buffers and RX_BLOCK ingest.  Each chain's entry points live in a file of their own: viterbi.cu,
// rx11a.cu, rx11b.cu, rx11n.cu, tx.cu and wideband.cu; handle.cuh holds what they share.
#include "handle.cuh"
#include <new>
#include <memory>

namespace {

// max(len) and an out-of-bounds flag over a device-resident slot table: res[0] = max frame_len, res[1] != 0 if any slot leaves [0, iq_total)
__global__ void k_slot_check(const uint64_t* __restrict__ off, const uint32_t* __restrict__ len, uint32_t n, uint64_t iq_total, uint32_t* __restrict__ res) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t l = 0, bad = 0;
    if (i < n) { l = len[i]; const uint64_t o = off[i]; bad = (l > iq_total || o > iq_total - l) ? 1u : 0u; }
    l = __reduce_max_sync(0xFFFFFFFFu, l); bad = __reduce_or_sync(0xFFFFFFFFu, bad);
    if ((threadIdx.x & 31) == 0) { if (l) atomicMax(res, l); if (bad) atomicOr(res + 1, 1u); }
}

} // namespace

static int upload_tables(sb200_handle* h) {
    std::unique_ptr<HostTables> H(new (std::nothrow) HostTables());
    if (!H) return h->fail(SB200_E_NOMEM, "host tables");
    build_host_tables(*H);
    uint16_t inv[624];
    const int offs[4] = {0, 48, 144, 336}, n[4] = {48, 96, 192, 288};
    for (int m = 0; m < 4; m++) for (int k = 0; k < n[m]; k++) inv[offs[m] + H->deint[offs[m] + k]] = (uint16_t)k;
    std::vector<uint32_t> rot(65536);
    for (int i = 0; i < 65536; i++) rot[i] = pack(mk((int)H->cos_lut[i], -(int)H->sin_lut[i]));
    TableArena ar;
    const size_t o_rot = ar.add(rot.data(), 262144), o_sin = ar.add(H->sin_lut.data(), 131072), o_cos = ar.add(H->cos_lut.data(), 131072),
                 o_at = ar.add(H->atan2_lut.data(), 131072), o_tw64 = ar.add(H->tw64, sizeof H->tw64), o_tw16 = ar.add(H->tw16, sizeof H->tw16),
                 o_sts = ar.add(H->sts, sizeof H->sts), o_deint = ar.add(H->deint, sizeof H->deint), o_inv = ar.add(inv, sizeof inv),
                 o_demap = ar.add(H->demap, sizeof H->demap), o_pil = ar.add(H->pilot_neg, 128), o_lts = ar.add(H->lts_pos, 64),
                 o_scr = ar.add(H->scramble, 128), o_crc = ar.add(H->crc32, 1024);
    const int rc = ar.upload(h, h->tab, "cudaMalloc tables", "table upload");
    if (rc != SB200_OK) return rc;
    const char* base = (const char*)h->tab.p;
    DevTables& T = h->T;
    T.sin_lut = (const int16_t*)(base + o_sin); T.cos_lut = (const int16_t*)(base + o_cos); T.atan2_lut = (const int16_t*)(base + o_at); T.rot = (const uint32_t*)(base + o_rot);
    T.tw64 = (const uint32_t*)(base + o_tw64); T.tw16 = (const uint32_t*)(base + o_tw16); T.sts = (const uint32_t*)(base + o_sts);
    T.deint = (const uint16_t*)(base + o_deint); T.demap = (const uint8_t*)(base + o_demap); T.pilot_neg = (const uint8_t*)(base + o_pil);
    T.lts_pos = (const uint8_t*)(base + o_lts); T.scramble = (const uint8_t*)(base + o_scr); T.crc32 = (const uint32_t*)(base + o_crc);
    h->inv_deint = (uint16_t*)(base + o_inv);
    return SB200_OK;
}

extern "C" int sb200_create(int device, const sb200_cfg* cfg, sb200_handle** out) {
    if (!out) return SB200_E_INVALID;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) { cudaGetLastError(); return SB200_E_NODEVICE; }
    sb200_handle* h = new (std::nothrow) sb200_handle();
    if (!h) return SB200_E_NOMEM;
    h->device = device;
    if (cfg && cfg->cca_pwr_threshold) h->cca_thr = cfg->cca_pwr_threshold;
    if (cudaSetDevice(device) != cudaSuccess) { delete h; return SB200_E_CUDA; }
    int rc = upload_tables(h);
    if (rc == SB200_OK && (cudaEventCreate(&h->ev0) != cudaSuccess || cudaEventCreate(&h->ev1) != cudaSuccess)) rc = SB200_E_CUDA;
    for (int i = 0; i < 5 && rc == SB200_OK; i++) if (cudaEventCreate(&h->evk[i]) != cudaSuccess) rc = SB200_E_CUDA;
    if (rc == SB200_OK && cudaEventCreateWithFlags(&h->ev_done, cudaEventDisableTiming) != cudaSuccess) rc = SB200_E_CUDA;
    if (rc == SB200_OK) rc = host_pipe_create(&h->pipe);
    if (rc != SB200_OK) { sb200_destroy(h); return rc; }
    *out = h;
    return SB200_OK;
}

extern "C" void sb200_destroy(sb200_handle* h) {
    if (!h) return;
    cudaSetDevice(h->device);                          // the workspaces (DevBuf) free themselves in `delete h`
    if (h->ev0) cudaEventDestroy(h->ev0);
    if (h->ev1) cudaEventDestroy(h->ev1);
    for (int i = 0; i < 5; i++) if (h->evk[i]) cudaEventDestroy(h->evk[i]);
    if (h->ev_done) cudaEventDestroy(h->ev_done);
    host_pipe_destroy(h->pipe);
    delete h;
}
extern "C" const char* sb200_last_error(const sb200_handle* h) { return h ? h->err.c_str() : "null handle"; }
extern "C" uint64_t sb200_launch_count(const sb200_handle* h) { return h ? h->launches : 0; }
extern "C" const char* sb200_last_viterbi_kernel(const sb200_handle* h) { return h ? h->last_vit : ""; }
extern "C" float sb200_last_kernel_ms(sb200_handle* h) {
    if (!h || !h->timed) return -1.f;
    float ms = -1.f;
    if (cudaEventSynchronize(h->ev1) != cudaSuccess) return -1.f;
    if (cudaEventElapsedTime(&ms, h->ev0, h->ev1) != cudaSuccess) return -1.f;
    return ms;
}

extern "C" int sb200_last_kernel_times(sb200_handle* h, float* ms4) {
    if (!h || !ms4 || !h->timed || h->nk != 4) return SB200_E_INVALID;
    if (cudaEventSynchronize(h->evk[4]) != cudaSuccess) return SB200_E_CUDA;
    for (int i = 0; i < 4; i++) if (cudaEventElapsedTime(&ms4[i], h->evk[i], h->evk[i + 1]) != cudaSuccess) return SB200_E_CUDA;
    return SB200_OK;
}

// Slot table of a call: bounds-checks every slot against iq_total and returns the largest slot length (workspaces are sized from it).
//   host tables   : checked on the host, copied to the device.
//   device tables : checked on the device (k_slot_check, one 8-byte read-back) on EVERY call; with `need_host_copy` the table is also copied back
//                   (the chunked host-IQ path stages sample ranges per chunk).  Only after set_option("slot_table_immutable", 1) — the caller's
//                   promise not to rewrite a device-resident table between calls — is the result cached by (pointers, count, total).
int slot_table(sb200_handle* h, const uint64_t* frame_off, const uint32_t* frame_len, uint32_t nframes, uint64_t iq_total, bool need_host_copy,
               cudaStream_t st, const uint64_t** d_off, const uint32_t** d_len, uint32_t* max_len, bool* host_valid) {
    const bool off_dev = is_device_ptr(frame_off), len_dev = is_device_ptr(frame_len);
    std::vector<uint64_t>& offh = h->offh; std::vector<uint32_t>& lenh = h->lenh;
    *host_valid = false;
    if (off_dev && len_dev) {
        const bool cached = h->tab_immutable && h->tab_off == frame_off && h->tab_len == frame_len && h->tab_n == nframes && h->tab_total == iq_total && (!need_host_copy || h->tab_host);
        if (!cached) {
            CK(h->slotchk.need(8));
            CK(cudaMemsetAsync(h->slotchk.p, 0, 8, st));
            k_slot_check<<<(nframes + 255) / 256, 256, 0, st>>>(frame_off, frame_len, nframes, iq_total, (uint32_t*)h->slotchk.p);
            uint32_t r[2] = {0, 0};
            CK(cudaMemcpyAsync(r, h->slotchk.p, 8, cudaMemcpyDeviceToHost, st));
            if (need_host_copy) {
                offh.resize(nframes); lenh.resize(nframes);
                CK(cudaMemcpyAsync(offh.data(), frame_off, nframes * 8ull, cudaMemcpyDeviceToHost, st)); CK(cudaMemcpyAsync(lenh.data(), frame_len, nframes * 4ull, cudaMemcpyDeviceToHost, st));
            }
            CK(cudaStreamSynchronize(st));
            h->tab_off = nullptr;
            if (r[1]) return h->fail(SB200_E_INVALID, "slot exceeds iq_total_samples");
            h->tab_max_len = r[0]; h->tab_host = need_host_copy;
            if (h->tab_immutable) { h->tab_off = frame_off; h->tab_len = frame_len; h->tab_n = nframes; h->tab_total = iq_total; }
        }
        *d_off = frame_off; *d_len = frame_len; *max_len = h->tab_max_len; *host_valid = h->tab_host && (cached || need_host_copy);
        return SB200_OK;
    }
    h->tab_off = nullptr;
    CK(read_table(st, frame_off, off_dev, frame_len, len_dev, nframes, offh, lenh));
    uint32_t mx = 0;
    for (uint32_t i = 0; i < nframes; i++) {
        if (!in_range(offh[i], lenh[i], iq_total)) return h->fail(SB200_E_INVALID, "slot exceeds iq_total_samples");
        if (lenh[i] > mx) mx = lenh[i];
    }
    CK(to_device(h->off, off_dev ? frame_off : offh.data(), off_dev, nframes * 8ull, st, d_off));   // host parts: the copy checked above
    CK(to_device(h->len, len_dev ? frame_len : lenh.data(), len_dev, nframes * 4ull, st, d_len));
    *max_len = mx; *host_valid = true;
    return SB200_OK;
}

// Page-locked host memory for capture buffers: what the reference's user-mode extension maps for a radio (SoraURadioMapRxSampleBuf,
// kernel/core/inc/_user_mode_ext.h:100) is DMA-able memory too.  Captures handed to the engine from such a buffer cross PCIe without a staging copy.
extern "C" void* sb200_host_alloc(size_t bytes) { void* p = nullptr; if (bytes == 0 || cudaHostAlloc(&p, bytes, cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return nullptr; } return p; }
extern "C" void sb200_host_free(void* p) { if (p) cudaFreeHost(p); }

// Capture table of a stream call: tables and results in host memory, every capture inside the samples, frame counts zeroed on the way.
int stream_table(sb200_handle* h, const uint64_t* stream_off, const uint32_t* stream_len, uint32_t nstreams, uint64_t iq_total,
                 const void* res, const void* out_bytes, uint32_t* nframes_out, bool antennas_apart) {
    if (is_device_ptr(res) || (out_bytes && is_device_ptr(out_bytes)) || is_device_ptr(stream_off) || is_device_ptr(stream_len) || is_device_ptr(nframes_out))
        return h->fail(SB200_E_INVALID, "stream mode takes its tables and returns its results in host memory");
    if (antennas_apart) return h->fail(SB200_E_INVALID, "both antenna buffers must live on the same side");
    for (uint32_t s = 0; s < nstreams; s++) { nframes_out[s] = 0; if (!in_range(stream_off[s], stream_len[s], iq_total)) return h->fail(SB200_E_INVALID, "capture exceeds iq_total_samples"); }
    return SB200_OK;
}

// ---- RX_BLOCK ingest (SURVEY.md §8(f) rank 3) -------------------------------------------------------------------------------
// A Sora capture (dump file, RX DMA ring) is a sequence of 128-byte RX_BLOCKs: a 16-byte descriptor followed by seven
// 16-byte sample units = 28 COMPLEX16 (kernel/core/inc/_rx_manager.h:79-113); LoadSoraDumpFile (kernel/brick/inc/brickutil.h:21-59)
// strips the descriptors on the CPU.  Here it is a device gather: one thread per 16-byte unit, 128-bit loads and stores, with the
// optional left shift that drops the invalid low bits of legacy 14-bit captures (RX_COMPLEX16_INVALID_BITS, core/inc/const.h:73).
__global__ void __launch_bounds__(256) k_rxblocks_unpack(const uint4* __restrict__ blocks, uint64_t nunits, uint32_t shift, uint4* __restrict__ out) {
    for (uint64_t u = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; u < nunits; u += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t b = u / 7u, j = u - 7u * b;
        uint4 v = __ldg(blocks + b * 8u + 1u + j);
        if (shift) {
            auto sh = [&](uint32_t w) { return (((w & 0xFFFFu) << shift) & 0xFFFFu) | ((w >> 16 << shift) << 16); };
            v.x = sh(v.x); v.y = sh(v.y); v.z = sh(v.z); v.w = sh(v.w);
        }
        out[u] = v;
    }
}
extern "C" int sb200_rxblocks_unpack(sb200_handle* h, const void* blocks, uint64_t nblocks, uint32_t left_shift, int16_t* iq_out, void* cuda_stream) {
    if (!h || !blocks || !iq_out || left_shift > 15) return h ? h->fail(SB200_E_INVALID, "bad argument") : SB200_E_INVALID;
    if (nblocks == 0) return SB200_OK;
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin()); call.reads(blocks);
    const uint4* d_in; uint4* d_out; Returns ret;
    CK(to_device(h->stage[0], (const uint4*)blocks, is_device_ptr(blocks), nblocks * 128ull, st, &d_in));
    CK(ret.bind(h->stage[1], (uint4*)iq_out, nblocks * 112ull, &d_out));
    const uint64_t nunits = nblocks * 7ull;
    const unsigned grid = (unsigned)((nunits + 255) / 256 < 148ull * 16 ? (nunits + 255) / 256 : 148ull * 16);
    k_rxblocks_unpack<<<grid, 256, 0, st>>>(d_in, nunits, left_shift, d_out);
    h->launches += 1;
    CK(cudaGetLastError());
    CK(ret.finish(st));
    return SB200_OK;
}

// descriptor words of every RX_BLOCK (___RX_DESC, _rx_manager.h:97-107): VStreamBits at byte 0, TimeStamp at byte 12
__global__ void __launch_bounds__(256) k_rxblocks_desc(const uint4* __restrict__ blocks, uint64_t nblocks, uint32_t* __restrict__ vbits, uint32_t* __restrict__ stamps) {
    for (uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; b < nblocks; b += (uint64_t)gridDim.x * blockDim.x) {
        const uint4 d = __ldg(blocks + b * 8u);
        if (vbits) vbits[b] = d.x;
        if (stamps) stamps[b] = d.w;
    }
}
extern "C" int sb200_rxblocks_desc(sb200_handle* h, const void* blocks, uint64_t nblocks, uint32_t* vstream_bits, uint32_t* timestamps, void* cuda_stream) {
    if (!h || !blocks || (!vstream_bits && !timestamps)) return h ? h->fail(SB200_E_INVALID, "bad argument") : SB200_E_INVALID;
    if (nblocks == 0) return SB200_OK;
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin()); call.reads(blocks);
    const uint4* d_in; uint32_t* d_v; uint32_t* d_t; Returns ret;
    CK(to_device(h->stage[0], (const uint4*)blocks, is_device_ptr(blocks), nblocks * 128ull, st, &d_in));
    CK(ret.bind(h->stage[1], vstream_bits, nblocks * 4ull, &d_v));
    CK(ret.bind(h->txns, timestamps, nblocks * 4ull, &d_t));
    const unsigned grid = (unsigned)((nblocks + 255) / 256 < 148ull * 8 ? (nblocks + 255) / 256 : 148ull * 8);
    k_rxblocks_desc<<<grid, 256, 0, st>>>(d_in, nblocks, d_v, d_t);
    h->launches += 1;
    CK(cudaGetLastError());
    CK(ret.finish(st));
    return SB200_OK;
}

extern "C" int sb200_set_option(sb200_handle* h, const char* name, uint64_t value) {
    if (!h || !name) return SB200_E_INVALID;
    if (!strcmp(name, "chunk_frames")) { h->chunk_frames = (uint32_t)value; return SB200_OK; }
    if (!strcmp(name, "chunk_frames_device")) { h->chunk_frames_device = (uint32_t)value; return SB200_OK; }
    if (!strcmp(name, "vq_pad_smem")) { h->vq_pad_smem = (uint32_t)value; return SB200_OK; }
    if (!strcmp(name, "front_stage")) { if (value > 2) return h->fail(SB200_E_INVALID, "front_stage is 0, 1 or 2"); h->front_stage = (uint32_t)value; return SB200_OK; }
    if (!strcmp(name, "host_decimate")) { h->host_decimate = (uint32_t)(value > 256 ? 256 : value); return SB200_OK; }
    if (!strcmp(name, "vl_defer_walk")) { h->vl_defer = value != 0; return SB200_OK; }
    if (!strcmp(name, "vl_hist_block")) { if (value != 6 && value != 8) return h->fail(SB200_E_INVALID, "vl_hist_block: 6 or 8"); h->vl_hb = (uint32_t)value; return SB200_OK; }
    if (!strcmp(name, "vl_l2_hints")) { h->vl_flags = (uint32_t)value & 3u; return SB200_OK; }   // bit 0 ring traffic evict_last, bit 1 soft values evict_first
    if (!strcmp(name, "vl_pad_smem")) { if (value > 48 * 1024) return h->fail(SB200_E_INVALID, "vl_pad_smem <= 49152"); h->vl_pad_smem = (uint32_t)value; return SB200_OK; }
    if (!strcmp(name, "viterbi_lane_min")) { h->lane_min = value > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)value; return SB200_OK; }
    if (!strcmp(name, "viterbi_lane_max")) { h->lane_max = value > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)value; return SB200_OK; }
    if (!strcmp(name, "host_stage_wc")) { h->hstage_wc = value != 0; return SB200_OK; }
    if (!strcmp(name, "host_decimate_mix")) { if (value > 2) return h->fail(SB200_E_INVALID, "host_decimate_mix: 0, 1 or 2"); h->host_mix = (uint32_t)value; host_pipe_forget_gather_cost(h->pipe); return SB200_OK; }
    if (!strcmp(name, "slot_table_immutable")) { h->tab_immutable = value != 0; h->tab_off = nullptr; return SB200_OK; }
    if (!strcmp(name, "ht_mcs_limit")) { if (value < 9 || value > 15) return h->fail(SB200_E_INVALID, "ht_mcs_limit is the first 802.11n MCS index refused: 9 .. 15 (11 = the reference's parser, 15 = MCS 8..14)"); h->ht_mcs_limit = (uint32_t)value; return SB200_OK; }
    return h->fail(SB200_E_INVALID, "unknown option");
}
