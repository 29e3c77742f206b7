// sora_b200 — what the host files of the C ABI (include/sora_b200.h) share: the handle, its device workspaces, the staging of a call's
// arguments and results, and the bookkeeping of a call; what only the 802.11a pipeline uses is HostPipe's (rx11a.cu).  Private to the library.
#pragma once
#include "../../include/sora_b200.h"
#include "tables.cuh"
#include <string.h>
#include <string>
#include <vector>

namespace sb {

struct FrameInfo;                                      // viterbi_k7_common.cuh
struct VitJob;

struct DevBuf {
    void* p = nullptr; size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete; DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    cudaError_t need(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = n + n / 8 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

inline bool is_device_ptr(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// Page-locked host memory (cudaHostAlloc, cudaHostRegister): a queued copy out of it reads it only when the stream reaches the copy.
// Pageable memory reports cudaMemoryTypeUnregistered; cudaMemcpyAsync copies it out before returning.
inline bool is_host_locked(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

// [off, off + len) lies inside [0, total), without the sum that a 64-bit offset near 2^64 would wrap
inline bool in_range(uint64_t off, uint64_t len, uint64_t total) { return len <= total && off <= total - len; }

// Host copy of a slot or payload table whose parts may each live on either side: one synchronise only if a part is on the device.
inline cudaError_t read_table(cudaStream_t st, const uint64_t* off, bool off_dev, const uint32_t* len, bool len_dev, uint32_t n,
                              std::vector<uint64_t>& offh, std::vector<uint32_t>& lenh) {
    offh.resize(n); lenh.resize(n);
    cudaError_t e = cudaSuccess;
    if (off_dev) e = cudaMemcpyAsync(offh.data(), off, n * 8ull, cudaMemcpyDeviceToHost, st); else memcpy(offh.data(), off, n * 8ull);
    if (e != cudaSuccess) return e;
    if (len_dev) e = cudaMemcpyAsync(lenh.data(), len, n * 4ull, cudaMemcpyDeviceToHost, st); else memcpy(lenh.data(), len, n * 4ull);
    if (e == cudaSuccess && (off_dev || len_dev)) e = cudaStreamSynchronize(st);
    return e;
}

// Device address of an input: `p` itself when it is device memory (`dev`), else workspace `b` (grown to bytes + slack) with the copy queued on `st`.
template <class T>
cudaError_t to_device(DevBuf& b, const T* p, bool dev, size_t bytes, cudaStream_t st, const T** d, size_t slack = 0) {
    if (dev) { *d = p; return cudaSuccess; }
    cudaError_t e = b.need(bytes + slack);
    if (e == cudaSuccess) e = cudaMemcpyAsync(b.p, p, bytes, cudaMemcpyHostToDevice, st);
    *d = (const T*)b.p;
    return e;
}

// The results of one call.  bind() gives the device address a kernel writes: the caller's buffer when it is device memory, else workspace `b`
// (grown to bytes + slack; a null result stays null).  bind2d() notes a strided copy of `rows` rows of `width` bytes out of a workspace into
// the caller's buffer on either side; copy() a linear one into host memory.  finish() queues the noted copies in the order they were noted
// and synchronises once if any of them goes to host memory.
struct Returns {
    struct Copy { void* dst; size_t dpitch; const void* src; size_t spitch, width, rows; bool to_host; };   // dpitch 0: one linear copy of width bytes
    Copy c[4]; int n = 0;                              // no call returns more than four results
    void copy(void* dst, const void* src, size_t bytes) { c[n++] = Copy{dst, 0, src, 0, bytes, 1, true}; }
    void bind2d(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t rows) {
        c[n++] = Copy{dst, dpitch, src, spitch, width, rows, !is_device_ptr(dst)};
    }
    template <class T>
    cudaError_t bind(DevBuf& b, T* p, size_t bytes, T** d, size_t slack = 0) {
        *d = p;
        if (!p || is_device_ptr(p)) return cudaSuccess;
        const cudaError_t e = b.need(bytes + slack);
        if (e != cudaSuccess) return e;
        *d = (T*)b.p; copy(p, b.p, bytes);
        return cudaSuccess;
    }
    cudaError_t finish(cudaStream_t st) {
        bool host = false;
        for (int i = 0; i < n; i++) {
            const Copy& k = c[i]; const cudaMemcpyKind kind = k.to_host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
            const cudaError_t e = k.dpitch ? cudaMemcpy2DAsync(k.dst, k.dpitch, k.src, k.spitch, k.width, k.rows, kind, st) : cudaMemcpyAsync(k.dst, k.src, k.width, kind, st);
            if (e != cudaSuccess) return e;
            host |= k.to_host;
        }
        return host ? cudaStreamSynchronize(st) : cudaSuccess;
    }
};

} // namespace sb

using namespace sb;

struct HostPipe;                                       // rx11a.cu: the chunked pipeline of the 802.11a batch receiver
int host_pipe_create(HostPipe** out);                 // SB200_E_CUDA without its streams or events; *out is set even then, for host_pipe_destroy
void host_pipe_destroy(HostPipe* p);                  // joins the host threads, then frees the pinned slabs
void host_pipe_forget_gather_cost(HostPipe* p);       // option host_decimate_mix: the next call measures the host gather anew

#define SB200_LANE_MIN_DEFAULT 16384u                 // the lane kernel for launches of 16 384 .. 49 152 code blocks, the four-lane kernel outside
#define SB200_LANE_MAX_DEFAULT 49152u                 // (tools/vit_crossover.py on an H100 SXM at 400 W: lane/four-lane time 1.46 at 8 192, 0.96 at 16 384, 0.85-0.93 up to 49 152, 1.03 at 65 536)

struct sb200_handle {
    int device = 0;
    uint32_t cca_thr = 1000 * 1000;
    DevTables T{};
    DevBuf tab, iq, off, len, info, soft, out, status, crc, res, taps[5], vlist, vcnt;
    uint16_t* inv_deint = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaEvent_t ev_done = nullptr; cudaStream_t last_st = nullptr; bool ordered = false;   // end of the previous call and its stream (CallScope)
    cudaEvent_t evk[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};   // boundaries of sync | front | viterbi | pack
    int nk = 0;
    bool timed = false;
    uint64_t launches = 0;
    uint32_t chunk_frames_device = 0;
    uint32_t chunk_frames = 4096;                      // slots per pipeline chunk (0 = one chunk, everything on the caller's stream)
    HostPipe* pipe = nullptr;                          // streams, events, pinned slabs and host threads of the chunked 802.11a calls (rx11a.cu)
    DevBuf stage[2], iq40, off40, len40, dcbuf;
    uint32_t ht_mcs_limit = 11;                        // first MCS the 802.11n HT-SIG parser refuses (PHY_11n.hpp:497); option "ht_mcs_limit"
    DevBuf soff, slen, spos, snev, sev;                // continuous-capture scout: current slot of every capture, position, event count, event list
    DevTablesTx X{}; DevBuf tabtx, txpay, txoff, txlen, txseed, txout, txns, txdesc, cca11n, ccaidx, tabtx11n, txout1, txpre; DevTablesTx11n XN{};   // 802.11a transmit tables (built on first use) and staging
    DevTables11n N{}; DevBuf tab11n, iq1;              // 802.11n tables (uploaded on first use) and the second antenna's samples
    std::vector<uint64_t> offh; std::vector<uint32_t> lenh;   // host copy of the slot table (cached for device-resident tables)
    const uint64_t* tab_off = nullptr; const uint32_t* tab_len = nullptr; uint32_t tab_n = 0, tab_max_len = 0; uint64_t tab_total = 0; bool tab_host = false;
    uint32_t front_stage = 1;                          // option: sample staging of k_front11a (0 direct loads, 1 register double buffer, 2 bulk async copy to shared memory)
    bool front_smem_set = false;                       // k_front11a<2> may use SB_FRONT_STAGE_SMEM bytes of dynamic shared memory on this device
    uint32_t host_decimate = 0;                        // option: host threads gathering the even samples of host-resident 40 Msps captures (0 = off)
    uint32_t host_mix = 1;                             // option host_decimate_mix: which chunks the pipeline gathers (0 all, 1 adaptive, 2 the odd ones)
    bool hstage_wc = false;                            // option host_stage_wc: pinned staging buffers of the decimating path allocated write-combined
    bool tab_immutable = false;                        // option slot_table_immutable: device-resident slot tables may be cached by address
    DevBuf slotchk;
    bool vl_defer = true;                              // option vl_defer_walk: the traceback spread over the step loop, one look-up per chunk (8-column blocks only)
    uint32_t vl_hb = 8;                                // option vl_hist_block: columns per history block of the lane kernel (6 | 8)
    uint32_t vl_flags = 1;                             // option vl_l2_hints: bit 0 ring traffic evict_last, bit 1 soft values evict_first (viterbi_k7_lane.cuh)
    uint32_t vl_pad_smem = 0;                          // experiment knob: the same for the lane kernel (fewer resident warps = a smaller history-ring working set in L2)
    uint32_t vq_pad_smem = 0;                          // experiment knob: extra dynamic shared memory per k_viterbi_re CTA of the 802.11a receiver (lowers occupancy)
    struct VrOcc { uint32_t smem = 0, ctas = 0; } vr_occ[3];      // k_viterbi_re<CR>: grid of its persistent CTAs, for `smem` bytes of padding
    // viterbi_k7_lane.cuh (one lane per code block, 32 per warp) needs a large batch to fill the machine: it decodes launches of at least
    // lane_min and at most lane_max code blocks, the four-lanes-per-code-block kernel the others.  Options "viterbi_lane_min" / "viterbi_lane_max".
    uint32_t lane_min = SB200_LANE_MIN_DEFAULT, lane_max = SB200_LANE_MAX_DEFAULT;
    const char* last_vit = "";                         // name of the Viterbi kernel the last launch used (sb200_last_viterbi_kernel)
    DevBuf nco;                                        // NCO table of the channelizer and the combiner (fir_kernels.cuh), built on first use
    uint64_t ch_smem_set = 0;                          // bit J (+ 32 for RAT): k_channelize<J, RAT> may use SB_CH_SMEM bytes of dynamic shared memory on this device
    int sms = 0;                                       // multiprocessors of the device (channel groups of k_channelize)
    uint32_t cb_smem_set = 0;                          // bit J (+ 16 for RAT): k_combine<J, RAT> may use SB_CB_SMEM (SB_CBR_SMEM_MAX) bytes of dynamic shared memory on this device
    DevBuf simtab, simlink, simtap;                    // channel simulator: its table (sim_kernels.cuh, built on first use), staged links and taps
    uint32_t sim_smem_set = 0;                         // bit J: k_channel_sim<J> may use its largest dynamic shared memory on this device
    DevBuf arbtab;                                     // sb200_channelize_arbitrary and sb200_combine_arbitrary: the NCO table and the call's H, staged per call (arb_kernels.cuh)
    uint32_t arb_smem_set = 0;                         // bit 0: k_channelize_arbitrary may use SB_ARB_SMEM_MAX bytes of dynamic shared memory on this device; bit J: k_combine_arbitrary<J> its budget
    DevBuf sptab, spwin;                               // sb200_spectrum: the twiddles of every stage size (built on first use) and the call's window
    uint32_t sp_smem_set = 0;                          // bit log2 N: k_spectrum<N> may use its dynamic shared memory on this device
    DevBuf vring;
    std::string err;
    int fail(int code, const char* what, cudaError_t e = cudaSuccess) {
        err = what; if (e != cudaSuccess) { err += ": "; err += cudaGetErrorString(e); }
        return code;
    }
};

#define CK(call) do { cudaError_t _e = (call); if (_e != cudaSuccess) return h->fail(SB200_E_CUDA, #call, _e); } while (0)

// One call of the C ABI on the caller's stream `st`.  Calls on one handle share its workspaces, so they run in the order they were made,
// whatever streams they are given: begin() makes `st` wait for the end of the handle's previous call when that ran on another stream (an
// event: no host synchronisation, no launch), and every call records its end on its stream.  cudaStreamPerThread names a different stream
// in every host thread, so it always waits.  reads(p) notes an input the call copies out of caller host memory on the stream: if it is
// page-locked, the call synchronises `st` once before it returns, so the caller may refill the buffer as soon as it has control back.
struct CallScope {
    sb200_handle* h; cudaStream_t st; bool locked = false;
    CallScope(sb200_handle* h_, cudaStream_t st_) : h(h_), st(st_) {}
    cudaError_t begin() const { return h->ordered && (h->last_st != st || st == cudaStreamPerThread) ? cudaStreamWaitEvent(st, h->ev_done, 0) : cudaSuccess; }
    void reads(const void* p) { if (p && !locked) locked = is_host_locked(p); }
    ~CallScope() {
        if (cudaEventRecord(h->ev_done, st) == cudaSuccess) { h->last_st = st; h->ordered = true; } else cudaGetLastError();
        if (locked) cudaStreamSynchronize(st);
    }
};

// Payload or slot table of a call, each half on either side.  load() reads it to the host and runs the call's own checks, check(i, inside =
// in_range(off, len, total)), which must refuse an entry not inside; upload() later places off and len in the call's workspaces.
struct FrameTable {
    const uint64_t* off; const uint32_t* len; uint32_t n;
    bool off_dev, len_dev;
    std::vector<uint64_t> offh; std::vector<uint32_t> lenh;
    FrameTable(const uint64_t* off_, const uint32_t* len_, uint32_t n_) : off(off_), len(len_), n(n_), off_dev(is_device_ptr(off_)), len_dev(is_device_ptr(len_)) {}
    template <class Check>
    int load(sb200_handle* h, cudaStream_t st, uint64_t total, Check check) {
        CK(read_table(st, off, off_dev, len, len_dev, n, offh, lenh));
        for (uint32_t i = 0; i < n; i++) { const int rc = check(i, in_range(offh[i], lenh[i], total)); if (rc != SB200_OK) return rc; }
        return SB200_OK;
    }
    cudaError_t upload(DevBuf& bo, DevBuf& bl, cudaStream_t st, const uint64_t** d_off, const uint32_t** d_len) {
        cudaError_t e = to_device(bo, off_dev ? off : offh.data(), off_dev, n * 8ull, st, d_off);
        return e != cudaSuccess ? e : to_device(bl, len_dev ? len : lenh.data(), len_dev, n * 4ull, st, d_len);
    }
};

// End of a timed call: ev1, nk (4 when evk[0..4] bound its stages), the launches not counted yet, the error check, the results' copies.
inline int finish_call(sb200_handle* h, cudaStream_t st, Returns& ret, int nk, uint64_t launches) {
    CK(cudaEventRecord(h->ev1, st));
    h->timed = true; h->nk = nk; h->launches += launches;
    CK(cudaGetLastError());
    CK(ret.finish(st));
    return SB200_OK;
}

// The five tap buffers of a *_taps call: sized and zeroed, filled by `run`, then back[i] bytes copied to every non-null dst[i].
template <class Run>
inline int run_with_taps(sb200_handle* h, const size_t (&size)[5], void* const (&dst)[5], const size_t (&back)[5], Run run) {
    for (int i = 0; i < 5; i++) { CK(h->taps[i].need(size[i])); CK(cudaMemset(h->taps[i].p, 0, size[i])); }
    const int rc = run();
    if (rc != SB200_OK) return rc;
    for (int i = 0; i < 5; i++) if (dst[i]) CK(cudaMemcpy(dst[i], h->taps[i].p, back[i], cudaMemcpyDeviceToHost));
    return SB200_OK;
}

// One allocation of 256-byte aligned tables: add() returns a part's offset (src null: a kernel fills it); upload() frees `b` on any failure.
// A cudaMemcpy from pageable memory may return before its DMA has landed, and a kernel on a non-blocking stream is not ordered after it:
// upload() synchronises the device once at the end (tables are uploaded once per handle).
struct TableArena {
    struct Part { size_t off; const void* src; size_t bytes; };
    std::vector<Part> parts; size_t size = 0;
    size_t add(const void* src, size_t bytes) { parts.push_back(Part{size, src, bytes}); size += (bytes + 255) & ~(size_t)255; return parts.back().off; }
    int upload(sb200_handle* h, DevBuf& b, const char* alloc_what, const char* copy_what) const {
        cudaError_t e = b.need(size);
        if (e != cudaSuccess) return h->fail(SB200_E_NOMEM, alloc_what, e);
        for (const Part& p : parts) if (p.src && e == cudaSuccess) e = cudaMemcpy((char*)b.p + p.off, p.src, p.bytes, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
        if (e != cudaSuccess) { b.release(); return h->fail(SB200_E_CUDA, copy_what, e); }
        return SB200_OK;
    }
};

// sb200.cu
int slot_table(sb200_handle* h, const uint64_t* frame_off, const uint32_t* frame_len, uint32_t nframes, uint64_t iq_total, bool need_host_copy,
               cudaStream_t st, const uint64_t** d_off, const uint32_t** d_len, uint32_t* max_len, bool* host_valid);
int stream_table(sb200_handle* h, const uint64_t* stream_off, const uint32_t* stream_len, uint32_t nstreams, uint64_t iq_total,
                 const void* res, const void* out_bytes, uint32_t* nframes_out, bool antennas_apart);
// viterbi.cu
int viterbi_stage(sb200_handle* h, uint32_t n, cudaStream_t s, const uint8_t* soft, uint64_t soft_stride, const FrameInfo* info, const VitJob& job,
                  uint8_t* out, uint64_t out_stride, uint32_t* status, uint32_t* crc, const int* rates, uint32_t nrates,
                  uint32_t first = 0, uint32_t slot = 0, uint32_t smem34 = 0);
