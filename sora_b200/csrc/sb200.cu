// sora_b200 — host side of the C ABI (include/sora_b200.h): workspaces, table upload, kernel launches.
// Single translation unit: the kernels live in the .cuh files included below.
#include "../../include/sora_b200.h"
#include "viterbi_k7_re.cuh"
#include "viterbi_k7_lane.cuh"
#include "rx11b_kernels.cuh"
#include "rx11n_kernels.cuh"
#include "tx11a_kernels.cuh"
#include "tx11b_kernels.cuh"
#include "tx11b_legacy_kernels.cuh"
#include "tx11a_legacy_kernels.cuh"
#include "tx11n_kernels.cuh"
#include "fir_kernels.cuh"
#include <stdlib.h>
#include <string>
#include <vector>
#include <chrono>
#include <string.h>
#include <new>
#include <memory>
#include <stdio.h>
#include <thread>
#include <mutex>
#include <condition_variable>
#include <atomic>
#include <emmintrin.h>

using namespace sb;

namespace {

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

__global__ void k_pack_results(const FrameInfo* __restrict__ info, const uint32_t* __restrict__ status,
                               const uint32_t* __restrict__ crc, uint32_t n, sb200_frame_result* __restrict__ res) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    FrameInfo fi = info[i];
    sb200_frame_result r;
    const bool decoded = fi.status == E_SUCCESS;       // otherwise the front end already reached a terminal code
    r.status = decoded ? status[i] : fi.status; r.rate_kbps = fi.rate_kbps; r.length = fi.length; r.crc32 = decoded ? crc[i] : 0u; r.nsym = fi.nsym_total;
    r.detect_index = fi.detect_vec == 0xFFFFFFFFu ? 0u : fi.detect_vec * 4u;
    r.cfo_est = (int16_t)fi.cfo_est; r.peak_index = (uint16_t)fi.peak_index;
    res[i] = r;
}

// Continuous-capture scout (sb200_rx11a_streams): after a header-only pass, move every live capture past the event it just found the way
// RxThread does (fb11a_demod.cpp:29-81: the driver sees the event after the source block that completed the last symbol, flushes, resets, and
// the source continues with the next 28-sample block; only CF_VecDC survives), and note the event as a slot for the batched decode that follows.
struct StreamEvent { uint64_t off; uint32_t len; uint32_t pos_after; int2 dc; };
__global__ void k_stream_advance(const FrameInfo* __restrict__ info, uint32_t n, uint64_t* __restrict__ off_cur, uint32_t* __restrict__ len_cur,
                                 int2* __restrict__ dc_cur, uint32_t* __restrict__ pos_cur, uint32_t* __restrict__ nev, uint32_t max_frames,
                                 StreamEvent* __restrict__ ev, uint32_t* __restrict__ live) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const uint32_t rem = len_cur[s];
    if (rem < 28u) return;                                   // finished earlier
    const FrameInfo fi = info[s];
    if (fi.status != E_SUCCESS && fi.status != E_PLCP_HEADER_FAIL) { len_cur[s] = 0; return; }     // ran out of samples: RxThread returns
    const uint32_t consumed = fi.status == E_PLCP_HEADER_FAIL ? 1u : fi.nsym_total;                 // OFDM symbols that went through the graph
    const uint64_t e20 = (uint64_t)fi.detect_vec * 4ull + 144ull + 80ull * consumed;               // 20 Msps samples up to the end of the last symbol
    const uint64_t v_last = e20 / 4ull - 1ull, blk = (8ull * v_last + 7ull) / 28ull;
    uint64_t adv = (blk + 1ull) * 28ull; if (adv > rem) adv = rem;
    const uint32_t j = nev[s];
    StreamEvent e; e.off = off_cur[s]; e.len = (uint32_t)adv; e.pos_after = pos_cur[s] + (uint32_t)adv; e.dc = dc_cur[s];
    ev[(size_t)s * max_frames + j] = e;
    nev[s] = j + 1u;
    dc_cur[s] = make_int2(fi.dc_re, fi.dc_im);
    off_cur[s] += adv; pos_cur[s] += (uint32_t)adv;
    const uint32_t left = rem - (uint32_t)adv;
    const bool go_on = j + 1u < max_frames && left >= 28u;
    len_cur[s] = go_on ? left : 0u;
    if (go_on) atomicAdd(live, 1u);
}

// max(len) and an out-of-bounds flag over a device-resident slot table: res[0] = max frame_len, res[1] != 0 if any slot leaves [0, iq_total)
__global__ void k_slot_check(const uint64_t* __restrict__ off, const uint32_t* __restrict__ len, uint32_t n, uint64_t iq_total, uint32_t* __restrict__ res) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t l = 0, bad = 0;
    if (i < n) { l = len[i]; const uint64_t o = off[i]; bad = (l > iq_total || o > iq_total - l) ? 1u : 0u; }
    l = __reduce_max_sync(0xFFFFFFFFu, l); bad = __reduce_or_sync(0xFFFFFFFFu, bad);
    if ((threadIdx.x & 31) == 0) { if (l) atomicMax(res, l); if (bad) atomicOr(res + 1, 1u); }
}

bool is_device_ptr(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// Page-locked host memory (cudaHostAlloc, cudaHostRegister): a queued copy out of it reads it only when the stream reaches the copy.
// Pageable memory reports cudaMemoryTypeUnregistered; cudaMemcpyAsync copies it out before returning.
bool is_host_locked(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

// [off, off + len) lies inside [0, total), without the sum that a 64-bit offset near 2^64 would wrap
inline bool in_range(uint64_t off, uint64_t len, uint64_t total) { return len <= total && off <= total - len; }

// Host copy of a slot or payload table whose parts may each live on either side: one synchronise only if a part is on the device.
cudaError_t read_table(cudaStream_t st, const uint64_t* off, bool off_dev, const uint32_t* len, bool len_dev, uint32_t n,
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

} // namespace

// ---- host-side TDownSample2 for host-resident captures ---------------------------------------------------------------------------------
// The 802.11a graph keeps samples 0 and 2 of every 4 (samples.hpp:27-49): half of a 40 Msps capture is dropped on arrival.  With the option
// "host_decimate" = T > 0 the chunked host-IQ path gathers the even samples of every slot of a chunk into pinned staging memory with T host
// threads and sends only those over PCIe (half the bytes); the kernels then read the packed copy with stride 1 (sh = 0).  Results are
// identical: the same samples reach the same arithmetic.
namespace sb { void gather_even(const uint32_t* src, uint32_t n2, uint32_t* dst); }      // host_gather.cpp: dst[j] = src[2 j], streaming stores, SSE2 / AVX-512 chosen at run time
static inline void decimate_slot(const uint32_t* src, uint32_t n2, uint32_t* dst) { sb::gather_even(src, n2, dst); }
struct DecimPool {
    // n worker threads; submit() hands them one chunk and returns, wait() blocks until it is gathered: the caller queues the previous chunk's
    // copies and kernels in between, so the host cores never wait for the launch path (and the launch path never waits for them).
    struct Job { const uint32_t* iq; const uint64_t* off; const uint32_t* len; const uint64_t* doff; uint32_t f0, f1; uint32_t* dst; };
    std::vector<std::thread> th; std::mutex m; std::condition_variable cv, cv_done;
    Job job{}; uint64_t gen = 0; int pending = 0; bool stop = false; int n = 0;
    std::chrono::steady_clock::time_point t_submit; double last_ms = 0.0;   // wall time from submit() to the last worker's end
    static void part(const Job& j, int w, int n) {
        const uint64_t cnt = j.f1 - j.f0; const uint32_t a = j.f0 + (uint32_t)(cnt * w / n), b = j.f0 + (uint32_t)(cnt * (w + 1) / n);
        for (uint32_t f = a; f < b; f++) decimate_slot(j.iq + j.off[f], (j.len[f] + 1u) / 2u, j.dst + (j.doff[f] - j.doff[j.f0]));
        _mm_sfence();                                   // streaming stores visible before the copy is queued
    }
    void start(int nthreads) {
        shutdown(); n = nthreads < 1 ? 1 : nthreads; stop = false;
        for (int w = 0; w < n; w++) th.emplace_back([this, w]() {
            uint64_t seen = 0;
            for (;;) {
                Job j;
                { std::unique_lock<std::mutex> l(m); cv.wait(l, [&] { return stop || gen != seen; }); if (stop) return; seen = gen; j = job; }
                part(j, w, n);
                { std::lock_guard<std::mutex> l(m);
                  if (--pending == 0) { last_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_submit).count(); cv_done.notify_all(); } }
            }
        });
    }
    void submit(const Job& j) {                         // one job in flight at a time: wait() first
        { std::lock_guard<std::mutex> l(m); job = j; gen++; pending = n; t_submit = std::chrono::steady_clock::now(); }
        cv.notify_all();
    }
    double wait() { std::unique_lock<std::mutex> l(m); cv_done.wait(l, [&] { return pending == 0; }); return last_ms; }
    void shutdown() {
        { std::lock_guard<std::mutex> l(m); stop = true; }
        cv.notify_all();
        for (auto& t : th) t.join();
        th.clear(); n = 0;
    }
    ~DecimPool() { shutdown(); }
};

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
    cudaStream_t s_copy = nullptr, s_front = nullptr;
    cudaEvent_t ev_start = nullptr, ev_h2d[2] = {nullptr, nullptr}, ev_front[2] = {nullptr, nullptr};
    DevBuf stage[2], iq40, off40, len40, dcbuf;
    double gather_ms = 0.0;                            // host_decimate: time the host threads spent gathering during the last call (SB200_TRACE prints it)
    uint32_t ht_mcs_limit = 11;                        // first MCS the 802.11n HT-SIG parser refuses (PHY_11n.hpp:497); option "ht_mcs_limit"
    DevBuf soff, slen, spos, snev, sev;                // continuous-capture scout: current slot of every capture, position, event count, event list
    DevTablesTx X{}; DevBuf tabtx, txpay, txoff, txlen, txseed, txout, txns, txdesc, cca11n, ccaidx, tabtx11n, txout1, txpre; DevTablesTx11n XN{};   // 802.11a transmit tables (built on first use) and staging
    DevTables11n N{}; DevBuf tab11n, iq1;              // 802.11n tables (uploaded on first use) and the second antenna's samples
    std::vector<uint64_t> offh; std::vector<uint32_t> lenh;   // host copy of the slot table (cached for device-resident tables)
    const uint64_t* tab_off = nullptr; const uint32_t* tab_len = nullptr; uint32_t tab_n = 0, tab_max_len = 0; uint64_t tab_total = 0; bool tab_host = false;
    uint32_t front_stage = 0;                          // option: sample staging of k_front11a (0 direct loads, 1 register double buffer, 2 bulk async copy to shared memory)
    uint32_t host_decimate = 0;                        // option: host threads gathering the even samples of host-resident 40 Msps captures (0 = off)
    DecimPool* pool = nullptr; void* hstage[4] = {nullptr, nullptr, nullptr, nullptr}; size_t hstage_cap = 0; cudaEvent_t ev_hfree[4] = {nullptr, nullptr, nullptr, nullptr};
    // host_decimate_mix (default 1 = adaptive): per chunk, the decimating path either gathers on the host threads (half the bytes cross) or,
    // when the copies already queued would run out before a gather could finish, sends the chunk as it is — the link and the host cores are
    // two resources and the call keeps both busy.  0 = every chunk gathered; 2 = alternate (tests).
    uint32_t host_mix = 1;
    bool hstage_wc = false, hstage_is_wc = false;      // option host_stage_wc: pinned staging buffers of the decimating path allocated write-combined
    std::vector<cudaEvent_t> ev_link; std::vector<uint64_t> link_bytes;     // one timed event per chunk copy of the current call, and its size
    double link_bpms = 50e6;                           // estimate of the link rate, bytes per ms (largest rate seen between two consecutive copy ends)
    double gather_ms_per_sample = 0.0;                 // running estimate of the host gather cost per 40 Msps sample (0 = not measured yet)
    uint64_t last_h2d_bytes = 0, last_gathered_chunks = 0, last_chunks = 0;
    std::vector<uint64_t> chunk_lo, chunk_hi; std::vector<int8_t> chunk_buf;   // per chunk of the current call: span in the capture, pinned buffer of a gathered chunk
    DevBuf doff; std::vector<uint64_t> doffh;
    bool tab_immutable = false;                        // option slot_table_immutable: device-resident slot tables may be cached by address
    DevBuf slotchk;
    bool vl_defer = true;                              // option vl_defer_walk: the traceback spread over the step loop, one look-up per chunk (8-column blocks only)
    uint32_t vl_hb = 8;                                // option vl_hist_block: columns per history block of the lane kernel (6 | 8)
    uint32_t vl_flags = 1;                             // option vl_l2_hints: bit 0 ring traffic evict_last, bit 1 soft values evict_first (viterbi_k7_lane.cuh)
    uint32_t vl_pad_smem = 0;                          // experiment knob: the same for the lane kernel (fewer resident warps = a smaller history-ring working set in L2)
    uint32_t vq_pad_smem = 0;                          // experiment knob: extra dynamic shared memory per Viterbi CTA (lowers occupancy)
    // viterbi_k7_lane.cuh (one lane per code block, 32 per warp) needs a large batch to fill the machine: it decodes launches of at least
    // lane_min and at most lane_max code blocks, the four-lanes-per-code-block kernel the others.  Options "viterbi_lane_min" / "viterbi_lane_max";
    // SB200_VITERBI=v8 forces it (0 .. 0xFFFFFFFF), v3 forbids it.
    uint32_t lane_min = SB200_LANE_MIN_DEFAULT, lane_max = SB200_LANE_MAX_DEFAULT;
    const char* last_vit = "";                         // name of the Viterbi kernel the last launch used (sb200_last_viterbi_kernel)
    DevBuf nco;                                        // channelizer NCO table (fir_kernels.cuh), built on first use
    uint32_t ch_smem_set = 0;                          // bit J: k_channelize<J> may use SB_CH_SMEM bytes of dynamic shared memory on this device
    int sms = 0;                                       // multiprocessors of the device (channel groups of k_channelize)
    DevBuf vring;
    bool use_pair = false;                             // SB200_VITERBI=v4: two lanes per code block, 16 code blocks per warp (A/B against four lanes)
    bool use_v2 = false;                               // SB200_VITERBI=v2 selects the per-step-mark quad kernel (A/B against the history-carrying one)
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
static int finish_call(sb200_handle* h, cudaStream_t st, Returns& ret, int nk, uint64_t launches) {
    CK(cudaEventRecord(h->ev1, st));
    h->timed = true; h->nk = nk; h->launches += launches;
    CK(cudaGetLastError());
    CK(ret.finish(st));
    return SB200_OK;
}

// The five tap buffers of a *_taps call: sized and zeroed, filled by `run`, then back[i] bytes copied to every non-null dst[i].
template <class Run>
static int run_with_taps(sb200_handle* h, const size_t (&size)[5], void* const (&dst)[5], const size_t (&back)[5], Run run) {
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
    { const char* e = getenv("SB200_VITERBI"); h->use_v2 = e && e[0] == 'v' && e[1] == '2'; h->use_pair = e && e[0] == 'v' && e[1] == '4'; if (e && e[0] == 'v' && e[1] == '8') { h->lane_min = 0; h->lane_max = 0xFFFFFFFFu; } else if (e && e[0] == 'v') h->lane_min = 0xFFFFFFFFu; }
    if (cudaSetDevice(device) != cudaSuccess) { delete h; return SB200_E_CUDA; }
    int rc = upload_tables(h);
    if (rc == SB200_OK && (cudaEventCreate(&h->ev0) != cudaSuccess || cudaEventCreate(&h->ev1) != cudaSuccess)) rc = SB200_E_CUDA;
    for (int i = 0; i < 5 && rc == SB200_OK; i++) if (cudaEventCreate(&h->evk[i]) != cudaSuccess) rc = SB200_E_CUDA;
    if (rc == SB200_OK && (cudaStreamCreateWithFlags(&h->s_copy, cudaStreamNonBlocking) != cudaSuccess || cudaStreamCreateWithFlags(&h->s_front, cudaStreamNonBlocking) != cudaSuccess)) rc = SB200_E_CUDA;
    if (rc == SB200_OK && (cudaEventCreateWithFlags(&h->ev_start, cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&h->ev_done, cudaEventDisableTiming) != cudaSuccess)) rc = SB200_E_CUDA;
    for (int i = 0; i < 2 && rc == SB200_OK; i++) if (cudaEventCreateWithFlags(&h->ev_h2d[i], cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&h->ev_front[i], cudaEventDisableTiming) != cudaSuccess) rc = SB200_E_CUDA;
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
    if (h->ev_start) cudaEventDestroy(h->ev_start);
    if (h->ev_done) cudaEventDestroy(h->ev_done);
    for (int i = 0; i < 2; i++) { if (h->ev_h2d[i]) cudaEventDestroy(h->ev_h2d[i]); if (h->ev_front[i]) cudaEventDestroy(h->ev_front[i]); }
    for (cudaEvent_t e : h->ev_link) cudaEventDestroy(e);
    delete h->pool; for (int i = 0; i < 4; i++) { if (h->hstage[i]) cudaFreeHost(h->hstage[i]); if (h->ev_hfree[i]) cudaEventDestroy(h->ev_hfree[i]); }
    if (h->s_copy) cudaStreamDestroy(h->s_copy);
    if (h->s_front) cudaStreamDestroy(h->s_front);
    delete h;
}
extern "C" const char* sb200_last_error(const sb200_handle* h) { return h ? h->err.c_str() : "null handle"; }
extern "C" uint64_t sb200_launch_count(const sb200_handle* h) { return h ? h->launches : 0; }
extern "C" const char* sb200_last_viterbi_kernel(const sb200_handle* h) { return h ? h->last_vit : ""; }
extern "C" int sb200_last_transfer(const sb200_handle* h, uint64_t* h2d_bytes, uint32_t* chunks, uint32_t* chunks_gathered) {
    if (!h) return SB200_E_INVALID;
    if (h2d_bytes) *h2d_bytes = h->last_h2d_bytes;
    if (chunks) *chunks = (uint32_t)h->last_chunks;
    if (chunks_gathered) *chunks_gathered = (uint32_t)h->last_gathered_chunks;
    return SB200_OK;
}
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
static int slot_table(sb200_handle* h, const uint64_t* frame_off, const uint32_t* frame_len, uint32_t nframes, uint64_t iq_total, bool need_host_copy,
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

// One launch of the Viterbi for code rate CR: SB200_VITERBI=v2 the per-step-mark quad kernel (dynamic shared memory `smem`); else the lane
// kernel (viterbi_k7_lane.cuh) for launches of lane_min .. lane_max code blocks, in the rendering the options select (8-column history blocks
// with the deferred walk unless told otherwise); below that the four-lanes-per-code-block kernel (SB200_VITERBI=v4: two lanes, for A/B).
// vring_need() sizes the lane kernel's history rings for n code blocks first.
static bool use_lane(const sb200_handle* h, uint32_t n) { return n >= h->lane_min && n <= h->lane_max; }
static cudaError_t vring_need(sb200_handle* h, uint32_t n) {
    if (use_lane(h, n)) return h->vring.need((size_t)((n + SB_VL_FR - 1) / SB_VL_FR) * SB_VL_NB8D * SB_VL_ENTRY * 16);   // the largest ring of the lane kernel's renderings
    return cudaSuccess;                                // the four- / two-lane kernels keep their ring in shared memory
}
template <int CR>
static void launch_viterbi(sb200_handle* h, uint32_t n, cudaStream_t s, const uint8_t* soft, uint64_t soft_stride, const uint32_t* list, const uint32_t* cnt,
                           const FrameInfo* info, const VitJob& job, uint8_t* out, uint64_t out_stride, uint32_t* status, uint32_t* crc, uint32_t smem) {
    if (h->use_v2) { k_viterbi_quad<CR><<<(n + SB_VQ_FR - 1) / SB_VQ_FR, 32 * SB_VQ_WARPS, smem, s>>>(soft, soft_stride, n, info, job, h->T, out, out_stride, status, crc); return; }
    const unsigned g = (n + SB_VR_FR - 1) / SB_VR_FR, gp = (n + 15) / 16;
    const uint32_t raw_off = info ? 14u : 0u; uint32_t* const nraw = status;   // frames are decoded 14 bytes into their row, raw blocks at its start
    uint4* const ring = (uint4*)h->vring.p;             // the lane kernel's history rings
    h->last_vit = use_lane(h, n) ? "k_viterbi_lane" : "k_viterbi_re";
    if (use_lane(h, n) && h->vl_hb == 8 && h->vl_defer) k_viterbi_lane<CR, 8, true><<<(n + SB_VL_FR - 1) / SB_VL_FR, 32, h->vl_pad_smem, s>>>(soft, soft_stride, n, list, cnt, info, job, out, out_stride, raw_off, nraw, ring, h->vl_flags);
    else if (use_lane(h, n) && h->vl_hb == 8) k_viterbi_lane<CR, 8><<<(n + SB_VL_FR - 1) / SB_VL_FR, 32, h->vl_pad_smem, s>>>(soft, soft_stride, n, list, cnt, info, job, out, out_stride, raw_off, nraw, ring, h->vl_flags);
    else if (use_lane(h, n))         k_viterbi_lane<CR, 6><<<(n + SB_VL_FR - 1) / SB_VL_FR, 32, h->vl_pad_smem, s>>>(soft, soft_stride, n, list, cnt, info, job, out, out_stride, raw_off, nraw, ring, h->vl_flags);
    else if (h->use_pair)            k_viterbi_re<CR, 1><<<gp, 32, 0, s>>>(soft, soft_stride, n, list, cnt, info, job, out, out_stride, raw_off, nraw);
    else                             k_viterbi_re<CR, 2><<<g, 32, 0, s>>>(soft, soft_stride, n, list, cnt, info, job, out, out_stride, raw_off, nraw);
}

// The Viterbi stage: one launch per code rate of `rates`, in that order.  Frames (`info` set) get work lists (vlist from frame `first`, vcnt
// block `slot`; the quad kernel needs none) and k_sink11a; raw code blocks (`info` null) neither.  `smem34`: the 802.11a vq_pad_smem knob.
static int viterbi_stage(sb200_handle* h, uint32_t n, cudaStream_t s, const uint8_t* soft, uint64_t soft_stride, const FrameInfo* info, const VitJob& job,
                         uint8_t* out, uint64_t out_stride, uint32_t* status, uint32_t* crc, const int* rates, uint32_t nrates,
                         uint32_t first = 0, uint32_t slot = 0, uint32_t smem34 = 0) {
    const uint32_t* list = nullptr; const uint32_t* cnt = nullptr;
    if (!h->use_v2) {
        CK(vring_need(h, n));
        if (info) {
            CK(h->vlist.need((first + (size_t)n) * 12ull)); CK(h->vcnt.need(16ull * (slot + 1u)));
            uint32_t* d_list = (uint32_t*)h->vlist.p + 3 * (size_t)first; uint32_t* d_cnt = (uint32_t*)h->vcnt.p + 4 * (size_t)slot;
            CK(cudaMemsetAsync(d_cnt, 0, 16, s));
            k_vit_lists<<<(n + 255) / 256, 256, 0, s>>>(info, n, d_cnt, d_list);
            list = d_list; cnt = d_cnt; h->launches += 1;
        }
    }
    for (uint32_t r = 0; r < nrates; r++) {
        const int cr = rates[r];
        if (cr == CR_34) launch_viterbi<CR_34>(h, n, s, soft, soft_stride, list, cnt, info, job, out, out_stride, status, crc, smem34);
        else if (cr == CR_12) launch_viterbi<CR_12>(h, n, s, soft, soft_stride, list, cnt, info, job, out, out_stride, status, crc, 0);
        else launch_viterbi<CR_23>(h, n, s, soft, soft_stride, list, cnt, info, job, out, out_stride, status, crc, 0);
    }
    h->launches += nrates;
    if (info && !h->use_v2) { k_sink11a<<<(n + 127) / 128, 128, 0, s>>>(out, out_stride, n, info, h->T, status, crc); h->launches += 1; }
    return SB200_OK;
}

// Launch the decode kernels for frames [f0, f1) of a call.  `iq_base + off[f]` must address slot f.
// sync + front end go to `sf`, the Viterbi launches to `sv` (sv waits for `front_done` when the streams differ).
static int launch_chunk(sb200_handle* h, const uint32_t* iq_base, const uint64_t* d_off, const uint32_t* d_len, uint32_t f0, uint32_t f1,
                        uint64_t soft_stride, uint64_t row, cudaStream_t sf, cudaStream_t sv, cudaEvent_t front_done, FrontTaps taps, bool timed, const int2* dc_init = nullptr, uint32_t chunk_idx = 0, uint32_t sh = 1, uint32_t lsh = 0) {
    const uint32_t n = f1 - f0;
    FrameInfo* d_info = (FrameInfo*)h->info.p + f0;
    uint8_t* d_soft = (uint8_t*)h->soft.p + (size_t)f0 * soft_stride;
    uint8_t* d_out = (uint8_t*)h->out.p + (size_t)f0 * row;
    uint32_t* d_status = (uint32_t*)h->status.p + f0; uint32_t* d_crc = (uint32_t*)h->crc.p + f0;
    if (timed) CK(cudaEventRecord(h->evk[0], sf));
    k_sync11a<<<(n + 127) / 128, 128, 0, sf>>>(iq_base, d_off + f0, d_len + f0, n, h->cca_thr, h->T, d_info, dc_init ? dc_init + f0 : nullptr, sh, lsh);
    if (timed) CK(cudaEventRecord(h->evk[1], sf));
    {   const dim3 g((n + SB_FRONT_WARPS - 1) / SB_FRONT_WARPS), b(32 * SB_FRONT_WARPS);
        if (h->front_stage == 2) k_front11a<2><<<g, b, 0, sf>>>(iq_base, d_off + f0, d_len + f0, n, h->T, d_info, d_soft, soft_stride, h->inv_deint, taps, sh, lsh);
        else if (h->front_stage == 1) k_front11a<1><<<g, b, 0, sf>>>(iq_base, d_off + f0, d_len + f0, n, h->T, d_info, d_soft, soft_stride, h->inv_deint, taps, sh, lsh);
        else k_front11a<0><<<g, b, 0, sf>>>(iq_base, d_off + f0, d_len + f0, n, h->T, d_info, d_soft, soft_stride, h->inv_deint, taps, sh, lsh); }
    if (timed) CK(cudaEventRecord(h->evk[2], sf));
    if (sv != sf) { CK(cudaEventRecord(front_done, sf)); CK(cudaStreamWaitEvent(sv, front_done, 0)); }
    h->launches += 2;
    VitJob job{}; job.depth = 256; job.lookahead = 24; job.raw = 0;
    static const int rates[3] = {CR_34, CR_12, CR_23};
    const int rc = viterbi_stage(h, n, sv, d_soft, soft_stride, d_info, job, d_out, row, d_status, d_crc, rates, 3, f0, chunk_idx, h->vq_pad_smem);
    if (rc != SB200_OK) return rc;
    if (timed) CK(cudaEventRecord(h->evk[3], sv));
    return SB200_OK;
}

// shared body of sb200_rx11a_batch / sb200_rx11a_taps.
// Large calls are cut into chunks of h->chunk_frames slots and pipelined over three streams: host->device copy of chunk
// k+1 (copy stream) | carrier sense + OFDM front end of chunk k+1 (front stream) | Viterbi of chunk k (caller's stream).
// The front end is latency bound and the Viterbi integer-issue bound, so they overlap well on the same SMs.
static int rx11a_run(sb200_handle* h, const int16_t* iq, uint64_t iq_total, const uint64_t* frame_off, const uint32_t* frame_len,
                     uint32_t nframes, uint8_t* out_bytes, uint32_t out_stride, sb200_frame_result* res, cudaStream_t st,
                     FrontTaps taps, uint8_t* soft_host, uint64_t soft_host_stride, const int2* dc_init = nullptr, bool no_chunk = false, bool rate20 = false) {
    if (!h || !iq || !frame_off || !frame_len || !res) return h ? h->fail(SB200_E_INVALID, "null argument") : SB200_E_INVALID;
    if (nframes == 0) return SB200_OK;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin()); call.reads(iq);
    // slot table: checked on every call (slot_table above); the chunked host-IQ path also needs it on the host
    const bool iq_dev = is_device_ptr(iq);
    std::vector<uint64_t>& offh = h->offh; std::vector<uint32_t>& lenh = h->lenh;
    const uint64_t* d_off; const uint32_t* d_len; uint32_t max_len = 0; bool tab_on_host = false;
    {
        const bool may_chunk = !no_chunk && !rate20 && !iq_dev && h->chunk_frames != 0 && nframes > h->chunk_frames;
        int rc = slot_table(h, frame_off, frame_len, nframes, iq_total, may_chunk, st, &d_off, &d_len, &max_len, &tab_on_host);
        if (rc != SB200_OK) return rc;
        if (rate20) { if (max_len > 0x7FFFFFFFu) return h->fail(SB200_E_INVALID, "slot too long"); max_len <<= 1; }   // slots counted in 20 Msps samples
    }
    // workspaces
    const uint64_t max_sym = (max_len / 2u) / 80u + 1u;
    const uint64_t soft_stride = ((max_sym * 288ull) + 15ull) & ~15ull;
    const uint64_t row = 2560;                         // >= 2500 (MTU, PHY_11a.hpp:571) + SERVICE
    CK(h->info.need(nframes * sizeof(FrameInfo)));
    CK(h->soft.need(nframes * soft_stride));
    CK(h->out.need(nframes * row));
    CK(h->status.need(nframes * 4ull)); CK(h->crc.need(nframes * 4ull)); CK(h->res.need(nframes * sizeof(sb200_frame_result)));
    CK(h->vlist.need(nframes * 12ull));
    const bool tapping = taps.freq_coeffs || taps.fft_out || soft_host || dc_init;
    // device-resident IQ gains nothing from chunking (a chunk's Viterbi grid no longer fills 132 SMs x 5 CTAs); host IQ does:
    // the PCIe copy of chunk k+1 hides behind the kernels of chunk k.  chunk_frames_device lets a caller force it anyway.
    const uint32_t want = (no_chunk || rate20) ? 0u : iq_dev ? h->chunk_frames_device : h->chunk_frames;
    const uint32_t chunk = (want == 0 || tapping || nframes <= want || (!iq_dev && !tab_on_host)) ? nframes : want;
    const bool pipelined = chunk < nframes;
    CK(h->vcnt.need(16ull * ((nframes + chunk - 1) / chunk)));
    const bool res_dev_all = is_device_ptr(res), out_dev_all = out_bytes && is_device_ptr(out_bytes);
    sb200_frame_result* d_res_all = res_dev_all ? res : (sb200_frame_result*)h->res.p;
    CK(cudaEventRecord(h->ev0, st));
    if (!pipelined) {
        const uint32_t* d_iq;
        CK(to_device(h->iq, (const uint32_t*)iq, iq_dev, iq_total * 4ull, st, &d_iq));
        if (!iq_dev) { h->last_h2d_bytes = iq_total * 4ull; h->last_gathered_chunks = 0; h->last_chunks = 1; }
        int rc = launch_chunk(h, d_iq, d_off, d_len, 0, nframes, soft_stride, row, st, st, nullptr, taps, true, dc_init, 0, rate20 ? 0u : 1u, rate20 ? 1u : 0u);
        if (rc != SB200_OK) return rc;
    } else {
        // host IQ: per-chunk sample range [lo, hi) staged through two device buffers; with host_decimate only the even samples of every slot
        // travel, gathered by the host threads into one of four pinned buffers while earlier chunks are on the wire / in the kernels
        const bool dec = !iq_dev && h->host_decimate > 0;
        const uint32_t mix = dec ? h->host_mix : 0u;
        const uint64_t* d_off_dec = nullptr; std::vector<uint64_t>& doffh = h->doffh;
        uint64_t stage_samples = 0, hstage_samples = 0;
        const uint32_t nchunks = (nframes + chunk - 1) / chunk;
        if (!iq_dev) {
            if (dec) {
                doffh.resize((size_t)nframes + 1); doffh[0] = 0;
                for (uint32_t i = 0; i < nframes; i++) doffh[i + 1] = doffh[i] + (lenh[i] + 1u) / 2u;
            }
            for (uint32_t f0 = 0; f0 < nframes; f0 += chunk) {
                const uint32_t f1 = f0 + chunk < nframes ? f0 + chunk : nframes;
                if (dec) { const uint64_t n = doffh[f1] - doffh[f0]; if (n > hstage_samples) hstage_samples = n; if (n > stage_samples) stage_samples = n; }
                if (!dec || mix) {
                    uint64_t lo = ~0ull, hi = 0;
                    for (uint32_t i = f0; i < f1; i++) { if (offh[i] < lo) lo = offh[i]; if (offh[i] + lenh[i] > hi) hi = offh[i] + lenh[i]; }
                    if (hi - lo > stage_samples) stage_samples = hi - lo;
                }
            }
            CK(h->stage[0].need(stage_samples * 4ull + 16)); CK(h->stage[1].need(stage_samples * 4ull + 16));
            if (dec) {
                if (!h->pool || h->pool->n != (int)h->host_decimate) { delete h->pool; h->pool = new (std::nothrow) DecimPool(); if (!h->pool) return h->fail(SB200_E_NOMEM, "host thread pool"); h->pool->start((int)h->host_decimate); }
                if (h->hstage_cap < hstage_samples * 4ull || h->hstage_wc != h->hstage_is_wc) {
                    for (int i = 0; i < 4; i++) if (h->ev_hfree[i]) CK(cudaEventSynchronize(h->ev_hfree[i]));     // no copy out of a buffer still queued
                    for (int i = 0; i < 4; i++) { if (h->hstage[i]) cudaFreeHost(h->hstage[i]); h->hstage[i] = nullptr; }
                    h->hstage_cap = 0;
                    const size_t want_b = hstage_samples * 4ull + hstage_samples / 2 + 256;
                    // the staging buffers are written once by the host threads (streaming stores) and read only by the copy engine: write-combined
                    // memory (option host_stage_wc) is not snooped on its way over PCIe
                    for (int i = 0; i < 4; i++) CK(cudaHostAlloc(&h->hstage[i], want_b, h->hstage_wc ? cudaHostAllocWriteCombined : cudaHostAllocDefault));
                    h->hstage_cap = want_b; h->hstage_is_wc = h->hstage_wc;
                }
                for (int i = 0; i < 4; i++) if (!h->ev_hfree[i]) CK(cudaEventCreateWithFlags(&h->ev_hfree[i], cudaEventDisableTiming));
                CK(h->doff.need(nframes * 8ull)); CK(cudaMemcpyAsync(h->doff.p, doffh.data(), nframes * 8ull, cudaMemcpyHostToDevice, st));
                d_off_dec = (const uint64_t*)h->doff.p;
            }
            while (h->ev_link.size() < nchunks) { cudaEvent_t e; CK(cudaEventCreate(&e)); h->ev_link.push_back(e); }
            h->link_bytes.assign(nchunks, 0);
        }
        CK(cudaEventRecord(h->ev_start, st));
        CK(cudaStreamWaitEvent(h->s_copy, h->ev_start, 0)); CK(cudaStreamWaitEvent(h->s_front, h->ev_start, 0));
        uint32_t k = 0, gk = 0, gsub = 0, link_head = 0;  // chunk index, gathered chunks queued on the link / handed to the host threads, first chunk whose copy may still be on the wire
        uint64_t h2d_bytes = 0;
        std::vector<uint64_t>& clo = h->chunk_lo; std::vector<uint64_t>& chi = h->chunk_hi; std::vector<int8_t>& cbuf = h->chunk_buf;
        if (!iq_dev) {
            h->gather_ms = 0.0;
            clo.assign(nchunks, 0); chi.assign(nchunks, 0); cbuf.assign(nchunks, -1);          // span of every chunk in the capture; pinned buffer of a gathered chunk (-1: sent as it is)
            if (!dec || mix) for (uint32_t c = 0; c < nchunks; c++) {
                const uint32_t f0 = c * chunk, f1 = f0 + chunk < nframes ? f0 + chunk : nframes; uint64_t lo = ~0ull, hi = 0;
                for (uint32_t i = f0; i < f1; i++) { if (offh[i] < lo) lo = offh[i]; if (offh[i] + lenh[i] > hi) hi = offh[i] + lenh[i]; }
                clo[c] = lo; chi[c] = hi;
            }
        }
        struct InFlight { DecimPool* p = nullptr; bool on = false; ~InFlight() { if (p && on) p->wait(); } } inflight;   // no return while the host threads still read the caller's capture
        inflight.p = h->pool;
        // Decide how chunk c travels and, if it is to be gathered, hand it to the host threads now: the caller then queues the previous
        // chunk's copies and kernels while they work.  `ahead` = bytes of the chunk that is about to be queued in front of it.
        auto plan = [&](const uint32_t c, const uint64_t ahead) -> int {
            const uint32_t f0 = c * chunk, f1 = f0 + chunk < nframes ? f0 + chunk : nframes;
            bool gather = dec;
            if (dec && mix == 2u) gather = (c & 1u) != 0u;
            else if (dec && mix) {
                // bytes still queued on the link: copies whose end event has not fired.  Two consecutive ends also give the link rate.
                uint64_t pend = ahead;
                for (uint32_t i = link_head; i + 1 < c; i++) {              // chunks 0 .. c-2 are queued; c-1 is `ahead`
                    const cudaError_t q = cudaEventQuery(h->ev_link[i]);
                    if (q == cudaSuccess) {
                        if (i == link_head) {
                            float ms = 0.f;
                            if (i > 0 && cudaEventElapsedTime(&ms, h->ev_link[i - 1], h->ev_link[i]) == cudaSuccess && ms > 0.f) {
                                const double r = (double)h->link_bytes[i] / ms;
                                h->link_bpms = r > h->link_bpms ? r : 0.95 * h->link_bpms + 0.05 * r;   // a gap before the copy only lowers r
                            }
                            link_head++;
                        }
                    } else if (q == cudaErrorNotReady) { (void)cudaGetLastError(); pend += h->link_bytes[i]; }
                    else return h->fail(SB200_E_CUDA, "cudaEventQuery", q);
                }
                const double pend_ms = (double)pend / h->link_bpms;
                const double gather_est = h->gather_ms_per_sample * (double)(chi[c] - clo[c]);
                // a gather whose copy would reach the link after it has run dry costs link time: send the chunk as it is instead.
                // Not measured yet: the first chunk goes as it is (the link is idle anyway), the second is gathered and gives the estimate
                gather = h->gather_ms_per_sample > 0.0 ? pend_ms >= gather_est : c != 0u;
            }
            if (!gather) return SB200_OK;
            const int hb = (int)(gsub % 4u);
            // pinned buffer hb is free once its last copy has crossed the link: the gathered chunk four back, or one of an earlier call that
            // returned with its copies still queued (an event never recorded counts as complete)
            CK(cudaEventSynchronize(h->ev_hfree[hb]));
            DecimPool::Job j{(const uint32_t*)iq, offh.data(), lenh.data(), doffh.data(), f0, f1, (uint32_t*)h->hstage[hb]};
            h->pool->submit(j); inflight.on = true;
            cbuf[c] = (int8_t)hb; gsub++;
            return SB200_OK;
        };
        if (!iq_dev) { const int rc = plan(0, 0); if (rc != SB200_OK) return rc; }
        for (uint32_t f0 = 0; f0 < nframes; f0 += chunk, k++) {
            const uint32_t f1 = f0 + chunk < nframes ? f0 + chunk : nframes; const int b = k & 1;
            const uint32_t* base = (const uint32_t*)iq;
            const uint64_t* d_off_k = d_off; uint32_t sh_k = 1u;
            if (!iq_dev) {
                const bool gathered = cbuf[k] >= 0;
                if (gathered) {                              // the host threads finish this chunk; its cost per sample feeds the next decisions
                    const double gms = h->pool->wait(); inflight.on = false;
                    h->gather_ms += gms;
                    const double per = gms / (double)(2u * (doffh[f1] - doffh[f0]) + 1u);
                    h->gather_ms_per_sample = h->gather_ms_per_sample > 0.0 ? 0.75 * h->gather_ms_per_sample + 0.25 * per : per;
                }
                h->link_bytes[k] = gathered ? (doffh[f1] - doffh[f0]) * 4ull : (chi[k] - clo[k]) * 4ull;
                if (k + 1 < nchunks) { const int rc = plan(k + 1, h->link_bytes[k]); if (rc != SB200_OK) return rc; }
                if (k >= 2) CK(cudaStreamWaitEvent(h->s_copy, h->ev_front[b], 0));            // device buffer b is free once chunk k-2's front end has read it
                if (gathered) {
                    CK(cudaMemcpyAsync(h->stage[b].p, h->hstage[cbuf[k]], h->link_bytes[k], cudaMemcpyHostToDevice, h->s_copy));
                    CK(cudaEventRecord(h->ev_hfree[cbuf[k]], h->s_copy));
                    base = (const uint32_t*)h->stage[b].p - doffh[f0]; d_off_k = d_off_dec; sh_k = 0u; gk++;
                } else {
                    CK(cudaMemcpyAsync(h->stage[b].p, (const uint32_t*)iq + clo[k], h->link_bytes[k], cudaMemcpyHostToDevice, h->s_copy));
                    base = (const uint32_t*)h->stage[b].p - clo[k];
                }
                h2d_bytes += h->link_bytes[k];
                CK(cudaEventRecord(h->ev_link[k], h->s_copy));
                CK(cudaEventRecord(h->ev_h2d[b], h->s_copy));
                CK(cudaStreamWaitEvent(h->s_front, h->ev_h2d[b], 0));
            }
            int rc = launch_chunk(h, base, d_off_k, d_len, f0, f1, soft_stride, row, h->s_front, st, h->ev_front[b], taps, false, nullptr, k, sh_k);
            if (rc != SB200_OK) return rc;
            // results of this chunk go back while the next chunks are still coming in (PCIe is full duplex): only the last chunk's
            // device-to-host copy is left exposed at the end of the call
            const uint32_t n = f1 - f0;
            k_pack_results<<<(n + 255) / 256, 256, 0, st>>>((const FrameInfo*)h->info.p + f0, (const uint32_t*)h->status.p + f0, (const uint32_t*)h->crc.p + f0, n, d_res_all + f0);
            h->launches += 1;
            if (out_bytes && out_stride && !out_dev_all) {
                const size_t w = out_stride < row ? out_stride : row;
                CK(cudaMemcpy2DAsync(out_bytes + (size_t)f0 * out_stride, out_stride, (const uint8_t*)h->out.p + (size_t)f0 * row, row, w, n, cudaMemcpyDeviceToHost, st));
            }
            if (!res_dev_all) CK(cudaMemcpyAsync(res + f0, d_res_all + f0, n * sizeof(sb200_frame_result), cudaMemcpyDeviceToHost, st));
        }
        if (!iq_dev) { h->last_h2d_bytes = h2d_bytes; h->last_gathered_chunks = gk; h->last_chunks = k; }
        if (dec && getenv("SB200_TRACE")) fprintf(stderr, "[sb200] rx11a host_decimate: %u chunks (%u gathered, %u sent as they are), host gather %.2f ms in total (%u threads), link estimate %.1f GB/s, %.1f MB copied\n", k, gk, k - gk, h->gather_ms, h->host_decimate, h->link_bpms / 1e6, h2d_bytes / 1e6);
        Returns none;                                   // everything that goes to the host was already queued per chunk
        const int rc = finish_call(h, st, none, 0, 0);
        if (rc != SB200_OK) return rc;
        if (out_bytes && out_stride && out_dev_all) { const size_t w = out_stride < row ? out_stride : row; CK(cudaMemcpy2DAsync(out_bytes, out_stride, h->out.p, row, w, nframes, cudaMemcpyDeviceToDevice, st)); }
        if ((out_bytes && out_stride && !out_dev_all) || !res_dev_all) CK(cudaStreamSynchronize(st));
        return SB200_OK;
    }
    k_pack_results<<<(nframes + 255) / 256, 256, 0, st>>>((const FrameInfo*)h->info.p, (const uint32_t*)h->status.p, (const uint32_t*)h->crc.p, nframes, d_res_all);
    h->launches += 1;
    CK(cudaEventRecord(h->evk[4], st));
    Returns ret;
    if (out_bytes && out_stride) ret.bind2d(out_bytes, out_stride, h->out.p, row, out_stride < row ? out_stride : row, nframes);
    if (!res_dev_all) ret.copy(res, d_res_all, nframes * sizeof(sb200_frame_result));
    if (soft_host) ret.bind2d(soft_host, soft_host_stride, h->soft.p, soft_stride, soft_host_stride < soft_stride ? soft_host_stride : soft_stride, nframes);
    return finish_call(h, st, ret, 4, 0);
}

// Many continuous captures at once.  Every pass decodes the next frame of every capture that still has samples (one slot per
// capture, from its cursor to its end, with its own carried DC), so the device sees a full batch per pass and the number of
// passes is the largest number of frames in any one capture.
// Page-locked host memory for capture buffers: what the reference's user-mode extension maps for a radio (SoraURadioMapRxSampleBuf,
// kernel/core/inc/_user_mode_ext.h:100) is DMA-able memory too.  Captures handed to the engine from such a buffer cross PCIe without a staging copy.
extern "C" void* sb200_host_alloc(size_t bytes) { void* p = nullptr; if (bytes == 0 || cudaHostAlloc(&p, bytes, cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return nullptr; } return p; }
extern "C" void sb200_host_free(void* p) { if (p) cudaFreeHost(p); }

// Capture table of a stream call: tables and results in host memory, every capture inside the samples, frame counts zeroed on the way.
static int stream_table(sb200_handle* h, const uint64_t* stream_off, const uint32_t* stream_len, uint32_t nstreams, uint64_t iq_total,
                        const void* res, const void* out_bytes, uint32_t* nframes_out, bool antennas_apart) {
    if (is_device_ptr(res) || (out_bytes && is_device_ptr(out_bytes)) || is_device_ptr(stream_off) || is_device_ptr(stream_len) || is_device_ptr(nframes_out))
        return h->fail(SB200_E_INVALID, "stream mode takes its tables and returns its results in host memory");
    if (antennas_apart) return h->fail(SB200_E_INVALID, "both antenna buffers must live on the same side");
    for (uint32_t s = 0; s < nstreams; s++) { nframes_out[s] = 0; if (!in_range(stream_off[s], stream_len[s], iq_total)) return h->fail(SB200_E_INVALID, "capture exceeds iq_total_samples"); }
    return SB200_OK;
}

extern "C" int sb200_rx11a_streams(sb200_handle* h, const int16_t* iq, uint64_t iq_total, const uint64_t* stream_off, const uint32_t* stream_len,
                                   uint32_t nstreams, uint32_t max_frames, uint8_t* out_bytes, uint32_t out_stride, sb200_frame_result* res,
                                   uint32_t* sample_index, uint32_t* nframes_out, void* cuda_stream) {
    if (!h || !iq || !stream_off || !stream_len || !res || !nframes_out) return h ? h->fail(SB200_E_INVALID, "null argument") : SB200_E_INVALID;
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin());          // results in host memory: the call synchronises anyway
    {   const int rc = stream_table(h, stream_off, stream_len, nstreams, iq_total, res, out_bytes, nframes_out, false); if (rc != SB200_OK) return rc; }
    if (nstreams == 0 || max_frames == 0) return SB200_OK;
    const int16_t* d_iq = iq;
    if (!is_device_ptr(iq)) {                           // host captures: only the ranges the streams name travel (they may be islands in a large arena)
        CK(h->iq.need(iq_total * 4ull));
        for (uint32_t s = 0; s < nstreams; s++) if (stream_len[s]) CK(cudaMemcpyAsync((char*)h->iq.p + stream_off[s] * 4ull, iq + 2ull * stream_off[s], stream_len[s] * 4ull, cudaMemcpyHostToDevice, st));
        d_iq = (const int16_t*)h->iq.p;
    }
    // Phase 1, scout: carrier sense + SIGNAL only, one pass per event of the busiest capture; positions, DC estimates and the event list stay on
    // the device, the host only reads a "captures still live" counter every few passes.  Where a frame ends depends on its header alone, so the
    // expensive part (data symbols, Viterbi) need not sit inside this serial chain.
    const uint32_t n = nstreams;
    const bool trace = getenv("SB200_TRACE") != nullptr; const auto t_begin = std::chrono::steady_clock::now();
    std::vector<uint64_t> off0(n); std::vector<uint32_t> len0(n);
    for (uint32_t s = 0; s < n; s++) { off0[s] = stream_off[s]; len0[s] = stream_len[s] >= 28u ? stream_len[s] : 0u; }
    CK(h->soff.need(n * 8ull)); CK(h->slen.need(n * 4ull)); CK(h->dcbuf.need(n * sizeof(int2))); CK(h->spos.need(n * 4ull)); CK(h->snev.need(n * 4ull + 64));
    CK(h->sev.need((size_t)n * max_frames * sizeof(StreamEvent))); CK(h->info.need(n * sizeof(FrameInfo)));
    CK(cudaMemcpyAsync(h->soff.p, off0.data(), n * 8ull, cudaMemcpyHostToDevice, st)); CK(cudaMemcpyAsync(h->slen.p, len0.data(), n * 4ull, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(h->dcbuf.p, 0, n * sizeof(int2), st)); CK(cudaMemsetAsync(h->spos.p, 0, n * 4ull, st)); CK(cudaMemsetAsync(h->snev.p, 0, n * 4ull + 64, st));
    uint32_t* d_live = (uint32_t*)h->snev.p + n;                      // one counter per pass of a round (<= 16)
    FrontTaps hdr{}; hdr.hdr_only = 1;
    const uint32_t ROUND = 8;
    for (uint32_t done_passes = 0; done_passes < max_frames;) {
        CK(cudaMemsetAsync(d_live, 0, ROUND * 4ull, st));
        uint32_t k = 0;
        for (; k < ROUND && done_passes + k < max_frames; k++) {
            k_sync11a<<<(n + 127) / 128, 128, 0, st>>>((const uint32_t*)d_iq, (const uint64_t*)h->soff.p, (const uint32_t*)h->slen.p, n, h->cca_thr, h->T, (FrameInfo*)h->info.p, (const int2*)h->dcbuf.p, 1u, 0u);
            k_front11a<0><<<(n + SB_FRONT_WARPS - 1) / SB_FRONT_WARPS, 32 * SB_FRONT_WARPS, 0, st>>>((const uint32_t*)d_iq, (const uint64_t*)h->soff.p, (const uint32_t*)h->slen.p, n, h->T, (FrameInfo*)h->info.p, nullptr, 0, h->inv_deint, hdr, 1u, 0u);
            k_stream_advance<<<(n + 127) / 128, 128, 0, st>>>((const FrameInfo*)h->info.p, n, (uint64_t*)h->soff.p, (uint32_t*)h->slen.p, (int2*)h->dcbuf.p, (uint32_t*)h->spos.p, (uint32_t*)h->snev.p, max_frames, (StreamEvent*)h->sev.p, d_live + k);
            h->launches += 3;
        }
        CK(cudaGetLastError());
        uint32_t live[16]; CK(cudaMemcpyAsync(live, d_live, ROUND * 4ull, cudaMemcpyDeviceToHost, st)); CK(cudaStreamSynchronize(st));
        done_passes += k;
        if (live[k - 1] == 0) break;
    }
    const auto t_scout = std::chrono::steady_clock::now();
    // Phase 2: every event is an independent slot (start of the search, length up to the block after its last symbol, the DC estimate the search
    // started with): one batch through the ordinary pipeline.
    std::vector<uint32_t> nev(n); CK(cudaMemcpy(nev.data(), h->snev.p, n * 4ull, cudaMemcpyDeviceToHost));
    size_t E = 0; for (uint32_t s = 0; s < n; s++) E += nev[s];
    if (E == 0) return SB200_OK;
    std::vector<StreamEvent> ev((size_t)n * max_frames);
    CK(cudaMemcpy(ev.data(), h->sev.p, ev.size() * sizeof(StreamEvent), cudaMemcpyDeviceToHost));
    std::vector<uint64_t> off(E); std::vector<uint32_t> len(E); std::vector<int2> dcv(E); std::vector<sb200_frame_result> r(E);
    const uint32_t row = out_bytes ? (out_stride < 2560u ? out_stride : 2560u) : 0u;
    std::vector<uint8_t> bytes((size_t)E * row);
    {   size_t e = 0;
        for (uint32_t s = 0; s < n; s++) for (uint32_t j = 0; j < nev[s]; j++, e++) { const StreamEvent& v = ev[(size_t)s * max_frames + j]; off[e] = v.off; len[e] = v.len; dcv[e] = v.dc; } }
    CK(h->dcbuf.need(E * sizeof(int2))); CK(cudaMemcpyAsync(h->dcbuf.p, dcv.data(), E * sizeof(int2), cudaMemcpyHostToDevice, st));
    FrontTaps taps{};
    int rc = rx11a_run(h, d_iq, iq_total, off.data(), len.data(), (uint32_t)E, row ? bytes.data() : nullptr, row, r.data(), st, taps, nullptr, 0, (const int2*)h->dcbuf.p, true);
    if (rc != SB200_OK) return rc;
    {   size_t e = 0;
        for (uint32_t s = 0; s < n; s++) {
            for (uint32_t j = 0; j < nev[s]; j++, e++) {
                const size_t slot = (size_t)s * max_frames + j;
                if (r[e].status == SB200_FRAME_NONE) return h->fail(SB200_E_CUDA, "internal: stream scout and batch decode disagree about a frame");
                res[slot] = r[e];
                if (sample_index) sample_index[slot] = ev[slot].pos_after;
                if (row) memcpy(out_bytes + slot * out_stride, bytes.data() + e * row, row);
            }
            nframes_out[s] = nev[s];
        } }
    if (trace) { const auto t_end = std::chrono::steady_clock::now();
        fprintf(stderr, "[sb200] rx11a_streams: %u captures, %zu events, %llu samples: scout %.3f ms, batch %.3f ms\n", n, E, (unsigned long long)iq_total,
                std::chrono::duration<double, std::milli>(t_scout - t_begin).count(), std::chrono::duration<double, std::milli>(t_end - t_scout).count()); }
    return rc;
}

// One continuous capture: frames are found one after another exactly like RxThread does (fb11a_demod.cpp:29-81): after every
// event the graph is flushed and reset, the source continues with the next 28-sample block, and only the DC estimate
// (CF_VecDC) survives.  Each frame is one pass of the batch pipeline over the remaining samples with that DC.
extern "C" int sb200_rx11a_stream(sb200_handle* h, const int16_t* iq, uint64_t nsamples, uint32_t max_frames, uint8_t* out_bytes, uint32_t out_stride,
                                  sb200_frame_result* res, uint32_t* sample_index, uint32_t* nframes_out, void* cuda_stream) {
    if (!h || !nframes_out) return h ? h->fail(SB200_E_INVALID, "null argument") : SB200_E_INVALID;
    if (nsamples > 0xFFFFFF00ull) return h->fail(SB200_E_INVALID, "capture longer than 2^32 samples: split it");
    const uint64_t off = 0; const uint32_t len = (uint32_t)nsamples;
    return sb200_rx11a_streams(h, iq, nsamples, &off, &len, 1, max_frames, out_bytes, out_stride, res, sample_index, nframes_out, cuda_stream);
}

// One launch of k_channelize (fir_kernels.cuh) over device buffers, between ev0 and the caller's finish_call.  Outputs per thread from D;
// channels split into groups (the input then read once per group) only as far as needed for four CTAs per multiprocessor.
template <int J>
static int channelize_launch_j(sb200_handle* h, cudaStream_t st, dim3 grid, const uint32_t* d_in, uint64_t n_in, const ChChannels& ch, uint32_t cpg,
                               uint32_t D, const ChTaps& T, uint32_t* d_out, uint64_t stride, uint64_t n_out) {
    if (!(h->ch_smem_set & (1u << J))) {
        CK(cudaFuncSetAttribute(k_channelize<J>, cudaFuncAttributeMaxDynamicSharedMemorySize, SB_CH_SMEM));
        h->ch_smem_set |= 1u << J;
    }
    CK(cudaEventRecord(h->ev0, st));
    k_channelize<J><<<grid, SB_FIR_THREADS, SB_CH_SMEM, st>>>(d_in, n_in, (const uint32_t*)h->nco.p, ch, cpg, D, T, d_out, stride, n_out);
    return SB200_OK;
}
static int channelize_launch(sb200_handle* h, cudaStream_t st, const uint32_t* d_in, uint64_t n_in, const ChChannels& ch, uint32_t D, const ChTaps& T,
                             uint32_t* d_out, uint64_t stride, uint64_t n_out) {
    if (!h->sms) CK(cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, h->device));
    const uint64_t tiles = (n_in + SB_FIR_TILE - 1) / SB_FIR_TILE;
    uint32_t groups = 1;
    while (groups < ch.n && tiles * groups < 4ull * (uint64_t)h->sms) groups++;
    const uint32_t cpg = (ch.n + groups - 1) / groups; groups = (ch.n + cpg - 1) / cpg;
    const dim3 grid((unsigned)tiles, groups);
    const uint32_t need = ((SB_FIR_TILE + D - 1) / D + SB_FIR_THREADS - 1) / SB_FIR_THREADS;     // outputs per thread of a tile
    if (need <= 1) return channelize_launch_j<1>(h, st, grid, d_in, n_in, ch, cpg, D, T, d_out, stride, n_out);
    if (need <= 2) return channelize_launch_j<2>(h, st, grid, d_in, n_in, ch, cpg, D, T, d_out, stride, n_out);
    if (need <= 4) return channelize_launch_j<4>(h, st, grid, d_in, n_in, ch, cpg, D, T, d_out, stride, n_out);
    if (need <= 8) return channelize_launch_j<8>(h, st, grid, d_in, n_in, ch, cpg, D, T, d_out, stride, n_out);
    return channelize_launch_j<16>(h, st, grid, d_in, n_in, ch, cpg, D, T, d_out, stride, n_out);
}

// 2:1 anti-alias FIR decimator (k_fir_decimate2): channel (0, 0) of the channelizer's arithmetic with D = 2,
// out[m] = sat16((sum_k taps[k] x[2m + k - (ntaps-1)/2] + 2^14) >> 15), zero outside the buffer.  taps == NULL selects the built-in 31-tap half-band low-pass (equiripple: +-0.05 dB to 8.3 MHz of a 40 Msps
// capture, 50 dB down beyond 11.7 MHz).
static const int16_t kHalfBand31[31] = {-121, 0, 209, 0, -381, 0, 644, 0, -1056, 0, 1759, 0, -3278, 0, 10391, 16434, 10391, 0, -3278, 0, 1759, 0, -1056, 0, 644, 0, -381, 0, 209, 0, -121};   // sum 32768 (unit DC gain)
extern "C" int sb200_fir_decimate2(sb200_handle* h, const int16_t* iq, uint64_t n_in, const int16_t* taps, uint32_t ntaps, int16_t* out, void* cuda_stream) {
    if (!h || !iq || !out) return h ? h->fail(SB200_E_INVALID, "null argument") : SB200_E_INVALID;
    if (!taps) { taps = kHalfBand31; ntaps = 31; }
    if ((ntaps & 1u) == 0 || ntaps > SB_FIR_MAXTAPS) return h->fail(SB200_E_INVALID, "ntaps must be odd and at most 63");
    if (n_in == 0) return SB200_OK;
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin()); call.reads(iq);
    const uint64_t n_out = (n_in + 1) / 2;
    const bool in_dev = is_device_ptr(iq);
    if (in_dev && ((uintptr_t)iq & 15u)) return h->fail(SB200_E_INVALID, "device input must be 16-byte aligned");
    const uint32_t* d_in; uint32_t* d_out; Returns ret;
    CK(to_device(h->iq, (const uint32_t*)iq, in_dev, n_in * 4ull, st, &d_in, 16));
    CK(ret.bind(h->iq40, (uint32_t*)out, n_out * 4ull, &d_out, 16));
    FirTaps T; memset(&T, 0, sizeof T); T.n = ntaps; for (uint32_t i = 0; i < ntaps; i++) T.t[i] = taps[i];
    CK(cudaEventRecord(h->ev0, st));
    k_fir_decimate2<<<(unsigned)((n_in + SB_FIR_TILE - 1) / SB_FIR_TILE), SB_FIR_THREADS, 0, st>>>(d_in, n_in, T, d_out, n_out);
    return finish_call(h, st, ret, 0, 1);
}

// Wideband channelizer (fir_kernels.cuh): every channel shifted by its NCO, filtered and decimated by `decim`; channel c in row c of `out`.
extern "C" int sb200_channelize(sb200_handle* h, const int16_t* iq, uint64_t n_in, const sb200_ddc_channel* channels, uint32_t nchannels, uint32_t decim,
                                const int16_t* taps, uint32_t ntaps, int16_t* out, uint64_t out_stride, void* cuda_stream) {
    if (!h) return SB200_E_INVALID;
    if (!iq || !channels || !taps || !out) return h->fail(SB200_E_INVALID, "null argument");
    if (nchannels < 1 || nchannels > SB_CH_MAXCH) return h->fail(SB200_E_INVALID, "nchannels must be 1 .. 16");
    if (decim < 1 || decim > SB_CH_MAXDECIM) return h->fail(SB200_E_INVALID, "decim must be 1 .. 16");
    if ((ntaps & 1u) == 0 || ntaps > SB_CH_MAXTAPS) return h->fail(SB200_E_INVALID, "ntaps must be odd and at most 255");
    uint32_t asum = 0; for (uint32_t i = 0; i < ntaps; i++) asum += (uint32_t)abs((int)taps[i]);
    if (asum > 65535u) return h->fail(SB200_E_INVALID, "sum of |taps| must be at most 65535 (the int32 accumulator must not wrap)");
    if (n_in > (1ull << 40)) return h->fail(SB200_E_INVALID, "n_in_samples must be at most 2^40");
    const uint64_t n_out = (n_in + decim - 1) / decim;
    if (out_stride < n_out || (out_stride & 3u) || out_stride > (1ull << 40)) return h->fail(SB200_E_INVALID, "out_stride must be at least ceil(n_in / decim), at most 2^40 and a multiple of 4");
    if (n_in == 0) return SB200_OK;
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    const bool in_dev = is_device_ptr(iq), out_dev = is_device_ptr(out);
    if ((in_dev && ((uintptr_t)iq & 15u)) || (out_dev && ((uintptr_t)out & 15u))) return h->fail(SB200_E_INVALID, "device input and output must be 16-byte aligned");
    CallScope call(h, st); CK(call.begin()); call.reads(iq);
    if (!h->nco.p) {                                   // (C, S) = (rint(2^14 cos 2 pi i / 4096), rint(2^14 sin 2 pi i / 4096)), packed like cs16
        std::vector<uint32_t> t(SB_CH_NCO);
        for (int i = 0; i < SB_CH_NCO; i++) { const double a = 2.0 * M_PI * i / 4096.0; t[i] = pack(mk((int)nearbyint(16384.0 * cos(a)), (int)nearbyint(16384.0 * sin(a)))); }
        cudaError_t e = h->nco.need(SB_CH_NCO * 4);
        if (e == cudaSuccess) e = cudaMemcpy(h->nco.p, t.data(), SB_CH_NCO * 4, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaDeviceSynchronize();   // landed before a kernel on a non-blocking stream reads it (TableArena::upload)
        if (e != cudaSuccess) { h->nco.release(); return h->fail(SB200_E_CUDA, "NCO table upload", e); }
    }
    const uint32_t* d_in; uint32_t* d_out = (uint32_t*)out; uint64_t d_stride = out_stride; Returns ret;
    CK(to_device(h->iq, (const uint32_t*)iq, in_dev, n_in * 4ull, st, &d_in, 16));
    if (!out_dev) {                                    // rows n_out (rounded to 4) apart in the workspace, copied into the caller's rows
        d_stride = (n_out + 3u) & ~3ull; CK(h->iq40.need(nchannels * d_stride * 4ull)); d_out = (uint32_t*)h->iq40.p;
        ret.bind2d(out, out_stride * 4ull, d_out, d_stride * 4ull, n_out * 4ull, nchannels);
    }
    ChTaps T; memset(&T, 0, sizeof T); T.n = ntaps; for (uint32_t i = 0; i < ntaps; i++) T.t[i] = taps[i];
    ChChannels ch; memset(&ch, 0, sizeof ch); ch.n = nchannels;
    for (uint32_t i = 0; i < nchannels; i++) { ch.inc[i] = channels[i].phase_inc; ch.phase0[i] = channels[i].phase0; }
    const int rc = channelize_launch(h, st, d_in, n_in, ch, decim, T, d_out, d_stride, n_out);
    return rc != SB200_OK ? rc : finish_call(h, st, ret, 0, 1);
}

extern "C" int sb200_rx11a_batch_ex(sb200_handle* h, const int16_t* iq, uint64_t iq_total, const uint64_t* frame_off, const uint32_t* frame_len,
                                    uint32_t nframes, uint32_t sample_rate_mhz, uint8_t* out_bytes, uint32_t out_stride,
                                    sb200_frame_result* res, void* cuda_stream) {
    if (!h) return SB200_E_INVALID;
    if (sample_rate_mhz == 40) return sb200_rx11a_batch(h, iq, iq_total, frame_off, frame_len, nframes, out_bytes, out_stride, res, cuda_stream);
    if (sample_rate_mhz == 20) {                        // already decimated (sb200_fir_decimate2, or a 20 Msps front end): what TDownSample2 would hand on
        FrontTaps taps{};
        return rx11a_run(h, iq, iq_total, frame_off, frame_len, nframes, out_bytes, out_stride, res, (cudaStream_t)cuda_stream, taps, nullptr, 0, nullptr, true, true);
    }
    if (sample_rate_mhz != 44) return h->fail(SB200_E_INVALID, "sample_rate_mhz must be 20, 40 or 44");
    if (!iq || !frame_off || !frame_len || !res) return h->fail(SB200_E_INVALID, "null argument");
    if (nframes == 0) return SB200_OK;
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin()); call.reads(iq);
    // slot table on the host (sizing) and on the device (kernel)
    FrameTable ft(frame_off, frame_len, nframes);
    const bool iq_dev = is_device_ptr(iq);
    uint32_t max40 = 28;
    const int rc = ft.load(h, st, iq_total, [&](uint32_t i, bool inside) {
        if (!inside) return h->fail(SB200_E_INVALID, "slot exceeds iq_total_samples");
        const uint32_t n40 = resampled_len_40(ft.lenh[i]); if (n40 > max40) max40 = n40;
        return SB200_OK;
    });
    if (rc != SB200_OK) return rc;
    const uint64_t stride40 = ((uint64_t)max40 + 3ull) & ~3ull;
    const uint32_t* d_iq; const uint64_t* d_off; const uint32_t* d_len;
    CK(to_device(h->iq, (const uint32_t*)iq, iq_dev, iq_total * 4ull, st, &d_iq));
    CK(ft.upload(h->off, h->len, st, &d_off, &d_len));
    CK(h->iq40.need(nframes * stride40 * 4ull)); CK(h->off40.need(nframes * 8ull)); CK(h->len40.need(nframes * 4ull));
    dim3 grid(nframes, (unsigned)((max40 + 255) / 256 > 64 ? 64 : (max40 + 255) / 256));   // slots on x: the y extent stops at 65535
    k_resample_44_40<<<grid, 256, 0, st>>>(d_iq, d_off, d_len, nframes, (uint32_t*)h->iq40.p, stride40, (uint64_t*)h->off40.p, (uint32_t*)h->len40.p);
    h->launches += 1;
    CK(cudaGetLastError());
    return sb200_rx11a_batch(h, (const int16_t*)h->iq40.p, nframes * stride40, (const uint64_t*)h->off40.p, (const uint32_t*)h->len40.p, nframes,
                             out_bytes, out_stride, res, cuda_stream);
}

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
    if (cr23 && h->use_v2) h->launches -= 1;           // the quad path has always counted two Viterbi launches here
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
    if (!strcmp(name, "host_decimate_mix")) { if (value > 2) return h->fail(SB200_E_INVALID, "host_decimate_mix: 0, 1 or 2"); h->host_mix = (uint32_t)value; h->gather_ms_per_sample = 0.0; return SB200_OK; }
    if (!strcmp(name, "slot_table_immutable")) { h->tab_immutable = value != 0; h->tab_off = nullptr; return SB200_OK; }
    if (!strcmp(name, "ht_mcs_limit")) { if (value < 9 || value > 15) return h->fail(SB200_E_INVALID, "ht_mcs_limit is the first 802.11n MCS index refused: 9 .. 15 (11 = the reference's parser, 15 = MCS 8..14)"); h->ht_mcs_limit = (uint32_t)value; return SB200_OK; }
    return h->fail(SB200_E_INVALID, "unknown option");
}

extern "C" int sb200_rx11a_batch(sb200_handle* h, const int16_t* iq, uint64_t iq_total_samples, const uint64_t* frame_off,
                                 const uint32_t* frame_len, uint32_t nframes, uint8_t* out_bytes, uint32_t out_stride,
                                 sb200_frame_result* res, void* cuda_stream) {
    FrontTaps taps{};
    return rx11a_run(h, iq, iq_total_samples, frame_off, frame_len, nframes, out_bytes, out_stride, res, (cudaStream_t)cuda_stream, taps, nullptr, 0);
}

extern "C" int sb200_rx11a_taps(sb200_handle* h, const int16_t* iq, uint64_t iq_total_samples, const uint64_t* frame_off,
                                const uint32_t* frame_len, uint32_t nframes, uint32_t max_sym, sb200_frame_result* res,
                                int16_t* freq_coeffs, int16_t* chan_coeffs, int16_t* fft_out, int16_t* equalized, int16_t* tracked,
                                uint8_t* soft, uint64_t soft_stride) {
    if (!h) return SB200_E_INVALID;
    CK(cudaSetDevice(h->device));
    const size_t c = (size_t)nframes * 64 * 4, s = (size_t)nframes * max_sym * 64 * 4, s4 = s ? s : 4;
    const size_t size[5] = {c, c, s4, s4, s4}, back[5] = {c, c, s, s, s};
    void* const dst[5] = {freq_coeffs, chan_coeffs, s ? fft_out : nullptr, s ? equalized : nullptr, s ? tracked : nullptr};
    return run_with_taps(h, size, dst, back, [&] {
        FrontTaps taps{};
        taps.freq_coeffs = (uint32_t*)h->taps[0].p; taps.chan_coeffs = (uint32_t*)h->taps[1].p;
        taps.fft_out = (uint32_t*)h->taps[2].p; taps.equalized = (uint32_t*)h->taps[3].p; taps.tracked = (uint32_t*)h->taps[4].p; taps.max_sym = max_sym;
        const int rc = rx11a_run(h, iq, iq_total_samples, frame_off, frame_len, nframes, nullptr, 0, res, 0, taps, soft, soft_stride);
        if (rc != SB200_OK) return rc;
        CK(cudaDeviceSynchronize());
        return SB200_OK;
    });
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
