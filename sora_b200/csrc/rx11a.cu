// sora_b200 — 802.11a receive (rx11a_kernels.cuh): the batch receiver, with HostPipe, the handle's pipeline of large calls (three streams,
// the pinned slabs and host threads of option host_decimate), the continuous-capture scout and the 44 Msps and stage-tap entry points.
#include "handle.cuh"
#include "rx11a_kernels.cuh"
#include <stdio.h>
#include <stdlib.h>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <new>
#include <thread>
#include <emmintrin.h>

namespace {

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

} // namespace

// ---- the chunked pipeline of the batch receiver ----------------------------------------------------------------------------------------
// The 802.11a graph keeps samples 0 and 2 of every 4 (samples.hpp:27-49).  With option "host_decimate" = T > 0, T host threads gather the
// even samples of every slot of a host-resident chunk into pinned memory and only those cross PCIe (half the bytes); the kernels read the
// packed copy with stride 1 (sh = 0), so the same samples reach the same arithmetic.
namespace sb { void gather_even(const uint32_t* src, uint32_t n2, uint32_t* dst); }      // host_gather.cpp: dst[j] = src[2 j], streaming stores, SSE2 / AVX-512 chosen at run time
struct DecimPool {
    // n worker threads; submit() hands them one chunk and returns, wait() blocks until it is gathered: the caller queues the previous chunk's
    // copies and kernels in between, so the host cores never wait for the launch path (and the launch path never waits for them).
    struct Job { const uint32_t* iq; const uint64_t* off; const uint32_t* len; const uint64_t* doff; uint32_t f0, f1; uint32_t* dst; };
    std::vector<std::thread> th; std::mutex m; std::condition_variable cv, cv_done;
    Job job{}; uint64_t gen = 0; int pending = 0; bool stop = false; int n = 0;
    std::chrono::steady_clock::time_point t_submit; double last_ms = 0.0;   // wall time from submit() to the last worker's end
    explicit DecimPool(int nthreads) : n(nthreads < 1 ? 1 : nthreads) {
        for (int w = 0; w < n; w++) th.emplace_back([this, w]() {
            uint64_t seen = 0;
            for (;;) {
                Job j;
                { std::unique_lock<std::mutex> l(m); cv.wait(l, [&] { return stop || gen != seen; }); if (stop) return; seen = gen; j = job; }
                const uint64_t cnt = j.f1 - j.f0; const uint32_t a = j.f0 + (uint32_t)(cnt * w / n), b = j.f0 + (uint32_t)(cnt * (w + 1) / n);   // this worker's slots
                for (uint32_t f = a; f < b; f++) sb::gather_even(j.iq + j.off[f], (j.len[f] + 1u) / 2u, j.dst + (j.doff[f] - j.doff[j.f0]));
                _mm_sfence();                           // streaming stores visible before the copy is queued
                { std::lock_guard<std::mutex> l(m);
                  if (--pending == 0) { last_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_submit).count(); cv_done.notify_all(); } }
            }
        });
    }
    void submit(const Job& j) {                         // one job in flight at a time: wait() first
        { std::lock_guard<std::mutex> l(m); job = j; gen++; pending = n; t_submit = std::chrono::steady_clock::now(); }
        cv.notify_all();
    }
    double wait() { std::unique_lock<std::mutex> l(m); cv_done.wait(l, [&] { return pending == 0; }); return last_ms; }   // at once when nothing is in flight
    ~DecimPool() {
        { std::lock_guard<std::mutex> l(m); stop = true; }
        cv.notify_all();
        for (auto& t : th) t.join();
    }
};

// One call of the batch receiver as rx11a_run has laid it out (d_res: where k_pack_results writes the results, `res` itself when res_dev).
struct Batch {
    const int16_t* iq; bool iq_dev; const uint64_t* d_off; const uint32_t* d_len; uint32_t nframes; uint64_t soft_stride, row; FrontTaps taps;
    cudaStream_t st; uint8_t* out_bytes; uint32_t out_stride; bool out_dev; sb200_frame_result* res; sb200_frame_result* d_res; bool res_dev;
};
// Where a launch finds the samples of slot f: from word base + off[f] on, every (1 << sh)-th word (sh = 1: a 40 Msps capture; 0: samples at
// 20 Msps), len[f] of them counted at 40 Msps (lsh = 0) or at 20 Msps (lsh = 1).  The DC estimate of slot f starts from dc[f] (null: zero).
struct Samples { const uint32_t* base; const uint64_t* off; uint32_t sh, lsh; const int2* dc; };

// Launch the decode kernels for slots [f0, f1) of `bt`, chunk `part` of the call, with their samples where `x` says: sync + front end on
// `sf`, the Viterbi on `sv` (sv waits for `front_done` when the streams differ); `timed` records evk[0..3].
static int launch_chunk(sb200_handle* h, const Batch& bt, const Samples& x, uint32_t f0, uint32_t f1, uint32_t part, cudaStream_t sf, cudaStream_t sv, cudaEvent_t front_done, bool timed) {
    const uint32_t n = f1 - f0;
    FrameInfo* d_info = (FrameInfo*)h->info.p + f0;
    uint8_t* d_soft = (uint8_t*)h->soft.p + (size_t)f0 * bt.soft_stride;
    uint8_t* d_out = (uint8_t*)h->out.p + (size_t)f0 * bt.row;
    uint32_t* d_status = (uint32_t*)h->status.p + f0; uint32_t* d_crc = (uint32_t*)h->crc.p + f0;
    if (timed) CK(cudaEventRecord(h->evk[0], sf));
    k_sync11a<<<(n + 127) / 128, 128, 0, sf>>>(x.base, x.off + f0, bt.d_len + f0, n, h->cca_thr, h->T, d_info, x.dc ? x.dc + f0 : nullptr, x.sh, x.lsh);
    if (timed) CK(cudaEventRecord(h->evk[1], sf));
    {   const dim3 g((n + SB_FRONT_SLOTS - 1) / SB_FRONT_SLOTS), b(32 * SB_FRONT_WARPS);
        if (h->front_stage == 2 && !h->front_smem_set) {
            CK(cudaFuncSetAttribute(k_front11a<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, SB_FRONT_STAGE_SMEM));
            h->front_smem_set = true;
        }
        const auto front = h->front_stage == 2 ? k_front11a<2> : h->front_stage == 1 ? k_front11a<1> : k_front11a<0>;
        front<<<g, b, h->front_stage == 2 ? SB_FRONT_STAGE_SMEM : 0, sf>>>(x.base, x.off + f0, bt.d_len + f0, n, h->T, d_info, d_soft, bt.soft_stride, h->inv_deint, bt.taps, x.sh, x.lsh); }
    if (timed) CK(cudaEventRecord(h->evk[2], sf));
    if (sv != sf) { CK(cudaEventRecord(front_done, sf)); CK(cudaStreamWaitEvent(sv, front_done, 0)); }
    h->launches += 2;
    VitJob job{}; job.depth = 256; job.lookahead = 24; job.raw = 0;
    static const int rates[3] = {CR_34, CR_12, CR_23};
    const int rc = viterbi_stage(h, n, sv, d_soft, bt.soft_stride, d_info, job, d_out, bt.row, d_status, d_crc, rates, 3, f0, part, h->vq_pad_smem);
    if (rc != SB200_OK) return rc;
    if (timed) CK(cudaEventRecord(h->evk[3], sv));
    return SB200_OK;
}

// The pipeline of large calls, one per handle: host->device copy of chunk k+1 (s_copy) | carrier sense + OFDM front end of chunk k+1
// (s_front) | Viterbi of chunk k (the caller's stream); the front end is latency bound and the Viterbi integer-issue bound, so they overlap
// well on the same SMs.  A host-resident chunk reaches one of two device buffers as its span of the capture or, with host_decimate, as the
// even samples of its slots, which the host threads gather into one of four pinned slabs while earlier chunks are in flight.  Mix 0 of
// host_decimate_mix gathers every chunk, 2 the odd ones, 1 (default) those whose gather would not outlast the copies already queued on the
// link, so that the link and the host cores are both kept busy.  Device-resident captures take the same loop without the copies.
struct HostPipe {
    cudaStream_t s_copy = nullptr, s_front = nullptr;
    cudaEvent_t ev_start = nullptr, ev_h2d[2] = {nullptr, nullptr}, ev_front[2] = {nullptr, nullptr};
    DecimPool* pool = nullptr;                         // the host threads, started by the first call that gathers
    void* hstage[4] = {nullptr, nullptr, nullptr, nullptr}; size_t hstage_cap = 0; cudaEvent_t ev_hfree[4] = {nullptr, nullptr, nullptr, nullptr};
    bool hstage_is_wc = false;                         // the pinned slabs were allocated write-combined (option host_stage_wc)
    std::vector<cudaEvent_t> ev_link; std::vector<uint64_t> link_bytes;     // one timed event per chunk copy of the current call, and its size
    double link_bpms = 50e6;                           // estimate of the link rate, bytes per ms (largest rate seen between two consecutive copy ends)
    double gather_ms_per_sample = 0.0;                 // running estimate of the host gather cost per 40 Msps sample (0 = not measured yet)
    std::vector<uint64_t> chunk_lo, chunk_hi; std::vector<int8_t> chunk_buf;   // per chunk of the current call: span in the capture, pinned slab of a gathered chunk
    DevBuf doff; std::vector<uint64_t> doffh;          // offset of every slot in the gathered copy of the call, on the device and on the host
    uint64_t last_h2d_bytes = 0, last_gathered_chunks = 0, last_chunks = 0;   // the last host-IQ call (sb200_last_transfer)
    ~HostPipe() {
        delete pool;                                    // the host threads have joined before the slabs they write go
        for (int i = 0; i < 4; i++) { if (hstage[i]) cudaFreeHost(hstage[i]); if (ev_hfree[i]) cudaEventDestroy(ev_hfree[i]); }
        for (cudaEvent_t e : ev_link) cudaEventDestroy(e);
        for (cudaEvent_t e : {ev_start, ev_h2d[0], ev_h2d[1], ev_front[0], ev_front[1]}) if (e) cudaEventDestroy(e);
        for (cudaStream_t s : {s_copy, s_front}) if (s) cudaStreamDestroy(s);
    }
    int run(sb200_handle* h, const Batch& bt, uint32_t chunk);
};

int host_pipe_create(HostPipe** out) {
    HostPipe* p = *out = new (std::nothrow) HostPipe();
    if (!p) return SB200_E_NOMEM;
    for (cudaStream_t* s : {&p->s_copy, &p->s_front}) if (cudaStreamCreateWithFlags(s, cudaStreamNonBlocking) != cudaSuccess) return SB200_E_CUDA;
    for (cudaEvent_t* e : {&p->ev_start, &p->ev_h2d[0], &p->ev_h2d[1], &p->ev_front[0], &p->ev_front[1], &p->ev_hfree[0], &p->ev_hfree[1], &p->ev_hfree[2], &p->ev_hfree[3]})
        if (cudaEventCreateWithFlags(e, cudaEventDisableTiming) != cudaSuccess) return SB200_E_CUDA;
    return SB200_OK;
}
void host_pipe_destroy(HostPipe* p) { delete p; }
void host_pipe_forget_gather_cost(HostPipe* p) { p->gather_ms_per_sample = 0.0; }
extern "C" int sb200_last_transfer(const sb200_handle* h, uint64_t* h2d_bytes, uint32_t* chunks, uint32_t* chunks_gathered) {
    if (!h) return SB200_E_INVALID;
    if (h2d_bytes) *h2d_bytes = h->pipe->last_h2d_bytes;
    if (chunks) *chunks = (uint32_t)h->pipe->last_chunks;
    if (chunks_gathered) *chunks_gathered = (uint32_t)h->pipe->last_gathered_chunks;
    return SB200_OK;
}

// One call in chunks of `chunk` slots.  Host IQ is sized first: the span [lo, hi) of every chunk that may travel as it is, the slot offsets
// in the gathered copy, and the staging for the largest chunk.
int HostPipe::run(sb200_handle* h, const Batch& bt, uint32_t chunk) {
    const std::vector<uint64_t>& offh = h->offh; const std::vector<uint32_t>& lenh = h->lenh;
    const uint32_t nframes = bt.nframes, nchunks = (nframes + chunk - 1) / chunk;
    const bool host = !bt.iq_dev, dec = host && h->host_decimate > 0;
    const uint32_t mix = dec ? h->host_mix : 0u;
    const bool out_host = bt.out_bytes && bt.out_stride && !bt.out_dev;     // the bytes go back chunk by chunk
    const size_t w = bt.out_stride < bt.row ? bt.out_stride : bt.row;
    if (host) {
        if (dec) {
            doffh.resize((size_t)nframes + 1); doffh[0] = 0;
            for (uint32_t i = 0; i < nframes; i++) doffh[i + 1] = doffh[i] + (lenh[i] + 1u) / 2u;
        }
        chunk_lo.assign(nchunks, 0); chunk_hi.assign(nchunks, 0); chunk_buf.assign(nchunks, -1);     // -1: sent as it is
        uint64_t stage_samples = 0, hstage_samples = 0;
        for (uint32_t c = 0, f0 = 0; c < nchunks; c++, f0 += chunk) {
            const uint32_t f1 = f0 + chunk < nframes ? f0 + chunk : nframes;
            if (dec && doffh[f1] - doffh[f0] > hstage_samples) hstage_samples = doffh[f1] - doffh[f0];
            if (dec && !mix) continue;                  // every chunk is gathered
            uint64_t lo = ~0ull, hi = 0;
            for (uint32_t i = f0; i < f1; i++) { if (offh[i] < lo) lo = offh[i]; if (offh[i] + lenh[i] > hi) hi = offh[i] + lenh[i]; }
            chunk_lo[c] = lo; chunk_hi[c] = hi;
            if (hi - lo > stage_samples) stage_samples = hi - lo;
        }
        if (hstage_samples > stage_samples) stage_samples = hstage_samples;
        CK(h->stage[0].need(stage_samples * 4ull + 16)); CK(h->stage[1].need(stage_samples * 4ull + 16));
        if (dec) {
            if (!pool || pool->n != (int)h->host_decimate) { delete pool; pool = new (std::nothrow) DecimPool((int)h->host_decimate); if (!pool) return h->fail(SB200_E_NOMEM, "host thread pool"); }
            if (hstage_cap < hstage_samples * 4ull || h->hstage_wc != hstage_is_wc) {
                hstage_cap = 0;
                for (int i = 0; i < 4; i++) { CK(cudaEventSynchronize(ev_hfree[i])); if (hstage[i]) cudaFreeHost(hstage[i]); hstage[i] = nullptr; }   // no copy out of a slab still queued
                const size_t want_b = hstage_samples * 4ull + hstage_samples / 2 + 256;
                // the staging buffers are written once by the host threads (streaming stores) and read only by the copy engine: write-combined
                // memory (option host_stage_wc) is not snooped on its way over PCIe
                for (int i = 0; i < 4; i++) CK(cudaHostAlloc(&hstage[i], want_b, h->hstage_wc ? cudaHostAllocWriteCombined : cudaHostAllocDefault));
                hstage_cap = want_b; hstage_is_wc = h->hstage_wc;
            }
            CK(doff.need(nframes * 8ull)); CK(cudaMemcpyAsync(doff.p, doffh.data(), nframes * 8ull, cudaMemcpyHostToDevice, bt.st));
        }
        while (ev_link.size() < nchunks) { cudaEvent_t e; CK(cudaEventCreate(&e)); ev_link.push_back(e); }
        link_bytes.assign(nchunks, 0);
    }
    CK(cudaEventRecord(ev_start, bt.st));
    CK(cudaStreamWaitEvent(s_copy, ev_start, 0)); CK(cudaStreamWaitEvent(s_front, ev_start, 0));
    uint32_t k = 0, gsub = 0, link_head = 0;          // chunk index, chunks handed to the host threads, first chunk whose copy may still be on the wire
    uint64_t h2d_bytes = 0;
    double gather_ms = 0.0;                            // time the host threads spent gathering (SB200_TRACE prints it)
    struct InFlight { DecimPool* p; ~InFlight() { if (p) p->wait(); } } inflight{pool};   // no return while the host threads still read the caller's capture
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
                const cudaError_t q = cudaEventQuery(ev_link[i]);
                if (q == cudaSuccess) {
                    if (i == link_head) {
                        float ms = 0.f;
                        if (i > 0 && cudaEventElapsedTime(&ms, ev_link[i - 1], ev_link[i]) == cudaSuccess && ms > 0.f) {
                            const double r = (double)link_bytes[i] / ms;
                            link_bpms = r > link_bpms ? r : 0.95 * link_bpms + 0.05 * r;   // a gap before the copy only lowers r
                        }
                        link_head++;
                    }
                } else if (q == cudaErrorNotReady) { (void)cudaGetLastError(); pend += link_bytes[i]; }
                else return h->fail(SB200_E_CUDA, "cudaEventQuery", q);
            }
            const double pend_ms = (double)pend / link_bpms;
            const double gather_est = gather_ms_per_sample * (double)(chunk_hi[c] - chunk_lo[c]);
            // a gather whose copy would reach the link after it has run dry costs link time: send the chunk as it is instead.
            // Not measured yet: the first chunk goes as it is (the link is idle anyway), the second is gathered and gives the estimate
            gather = gather_ms_per_sample > 0.0 ? pend_ms >= gather_est : c != 0u;
        }
        if (!gather) return SB200_OK;
        const int hb = (int)(gsub % 4u);
        // pinned buffer hb is free once its last copy has crossed the link: the gathered chunk four back, or one of an earlier call that
        // returned with its copies still queued (an event never recorded counts as complete)
        CK(cudaEventSynchronize(ev_hfree[hb]));
        pool->submit(DecimPool::Job{(const uint32_t*)bt.iq, offh.data(), lenh.data(), doffh.data(), f0, f1, (uint32_t*)hstage[hb]});
        chunk_buf[c] = (int8_t)hb; gsub++;
        return SB200_OK;
    };
    if (host) { const int rc = plan(0, 0); if (rc != SB200_OK) return rc; }
    for (uint32_t f0 = 0; f0 < nframes; f0 += chunk, k++) {
        const uint32_t f1 = f0 + chunk < nframes ? f0 + chunk : nframes; const int b = k & 1;
        Samples x{(const uint32_t*)bt.iq, bt.d_off, 1u, 0u, nullptr};
        if (host) {
            const bool gathered = chunk_buf[k] >= 0;
            if (gathered) {                              // the host threads finish this chunk; its cost per sample feeds the next decisions
                const double gms = pool->wait();
                gather_ms += gms;
                const double per = gms / (double)(2u * (doffh[f1] - doffh[f0]) + 1u);
                gather_ms_per_sample = gather_ms_per_sample > 0.0 ? 0.75 * gather_ms_per_sample + 0.25 * per : per;
            }
            link_bytes[k] = gathered ? (doffh[f1] - doffh[f0]) * 4ull : (chunk_hi[k] - chunk_lo[k]) * 4ull;
            if (k + 1 < nchunks) { const int rc = plan(k + 1, link_bytes[k]); if (rc != SB200_OK) return rc; }
            if (k >= 2) CK(cudaStreamWaitEvent(s_copy, ev_front[b], 0));            // device buffer b is free once chunk k-2's front end has read it
            if (gathered) {
                CK(cudaMemcpyAsync(h->stage[b].p, hstage[chunk_buf[k]], link_bytes[k], cudaMemcpyHostToDevice, s_copy));
                CK(cudaEventRecord(ev_hfree[chunk_buf[k]], s_copy));
                x = Samples{(const uint32_t*)h->stage[b].p - doffh[f0], (const uint64_t*)doff.p, 0u, 0u, nullptr};
            } else {
                CK(cudaMemcpyAsync(h->stage[b].p, (const uint32_t*)bt.iq + chunk_lo[k], link_bytes[k], cudaMemcpyHostToDevice, s_copy));
                x.base = (const uint32_t*)h->stage[b].p - chunk_lo[k];
            }
            h2d_bytes += link_bytes[k];
            CK(cudaEventRecord(ev_link[k], s_copy));
            CK(cudaEventRecord(ev_h2d[b], s_copy));
            CK(cudaStreamWaitEvent(s_front, ev_h2d[b], 0));
        }
        int rc = launch_chunk(h, bt, x, f0, f1, k, s_front, bt.st, ev_front[b], false);
        if (rc != SB200_OK) return rc;
        // results of this chunk go back while the next chunks are still coming in (PCIe is full duplex): only the last chunk's
        // device-to-host copy is left exposed at the end of the call
        const uint32_t n = f1 - f0;
        k_pack_results<<<(n + 255) / 256, 256, 0, bt.st>>>((const FrameInfo*)h->info.p + f0, (const uint32_t*)h->status.p + f0, (const uint32_t*)h->crc.p + f0, n, bt.d_res + f0);
        if (out_host) CK(cudaMemcpy2DAsync(bt.out_bytes + (size_t)f0 * bt.out_stride, bt.out_stride, (const uint8_t*)h->out.p + (size_t)f0 * bt.row, bt.row, w, n, cudaMemcpyDeviceToHost, bt.st));
        if (!bt.res_dev) CK(cudaMemcpyAsync(bt.res + f0, bt.d_res + f0, n * sizeof(sb200_frame_result), cudaMemcpyDeviceToHost, bt.st));
    }
    if (host) { last_h2d_bytes = h2d_bytes; last_gathered_chunks = gsub; last_chunks = k; }
    if (dec && getenv("SB200_TRACE")) fprintf(stderr, "[sb200] rx11a host_decimate: %u chunks (%u gathered, %u sent as they are), host gather %.2f ms in total (%u threads), link estimate %.1f GB/s, %.1f MB copied\n", k, gsub, k - gsub, gather_ms, h->host_decimate, link_bpms / 1e6, h2d_bytes / 1e6);
    Returns ret;                                        // what goes to the host was already queued chunk by chunk
    if (bt.out_bytes && bt.out_stride && bt.out_dev) ret.bind2d(bt.out_bytes, bt.out_stride, h->out.p, bt.row, w, nframes);
    const int rc = finish_call(h, bt.st, ret, 0, k);     // k launches of k_pack_results
    if (rc == SB200_OK && (out_host || !bt.res_dev)) CK(cudaStreamSynchronize(bt.st));
    return rc;
}

// shared body of sb200_rx11a_batch / sb200_rx11a_taps: the checks, the slot table and the workspaces, then one pass on the caller's stream
// or, for a large call, the handle's pipeline.
static int rx11a_run(sb200_handle* h, const int16_t* iq, uint64_t iq_total, const uint64_t* frame_off, const uint32_t* frame_len,
                     uint32_t nframes, uint8_t* out_bytes, uint32_t out_stride, sb200_frame_result* res, cudaStream_t st,
                     FrontTaps taps, uint8_t* soft_host, uint64_t soft_host_stride, const int2* dc_init = nullptr, bool no_chunk = false, bool rate20 = false) {
    if (!h || !iq || !frame_off || !frame_len || !res) return h ? h->fail(SB200_E_INVALID, "null argument") : SB200_E_INVALID;
    if (nframes == 0) return SB200_OK;
    CK(cudaSetDevice(h->device));
    CallScope call(h, st); CK(call.begin()); call.reads(iq);
    // slot table: checked on every call (slot_table, sb200.cu); the chunked host-IQ path also needs it on the host
    const bool iq_dev = is_device_ptr(iq);
    const uint64_t* d_off; const uint32_t* d_len; uint32_t max_len = 0; bool tab_on_host = false;
    const bool may_chunk = !no_chunk && !rate20 && !iq_dev && h->chunk_frames != 0 && nframes > h->chunk_frames;
    int rc = slot_table(h, frame_off, frame_len, nframes, iq_total, may_chunk, st, &d_off, &d_len, &max_len, &tab_on_host);
    if (rc != SB200_OK) return rc;
    if (rate20) { if (max_len > 0x7FFFFFFFu) return h->fail(SB200_E_INVALID, "slot too long"); max_len <<= 1; }   // slots counted in 20 Msps samples
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
    CK(h->vcnt.need(32ull * ((nframes + chunk - 1) / chunk)));
    const bool res_dev = is_device_ptr(res);
    const Batch bt{iq, iq_dev, d_off, d_len, nframes, soft_stride, row, taps, st, out_bytes, out_stride, out_bytes && is_device_ptr(out_bytes),
                   res, res_dev ? res : (sb200_frame_result*)h->res.p, res_dev};
    CK(cudaEventRecord(h->ev0, st));
    if (chunk < nframes) return h->pipe->run(h, bt, chunk);
    const uint32_t* d_iq;
    CK(to_device(h->iq, (const uint32_t*)iq, iq_dev, iq_total * 4ull, st, &d_iq));
    if (!iq_dev) { h->pipe->last_h2d_bytes = iq_total * 4ull; h->pipe->last_gathered_chunks = 0; h->pipe->last_chunks = 1; }
    rc = launch_chunk(h, bt, Samples{d_iq, d_off, rate20 ? 0u : 1u, rate20 ? 1u : 0u, dc_init}, 0, nframes, 0, st, st, nullptr, true);
    if (rc != SB200_OK) return rc;
    k_pack_results<<<(nframes + 255) / 256, 256, 0, st>>>((const FrameInfo*)h->info.p, (const uint32_t*)h->status.p, (const uint32_t*)h->crc.p, nframes, bt.d_res);
    CK(cudaEventRecord(h->evk[4], st));
    Returns ret;
    if (out_bytes && out_stride) ret.bind2d(out_bytes, out_stride, h->out.p, row, out_stride < row ? out_stride : row, nframes);
    if (!res_dev) ret.copy(res, bt.d_res, nframes * sizeof(sb200_frame_result));
    if (soft_host) ret.bind2d(soft_host, soft_host_stride, h->soft.p, soft_stride, soft_host_stride < soft_stride ? soft_host_stride : soft_stride, nframes);
    return finish_call(h, st, ret, 4, 1);
}

// Many continuous captures at once.  Every pass decodes the next frame of every capture that still has samples (one slot per
// capture, from its cursor to its end, with its own carried DC), so the device sees a full batch per pass and the number of
// passes is the largest number of frames in any one capture.
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
            k_front11a<0><<<(n + SB_FRONT_SLOTS - 1) / SB_FRONT_SLOTS, 32 * SB_FRONT_WARPS, 0, st>>>((const uint32_t*)d_iq, (const uint64_t*)h->soff.p, (const uint32_t*)h->slen.p, n, h->T, (FrameInfo*)h->info.p, nullptr, 0, h->inv_deint, hdr, 1u, 0u);
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
