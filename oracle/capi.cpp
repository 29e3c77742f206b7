// ORACLE — TEST INFRASTRUCTURE ONLY (see ops.h).  C entry points for tests/ (ctypes) and bench.py's cpu_baseline.
#include "rx11b.h"
#include "rx11n.h"
#include "tx11a.h"
#include "tx11b.h"
#include "tx11n.h"
#include <thread>
#include <atomic>
#include <vector>

using namespace sbo;

static uint32_t g_cca_thr = 1000 * 1000;   // CF_11CCA::cca_pwr_threshold used by the 802.11a entry points below (fb11ademod_config.hpp:107 default)

extern "C" {
void sbo_set_cca_threshold(uint32_t thr) { g_cca_thr = thr ? thr : 1000 * 1000; }

struct sbo_frame_result {           // mirrors sbo::FrameResult; keep in sync with tests/oracle_py.py
    uint32_t status, rate_kbps, length, crc32, nsym, sample_index, detect_index;
    int16_t cfo_est; uint16_t peak_index;
};

int sbo_rx11a_run(const int16_t* iq, uint64_t nsamples, int max_frames, sbo_frame_result* res,
                  uint8_t* out, uint64_t out_stride) {
    Rx11a rx; rx.cca_pwr_threshold = g_cca_thr;
    return rx.run((const c16*)iq, (size_t)nsamples, (FrameResult*)res, out, (size_t)out_stride, max_frames);
}

// Batched "one capture slot per frame" mode: slot i = iq[off[i] .. off[i]+len[i]) decoded from a fresh context,
// first event reported (status E_NO_FRAME if none).  nthreads host threads over independent slots.
void sbo_rx11a_batch(const int16_t* iq, const uint64_t* off, const uint32_t* len, uint32_t nframes,
                     sbo_frame_result* res, uint8_t* out, uint64_t out_stride, int nthreads) {
    std::atomic<uint32_t> next(0);
    auto work = [&]() {
        Rx11a rx; rx.cca_pwr_threshold = g_cca_thr;
        for (;;) {
            uint32_t i = next.fetch_add(1); if (i >= nframes) break;
            FrameResult r; memset(&r, 0, sizeof r);
            int n = rx.run((const c16*)iq + off[i], len[i], &r, out ? out + (size_t)i * out_stride : nullptr, (size_t)out_stride, 1);
            if (n == 0) { memset(&r, 0, sizeof r); r.status = E_NO_FRAME; }
            memcpy(&res[i], &r, sizeof r);
        }
    };
    if (nthreads <= 1) { work(); return; }
    std::vector<std::thread> th; for (int t = 0; t < nthreads; t++) th.emplace_back(work);
    for (auto& t : th) t.join();
}

// The same batch through the reference's two-thread topology: every pipeline = one front-end thread (carrier sense .. de-interleaver) and one
// Viterbi thread (T11aViterbi .. frame sink) joined by a single-producer / single-consumer ring, like TThreadSeparator<> (stdbrick.hpp:91-248).
// npipes pipelines share the slots through an atomic counter.  Results are identical to sbo_rx11a_batch (tests/test_cpu_oracle.py).
namespace {
struct SplitRing : Rx11a::SoftSplit {
    struct Rec { uint32_t kind, slot; int code_rate; uint16_t frame_length; int ncbps; uint8_t soft[288]; };   // kind 0 begin, 1 symbol, 2 frame complete, 3 stop, 4 slot ended without a complete frame
    static const uint32_t N = 512;
    std::vector<Rec> ring; std::atomic<uint32_t> head{0}, tail{0}; uint32_t cur_slot = 0;
    SplitRing() : ring(N) {}
    Rec& claim() { uint32_t h = head.load(std::memory_order_relaxed); while (h - tail.load(std::memory_order_acquire) >= N) std::this_thread::yield(); return ring[h % N]; }
    void publish() { head.store(head.load(std::memory_order_relaxed) + 1, std::memory_order_release); }
    void begin(int code_rate, uint16_t frame_length) override { Rec& r = claim(); r.kind = 0; r.slot = cur_slot; r.code_rate = code_rate; r.frame_length = frame_length; publish(); }
    void symbol(const uint8_t* dsoft, int ncbps) override { Rec& r = claim(); r.kind = 1; r.slot = cur_slot; r.ncbps = ncbps; memcpy(r.soft, dsoft, (size_t)ncbps); publish(); }
    void mark(uint32_t kind, uint32_t slot) { Rec& r = claim(); r.kind = kind; r.slot = slot; publish(); }
    const Rec* peek() { uint32_t t = tail.load(std::memory_order_relaxed); while (head.load(std::memory_order_acquire) == t) std::this_thread::yield(); return &ring[t % N]; }
    void pop() { tail.store(tail.load(std::memory_order_relaxed) + 1, std::memory_order_release); }
};
}
void sbo_rx11a_batch_2t(const int16_t* iq, const uint64_t* off, const uint32_t* len, uint32_t nframes,
                        sbo_frame_result* res, uint8_t* out, uint64_t out_stride, int npipes) {
    std::atomic<uint32_t> next(0);
    auto pipeline = [&]() {
        SplitRing q;
        std::thread back([&]() {                        // Viterbi thread
            Rx11a vb; bool open = false;
            for (;;) {
                const SplitRing::Rec* r = q.peek(); const uint32_t kind = r->kind, slot = r->slot;
                if (kind == 3) { q.pop(); break; }
                if (kind == 0) { vb.back_begin(r->code_rate, r->frame_length); open = true; }
                else if (kind == 1) vb.back_symbol(r->soft, r->ncbps);
                else if (kind == 2 && open) {           // the slot's frame is complete: verdict, FCS and bytes come from this side
                    uint32_t st = vb.back_status(); if (st == E_SUCCESS) st = E_FAILED;
                    res[slot].status = st; res[slot].crc32 = vb.back_crc32();
                    if (out) { size_t nb = res[slot].length < out_stride ? res[slot].length : out_stride; memcpy(out + (size_t)slot * out_stride, vb.frame_bytes(), nb); }
                    open = false;
                } else if (kind == 4) open = false;     // the capture ended inside the frame: nothing to report from this side
                q.pop();
            }
        });
        Rx11a rx; rx.cca_pwr_threshold = g_cca_thr; rx.split = &q;
        for (;;) {
            uint32_t i = next.fetch_add(1); if (i >= nframes) break;
            q.cur_slot = i;
            FrameResult r; memset(&r, 0, sizeof r);
            int n = rx.run((const c16*)iq + off[i], len[i], &r, nullptr, 0, 1);
            if (n == 0) { memset(&r, 0, sizeof r); r.status = E_NO_FRAME; }
            memcpy(&res[i], &r, sizeof r);              // front-end fields; a decoded frame's status / crc32 / bytes are overwritten by the Viterbi thread
            q.mark(n > 0 && r.status == E_FAILED ? 2u : 4u, i);   // E_FAILED = all symbols went through, the verdict is the Viterbi thread's
        }
        q.mark(3, 0);
        back.join();
    };
    if (npipes <= 1) { pipeline(); return; }
    std::vector<std::thread> th; for (int t = 0; t < npipes; t++) th.emplace_back(pipeline);
    for (auto& t : th) t.join();
}

// Stage taps of the first frame in a buffer.  Buffers sized by the caller: coeffs 64 c16 each;
// per-symbol arrays max_sym*64 c16 (fft_in, may be null: what fft64 was handed, fft_out: what it returned); soft max_sym*288 bytes;
// lts_in (may be null) 144 c16: the block T11aLTS is handed; sym_in (may be null) max_sym*80 c16: the blocks T11aDataSymbol is handed.
// Returns number of symbols captured (incl. SIGNAL).
int sbo_rx11a_taps_blocks(const int16_t* iq, uint64_t nsamples, sbo_frame_result* res,
                          int16_t* freq_coeffs, int16_t* chan_coeffs, int16_t* fft_out, int16_t* equalized, int16_t* tracked,
                          uint8_t* soft, uint32_t* soft_off, int max_sym, int16_t* fft_in, int16_t* lts_in, int16_t* sym_in) {
    Rx11a rx; rx.cca_pwr_threshold = g_cca_thr; rx.taps.enable = true;
    FrameResult r; memset(&r, 0, sizeof r);
    int n = rx.run((const c16*)iq, (size_t)nsamples, &r, nullptr, 0, 1);
    if (n == 0) r.status = E_NO_FRAME;
    memcpy(res, &r, sizeof r);
    const Taps& t = rx.taps;
    if (t.freq_coeffs.size() == 64) { memcpy(freq_coeffs, t.freq_coeffs.data(), 256); memcpy(chan_coeffs, t.chan_coeffs.data(), 256); }
    int ns = (int)(t.fft_out.size() / 64); if (ns > max_sym) ns = max_sym;
    if (fft_in) memcpy(fft_in, t.fft_in.data(), (size_t)ns * 256);
    if (lts_in && t.lts_in.size() == 144) memcpy(lts_in, t.lts_in.data(), 144 * 4);
    if (sym_in) memcpy(sym_in, t.sym_in.data(), (size_t)ns * 320);
    memcpy(fft_out, t.fft_out.data(), (size_t)ns * 256); memcpy(equalized, t.equalized.data(), (size_t)ns * 256);
    memcpy(tracked, t.tracked.data(), (size_t)ns * 256);
    for (int i = 0; i < ns; i++) {
        soft_off[i] = t.soft_off[i];
        size_t end = (i + 1 < (int)t.soft_off.size()) ? t.soft_off[i + 1] : t.soft.size();
        memcpy(soft + t.soft_off[i], t.soft.data() + t.soft_off[i], end - t.soft_off[i]);
    }
    soft_off[ns] = (uint32_t)(ns < (int)t.soft_off.size() ? t.soft_off[ns] : t.soft.size());
    return ns;
}
// The carrier-sense trace up to the first frame event: per 20 Msps vector handed to cca_process, 13 int32 after it (cca_state,
// error_code, DC as 8 int16 lanes, cca_peak_index, cca_pwr_reading, the vector's 20 Msps index).  Returns the number of vectors
// (at most max_vec); *detect = detect_index of the first detection, or -1.
uint64_t sbo_rx11a_cs_trace(const int16_t* iq, uint64_t nsamples, int32_t* rec, uint64_t max_vec, int64_t* detect) {
    Rx11a rx; rx.cca_pwr_threshold = g_cca_thr; rx.taps.enable = true;
    FrameResult r; memset(&r, 0, sizeof r);
    int n = rx.run((const c16*)iq, (size_t)nsamples, &r, nullptr, 0, 1);
    const std::vector<int32_t>& t = rx.taps.cs;
    size_t m = t.size() / 13; if (m > max_vec) m = max_vec;
    memcpy(rec, t.data(), m * 13 * sizeof(int32_t));
    bool det = n > 0 || (!t.empty() && t[t.size() - 13] == 1);
    *detect = det ? (int64_t)t[t.size() - 1] + 1 : -1;
    return m;
}
// the same without the LTS and symbol-block taps
int sbo_rx11a_taps_in(const int16_t* iq, uint64_t nsamples, sbo_frame_result* res,
                      int16_t* freq_coeffs, int16_t* chan_coeffs, int16_t* fft_out, int16_t* equalized, int16_t* tracked,
                      uint8_t* soft, uint32_t* soft_off, int max_sym, int16_t* fft_in) {
    return sbo_rx11a_taps_blocks(iq, nsamples, res, freq_coeffs, chan_coeffs, fft_out, equalized, tracked, soft, soft_off, max_sym, fft_in,
                                 nullptr, nullptr);
}
// the same without the fft_in tap (the entry point's original argument list)
int sbo_rx11a_taps(const int16_t* iq, uint64_t nsamples, sbo_frame_result* res,
                   int16_t* freq_coeffs, int16_t* chan_coeffs, int16_t* fft_out, int16_t* equalized, int16_t* tracked,
                   uint8_t* soft, uint32_t* soft_off, int max_sym) {
    return sbo_rx11a_taps_in(iq, nsamples, res, freq_coeffs, chan_coeffs, fft_out, equalized, tracked, soft, soft_off, max_sym, nullptr);
}

// Standalone Viterbi block decode (BASELINE config #5): soft = nsoft coded soft values (0..7) at code_rate,
// frame_len_bytes L defines the flush point 8L+16+6; writes L+2 bytes... (SERVICE + PSDU, still scrambled).
uint64_t sbo_viterbi_block(const uint8_t* soft, uint64_t nsoft, int code_rate, uint32_t frame_len_bytes,
                           uint32_t depth, uint32_t lookahead, uint8_t* out) {
    ViterbiCore v; v.max_steps = (uint32_t)nsoft + 8; v.reset();
    uint32_t ob = 0;
    return viterbi_decode_block(v, soft, (size_t)nsoft, code_rate, frame_len_bytes, depth, lookahead, out, ob);
}
// nblocks blocks of one layout; nbytes (may be null): bytes each block produced.  A block whose soft values end before its flush point
// produces only the windows that fired; the rest of its output row is left untouched.
void sbo_viterbi_blocks_n(const uint8_t* soft, uint64_t nsoft_per_block, uint32_t nblocks, int code_rate, uint32_t frame_len_bytes,
                          uint32_t depth, uint32_t lookahead, uint8_t* out, uint64_t out_stride, uint32_t* nbytes, int nthreads) {
    std::atomic<uint32_t> next(0);
    auto work = [&]() {
        ViterbiCore v; v.max_steps = (uint32_t)nsoft_per_block + 8;
        for (;;) { uint32_t i = next.fetch_add(1); if (i >= nblocks) break;
            v.reset(); uint32_t ob = 0;
            const size_t n = viterbi_decode_block(v, soft + (size_t)i * nsoft_per_block, (size_t)nsoft_per_block, code_rate, frame_len_bytes, depth, lookahead,
                                                  out + (size_t)i * out_stride, ob);
            if (nbytes) nbytes[i] = (uint32_t)n; }
    };
    if (nthreads <= 1) { work(); return; }
    std::vector<std::thread> th; for (int t = 0; t < nthreads; t++) th.emplace_back(work);
    for (auto& t : th) t.join();
}
void sbo_viterbi_blocks(const uint8_t* soft, uint64_t nsoft_per_block, uint32_t nblocks, int code_rate, uint32_t frame_len_bytes,
                        uint32_t depth, uint32_t lookahead, uint8_t* out, uint64_t out_stride, int nthreads) {
    sbo_viterbi_blocks_n(soft, nsoft_per_block, nblocks, code_rate, frame_len_bytes, depth, lookahead, out, out_stride, nullptr, nthreads);
}
uint32_t sbo_viterbi_signal(const uint8_t* soft48) { return viterbi_signal(soft48); }

void sbo_fft64(const int16_t* in, int16_t* out) { alignas(16) c16 t[64]; memcpy(t, in, 256); alignas(16) c16 o[64]; fft64((v128*)t, (v128*)o); memcpy(out, o, 256); }
void sbo_ifft64(const int16_t* in, int16_t* out) { alignas(16) c16 t[64]; memcpy(t, in, 256); alignas(16) c16 o[64]; ifft64((v128*)t, (v128*)o); memcpy(out, o, 256); }
// n vectors of 64 (128) c16 each, back to back
void sbo_fft64_n(uint64_t n, const int16_t* in, int16_t* out) { for (uint64_t i = 0; i < n; i++) sbo_fft64(in + 128 * i, out + 128 * i); }
void sbo_ifft64_n(uint64_t n, const int16_t* in, int16_t* out) { for (uint64_t i = 0; i < n; i++) sbo_ifft64(in + 128 * i, out + 128 * i); }
int16_t sbo_uatan2(int y, int x) { return uatan2(y, x); }
int16_t sbo_usin(int16_t r) { return usin(r); }
int16_t sbo_ucos(int16_t r) { return ucos(r); }
void sbo_demap(const int16_t* eq, uint8_t* out, int nbpsc) { demap_symbol((const c16*)eq, out, nbpsc); }
void sbo_deinterleave(const uint8_t* in, uint8_t* out, int ncbps) { deinterleave(in, out, ncbps); }
const int16_t* sbo_sts_pattern() { return (const int16_t*)tables().sts_pattern; }
void sbo_tables(const uint8_t** vit_ma, const uint8_t** vit_mb, const uint8_t** demap4 /*4x256*/) {
    const Tables& T = tables(); *vit_ma = &T.vit_ma[0][0]; *vit_mb = &T.vit_mb[0][0]; *demap4 = T.demap_bpsk;
}
// The descrambler of Rx11a::sink_byte / Rx11n::sink_byte on decoded bytes (SERVICE + PSDU): n - 2 PSDU bytes out
void sbo_descramble(const uint8_t* in, uint32_t n, uint8_t* out) {
    uint8_t reg = n > 1 ? in[1] >> 1 : 0;
    for (uint32_t i = 2; i < n; i++) { reg = tables().scramble_lut[reg]; out[i - 2] = in[i] ^ reg; reg >>= 1; }
}
uint64_t sbo_resample_44_40(const int16_t* in, uint64_t n_in, int16_t* out) { return resample_44_40((const c16*)in, (size_t)n_in, (c16*)out); }

// ---- 802.11b ----
struct sbo_frame_result_11b { uint32_t status, rate_kbps, length, crc32, sample_index, detect_vec; };
int sbo_rx11b_run(const int16_t* iq, uint64_t nsamples, int max_frames, sbo_frame_result_11b* res, uint8_t* out, uint64_t out_stride) {
    Rx11b rx;
    return rx.run((const c16*)iq, (size_t)nsamples, (FrameResult11b*)res, out, (size_t)out_stride, max_frames);
}
void sbo_rx11b_batch(const int16_t* iq, const uint64_t* off, const uint32_t* len, uint32_t nframes,
                     sbo_frame_result_11b* res, uint8_t* out, uint64_t out_stride, int nthreads) {
    std::atomic<uint32_t> next(0);
    auto work = [&]() {
        Rx11b rx;
        for (;;) {
            uint32_t i = next.fetch_add(1); if (i >= nframes) break;
            FrameResult11b r; memset(&r, 0, sizeof r);
            int n = rx.run((const c16*)iq + off[i], len[i], &r, out ? out + (size_t)i * out_stride : nullptr, (size_t)out_stride, 1);
            if (n == 0) { memset(&r, 0, sizeof r); r.status = E_NO_FRAME; }
            memcpy(&res[i], &r, sizeof r);
        }
    };
    if (nthreads <= 1) { work(); return; }
    std::vector<std::thread> th; for (int t = 0; t < nthreads; t++) th.emplace_back(work);
    for (auto& t : th) t.join();
}
// the CCK decoders the chain runs, on n symbols (CCK-11: 8 chips, is_even from 0) / bytes (CCK-5.5: 16 chips) in turn; last2 in / out
void sbo_cck11_decode_n(const int16_t* chips, uint64_t n, int16_t* last2, uint8_t* out) {
    c16 l{last2[0], last2[1]}; int even = 0;
    for (uint64_t i = 0; i < n; i++) out[i] = cck11_decode((const c16*)chips + 8 * i, l, even);
    last2[0] = l.re; last2[1] = l.im;
}
void sbo_cck5_decode_n(const int16_t* chips, uint64_t n, int16_t* last2, uint8_t* out) {
    c16 l{last2[0], last2[1]};
    for (uint64_t i = 0; i < n; i++) out[i] = cck5_decode((const c16*)chips + 16 * i, l);
    last2[0] = l.re; last2[1] = l.im;
}
// the Barker branches the chain runs: despread on n blocks of 11 chips; DBPSK / DQPSK on n bytes of 8 / 4 symbols in turn, last2 in / out
void sbo_despread_n(const int16_t* chips, uint64_t n, int16_t* out) {
    for (uint64_t i = 0; i < n; i++) { c16 s = barker_despread((const c16*)chips + 11 * i); out[2 * i] = s.re; out[2 * i + 1] = s.im; }
}
void sbo_dbpsk_demap_n(const int16_t* sym, uint64_t n, int16_t* last2, uint8_t* out) {
    c16 l{last2[0], last2[1]};
    for (uint64_t i = 0; i < n; i++) out[i] = dbpsk_demap((const c16*)sym + 8 * i, l);
    last2[0] = l.re; last2[1] = l.im;
}
void sbo_dqpsk_demap_n(const int16_t* sym, uint64_t n, int16_t* last2, uint8_t* out) {
    c16 l{last2[0], last2[1]};
    for (uint64_t i = 0; i < n; i++) out[i] = dqpsk_demap((const c16*)sym + 4 * i, l);
    last2[0] = l.re; last2[1] = l.im;
}
uint8_t sbo_cck11_decode(const int16_t* chips8, int16_t* last2, int* even) { c16 l{last2[0], last2[1]}; uint8_t b = cck11_decode((const c16*)chips8, l, *even); last2[0] = l.re; last2[1] = l.im; return b; }

// ---- 802.11n 2x2 -----------------------------------------------------------------------------------------------------
int sbo_rx11n_run(const int16_t* iq0, const int16_t* iq1, uint64_t nsamples, int max_frames, void* res, uint8_t* out, uint64_t out_stride) {
    Rx11n rx;
    return rx.run((const c16*)iq0, (const c16*)iq1, (size_t)nsamples, (FrameResult11n*)res, out, (size_t)out_stride, max_frames);
}
void sbo_rx11n_batch(const int16_t* iq0, const int16_t* iq1, const uint64_t* off, const uint32_t* len, uint32_t nframes,
                     void* res_, uint8_t* out, uint64_t out_stride, int nthreads) {
    FrameResult11n* res = (FrameResult11n*)res_;
    std::atomic<uint32_t> next(0);
    auto work = [&]() {
        Rx11n rx;
        for (;;) {
            uint32_t i = next.fetch_add(1); if (i >= nframes) break;
            FrameResult11n r; memset(&r, 0, sizeof r);
            int n = rx.run((const c16*)iq0 + off[i], (const c16*)iq1 + off[i], len[i], &r, out ? out + (size_t)i * out_stride : nullptr, (size_t)out_stride, 1);
            if (n == 0) { memset(&r, 0, sizeof r); r.status = E_NO_FRAME; }
            memcpy(&res[i], &r, sizeof r);
        }
    };
    if (nthreads <= 1) { work(); return; }
    std::vector<std::thread> th; for (int t = 0; t < nthreads; t++) th.emplace_back(work);
    for (auto& t : th) t.join();
}
// stage taps of the first frame: siso [2][64], hinv [4][64], fft_out [2][max_sym][64] (every 64-point FFT in order: 2 L-LTF + symbols) and
// fft_in [2][max_sym][64] (may be null: what each of those FFTs was handed),
// eq [2][max_sym][64] (data symbols), soft (stream-parsed, concatenated), theta per data symbol, sig 9 bytes.  Returns #data symbols.
int sbo_rx11n_taps_in(const int16_t* iq0, const int16_t* iq1, uint64_t nsamples, void* res, int16_t* siso, int16_t* hinv, int16_t* fft_out, int16_t* eq,
                      uint8_t* soft, uint32_t* nsoft, int16_t* theta, uint8_t* sig, int max_sym, int* nfft, int16_t* fft_in) {
    Rx11n rx; rx.taps.enable = true;
    FrameResult11n r; memset(&r, 0, sizeof r);
    int n = rx.run((const c16*)iq0, (const c16*)iq1, (size_t)nsamples, &r, nullptr, 0, 1);
    if (n == 0) r.status = E_NO_FRAME;
    memcpy(res, &r, sizeof r);
    const Taps11n& t = rx.taps;
    for (int a = 0; a < 2; a++) {
        if (t.siso[a].size() == 64) memcpy(siso + a * 128, t.siso[a].data(), 256);
        size_t nf = t.fft_out[a].size() / 64; if (nf > (size_t)max_sym) nf = max_sym;
        memcpy(fft_out + (size_t)a * max_sym * 128, t.fft_out[a].data(), nf * 256); *nfft = (int)nf;
        if (fft_in) memcpy(fft_in + (size_t)a * max_sym * 128, t.fft_in[a].data(), nf * 256);
        size_t ne = t.eq[a].size() / 64; if (ne > (size_t)max_sym) ne = max_sym;
        memcpy(eq + (size_t)a * max_sym * 128, t.eq[a].data(), ne * 256);
    }
    if (t.hinv.size() == 256) memcpy(hinv, t.hinv.data(), 1024);
    size_t ns = t.soft.size(); memcpy(soft, t.soft.data(), ns); *nsoft = (uint32_t)ns;
    size_t nd = t.theta.size(); if (nd > (size_t)max_sym) nd = max_sym;
    memcpy(theta, t.theta.data(), nd * 2); memcpy(sig, t.sig, 9);
    return (int)nd;
}
// the same without the fft_in tap (the entry point's original argument list)
int sbo_rx11n_taps(const int16_t* iq0, const int16_t* iq1, uint64_t nsamples, void* res, int16_t* siso, int16_t* hinv, int16_t* fft_out, int16_t* eq,
                   uint8_t* soft, uint32_t* nsoft, int16_t* theta, uint8_t* sig, int max_sym, int* nfft) {
    return sbo_rx11n_taps_in(iq0, iq1, nsamples, res, siso, hinv, fft_out, eq, soft, nsoft, theta, sig, max_sym, nfft, nullptr);
}
int16_t sbo_dsp_atan(int x, int y) { return dsp_atan(x, y); }
void sbo_set_ht_mcs_limit(uint32_t first_refused) { set_ht_mcs_limit(first_refused); }
uint32_t sbo_ht_mcs_limit() { return ht_mcs_limit(); }
void sbo_tables11n_qam(uint8_t* demap16, uint8_t* demap64) { const Tables11n& T = tables11n(); memcpy(demap16, T.demap16, sizeof T.demap16); memcpy(demap64, T.demap64, sizeof T.demap64); }
void sbo_tables11n(int16_t* sincos, int16_t* atan_lut, uint8_t* demap, uint8_t* crc8, uint16_t* deint, uint8_t* lltf_sign, uint8_t* htltf_sign) {
    const Tables11n& T = tables11n();
    memcpy(sincos, T.sincos, sizeof T.sincos); memcpy(atan_lut, T.atan_lut, sizeof T.atan_lut); memcpy(demap, T.demap, 256); memcpy(crc8, T.crc8, 256);
    memcpy(deint, T.deint, sizeof T.deint); memcpy(lltf_sign, T.lltf_sign, 64); memcpy(htltf_sign, T.htltf_sign, 64);
}

// ---- 802.11a transmit ---------------------------------------------------------------------------------------------------
uint64_t sbo_tx11a_modulate(const uint8_t* payload, uint32_t len, uint32_t rate_kbps, uint8_t seed, int8_t* out, uint64_t cap_samples, uint32_t tail_zeros) {
    return tx11a_modulate(payload, len, rate_kbps, seed, out, (size_t)cap_samples, tail_zeros);
}
uint32_t sbo_tx11a_nsym(uint32_t len, uint32_t rate_kbps) { return tx11a_nsym(len, rate_kbps); }
// the 802.11a transmit stages on their own (tx11a.h); bits one per byte
void sbo_tx11a_scramble_n(const uint8_t* in, const uint8_t* ctrl, uint64_t n, uint8_t seed, uint8_t* out) { uint8_t reg = seed; tx11a_scramble(in, ctrl, (size_t)n, reg, out); }
uint64_t sbo_tx11a_encode_bits(const uint8_t* in, uint64_t n, int cr, uint8_t* out) {
    std::vector<uint8_t> b(in, in + n), c; tx11a_encode_bits(b, cr, c); memcpy(out, c.data(), c.size()); return c.size();
}
void sbo_tx11a_interleave_n(const uint8_t* coded, uint64_t nsym, int nbpsc, uint8_t* air) {
    for (uint64_t s = 0; s < nsym; s++) tx11a_interleave(coded + 48 * nbpsc * s, nbpsc, air + 48 * nbpsc * s);
}
void sbo_tx11a_map_n(const uint8_t* air, uint64_t nsym, int nbpsc, int16_t* d48) {
    for (uint64_t s = 0; s < nsym; s++) tx11a_map(air + 48 * nbpsc * s, nbpsc, (c16*)d48 + 48 * s);
}
void sbo_tx11a_add_pilot_n(const int16_t* d48, uint64_t nsym, int16_t* f64) {          // pilot index 127 first, as after T11aAddPilot::Reset
    unsigned pi = 127; for (uint64_t s = 0; s < nsym; s++) tx11a_add_pilot((const c16*)d48 + 48 * s, pi, (c16*)f64 + 64 * s);
}
void sbo_tx11a_ifftx_n(const int16_t* f64, uint64_t nsym, int16_t* out160) {
    for (uint64_t s = 0; s < nsym; s++) tx11a_ifftx((const c16*)f64 + 64 * s, (c16*)out160 + 160 * s);
}
void sbo_tx11a_pack8_n(const int16_t* in, uint64_t n, int8_t* out) { tx11a_pack8((const c16*)in, (size_t)n, out); }
uint64_t sbo_tx11a_legacy_modulate(const uint8_t* mpdu, uint32_t len, int append_crc, uint32_t rate_kbps, const int16_t* preamble640, int8_t* out, uint64_t cap_samples) {
    return tx11a_legacy_modulate(mpdu, len, append_crc, rate_kbps, (const c16*)preamble640, out, (size_t)cap_samples);
}
uint32_t sbo_tx11a_legacy_nsym(uint32_t psdu_len, uint32_t rate_kbps) { return tx11a_legacy_nsym(psdu_len, rate_kbps); }
void sbo_ifft128(const int16_t* in, int16_t* out) { alignas(16) c16 t[128]; memcpy(t, in, 512); alignas(16) c16 o[128]; ifft128((v128*)t, (v128*)o); memcpy(out, o, 512); }
void sbo_ifft128_n(uint64_t n, const int16_t* in, int16_t* out) { for (uint64_t i = 0; i < n; i++) sbo_ifft128(in + 256 * i, out + 256 * i); }
// Start logging the inputs of every ifft128 on the calling thread (the transmitters run on it); sbo_ifft128_log_end stops, copies up to
// max of them (128 c16 each) and returns how many there were; the log is kept until the next sbo_ifft128_log_begin.
static thread_local std::vector<c16> g_ifft128_log;
void sbo_ifft128_log_begin() { g_ifft128_log.clear(); ifft128_log = &g_ifft128_log; }
uint64_t sbo_ifft128_log_end(int16_t* out, uint64_t max) {
    ifft128_log = nullptr; const uint64_t n = g_ifft128_log.size() / 128;
    if (out && max) memcpy(out, g_ifft128_log.data(), (size_t)(n < max ? n : max) * 512);
    return n;
}

// ---- 802.11b transmit ---------------------------------------------------------------------------------------------------
uint64_t sbo_tx11b_modulate(const uint8_t* payload, uint32_t len, uint32_t rate_kbps, uint32_t init_phase, int8_t* out, uint64_t cap_samples, uint32_t* final_phase) {
    return tx11b_modulate(payload, len, rate_kbps, init_phase, out, (size_t)cap_samples, final_phase);
}
uint32_t sbo_tx11b_nsamples(uint32_t len, uint32_t rate_kbps) { return tx11b_nsamples(len, rate_kbps); }
void sbo_tx11b_taps(int16_t* out20) { tx11b_taps(out20); }

// ---- 802.11n transmit ---------------------------------------------------------------------------------------------------
uint64_t sbo_tx11n_modulate(const uint8_t* payload, uint32_t len, uint32_t mcs, uint8_t seed, int16_t* out0, int16_t* out1, uint64_t cap_samples) {
    return tx11n_modulate(payload, len, mcs, seed, (c16*)out0, (c16*)out1, (size_t)cap_samples);
}
uint32_t sbo_tx11n_nsym(uint32_t len, uint32_t mcs, uint32_t* signalled) { return tx11n_nsym(len, mcs, signalled); }
void sbo_tx11n_preamble_tables(int16_t* lstf, int16_t* lltf, int16_t* htstf, int16_t* htltf) { tx11n_preamble_tables((c16*)lstf, (c16*)lltf, (c16*)htstf, (c16*)htltf); }

// ---- the header parsers and the back end on their own ---------------------------------------------------------------------
// T11aPLCPParser on each of n SIGNAL words, each from a context just Reset: 6 uint32 per word (Rx11a::plcp_parse_only)
void sbo_plcp11a_parse(const uint32_t* words, uint64_t n, uint32_t* out) {
    Rx11a* rx = new Rx11a();
    for (uint64_t i = 0; i < n; i++) rx->plcp_parse_only(words[i], out + 6 * i);
    delete rx;
}
// T11nSigParser on n blocks of 9 bytes in turn, one context: 8 uint32 per block (Rx11n::sig_parse_only); CF_HTRxVector starts at 0
void sbo_sig11n_parse(const uint8_t* sig9, uint64_t n, uint32_t* out) {
    Rx11n* rx = new Rx11n();
    for (uint64_t i = 0; i < n; i++) rx->sig_parse_only(sig9 + 9 * i, out + 8 * i);
    delete rx;
}
// T11aDesc -> TBB11aFrameSink as the 802.11a (chain 0) or the 802.11n (chain 1) receiver runs them, fed n decoded bytes for a frame of
// frame_length bytes: returns the error code, *crc32 = CF_11aRxVector::crc32, out = the frame buffer's first frame_length bytes
uint32_t sbo_desc_sink(int chain, const uint8_t* in, uint64_t n, uint16_t frame_length, uint8_t* out, uint32_t* crc32) {
    uint32_t e;
    if (chain == 0) { Rx11a* rx = new Rx11a(); e = rx->desc_sink_only(in, (size_t)n, frame_length); *crc32 = rx->back_crc32();
                      memcpy(out, rx->frame_bytes(), frame_length < 4096 ? frame_length : 4096); delete rx; }
    else { Rx11n* rx = new Rx11n(); e = rx->desc_sink_only(in, (size_t)n, frame_length); *crc32 = rx->crc32();
           memcpy(out, rx->frame_bytes(), frame_length < 4096 ? frame_length : 4096); delete rx; }
    return e;
}

uint32_t sbo_crc32(const uint8_t* p, uint64_t n) { uint32_t c = 0xFFFFFFFFu; for (uint64_t i = 0; i < n; i++) c = (c >> 8) ^ tables().crc32_lut[p[i] ^ (c & 0xFF)]; return ~c; }

} // extern "C"
