// sora_b200 — the spectrum and power meters: sb200_spectrum and sb200_power_meter (spectrum_kernels.cuh).
#include "handle.cuh"
#include "spectrum_kernels.cuh"
#include <math.h>

// The twiddles of every radix-4 stage size, uploaded on first use (sp_tw_off): the reference's wFFTLUT{L}_{M} tables follow the closed
// form at every size, so nothing of them is stored.
static int upload_sptab(sb200_handle* h) {
    if (h->sptab.p) return SB200_OK;
    std::vector<uint32_t> t(SB_SP_TW);
    for (uint32_t L = 16; L <= SB_SP_MAXN; L *= 2)
        for (uint32_t M = 1; M <= 3; M++)
            for (uint32_t j = 0; j < L / 4; j++) {
                const double a = 2.0 * M_PI * j * M / L;
                t[sp_tw_off(L) + (M - 1) * (L / 4) + j] = pack(mk((int)trunc(32767.0 * cos(a)), (int)trunc(-32767.0 * sin(a))));
            }
    TableArena ar; ar.add(t.data(), t.size() * 4);
    return ar.upload(h, h->sptab, "cudaMalloc spectrum twiddle table", "spectrum twiddle table upload");
}

// The rows of both meters: 1 .. 64 rows row_stride apart, row_stride at least n_in, at most 2^40 and a multiple of 4; n_in at most 2^40.
static int check_meter_rows(sb200_handle* h, uint64_t row_stride, uint32_t nrows, uint64_t n_in) {
    if (nrows < 1 || nrows > SB_SP_MAXROWS) return h->fail(SB200_E_INVALID, "nrows must be 1 .. 64");
    if (n_in > (1ull << 40)) return h->fail(SB200_E_INVALID, "n_in_samples must be at most 2^40");
    if (row_stride < n_in || (row_stride & 3u) || row_stride > (1ull << 40)) return h->fail(SB200_E_INVALID, "row_stride must be at least n_in, at most 2^40 and a multiple of 4");
    return SB200_OK;
}

// Residency and staging of both meters, after their own checks: host rows go up into the workspace, `used` samples of each (rounded to
// 4) apart; a host `out` is bound to the workspace; then launch(st, d_in, d_stride, d_out) launches the kernel between ev0 and finish_call.
template <class T, class Launch>
static int meter_run(sb200_handle* h, const int16_t* iq, uint64_t row_stride, uint32_t nrows, uint64_t used, T* out, uint64_t out_words,
                     void* cuda_stream, Launch launch) {
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    const bool in_dev = is_device_ptr(iq), out_dev = is_device_ptr(out);
    if ((in_dev && ((uintptr_t)iq & 15u)) || (out_dev && ((uintptr_t)out & 15u))) return h->fail(SB200_E_INVALID, "device input and output must be 16-byte aligned");
    CallScope call(h, st); CK(call.begin()); call.reads(iq);
    const uint32_t* d_in = (const uint32_t*)iq; uint64_t d_stride = row_stride; T* d_out; Returns ret;
    if (!in_dev) {
        d_stride = (used + 3u) & ~3ull; CK(h->iq.need(nrows * d_stride * 4ull + 16)); d_in = (const uint32_t*)h->iq.p;
        CK(cudaMemcpy2DAsync(h->iq.p, d_stride * 4ull, iq, row_stride * 4ull, used * 4ull, nrows, cudaMemcpyHostToDevice, st));
    }
    CK(ret.bind(h->iq40, out, out_words * sizeof(T), &d_out, 16));
    const int rc = launch(st, d_in, d_stride, d_out);
    return rc != SB200_OK ? rc : finish_call(h, st, ret, 0, 1);
}

// f(std::integral_constant<int, N>()) for a transform size N of 4 .. 32768 (a power of two, checked by the caller).
template <class F>
static void with_fft_len(uint32_t N, F f) {
    switch (N) {
        case 4:     f(std::integral_constant<int, 4>()); break;
        case 8:     f(std::integral_constant<int, 8>()); break;
        case 16:    f(std::integral_constant<int, 16>()); break;
        case 32:    f(std::integral_constant<int, 32>()); break;
        case 64:    f(std::integral_constant<int, 64>()); break;
        case 128:   f(std::integral_constant<int, 128>()); break;
        case 256:   f(std::integral_constant<int, 256>()); break;
        case 512:   f(std::integral_constant<int, 512>()); break;
        case 1024:  f(std::integral_constant<int, 1024>()); break;
        case 2048:  f(std::integral_constant<int, 2048>()); break;
        case 4096:  f(std::integral_constant<int, 4096>()); break;
        case 8192:  f(std::integral_constant<int, 8192>()); break;
        case 16384: f(std::integral_constant<int, 16384>()); break;
        default:    f(std::integral_constant<int, 32768>()); break;
    }
}

// One launch of k_spectrum<N>: as many CTAs as fit the device at once (at most one per work unit), grid-stride over the units.  The
// frames of N >= 16384 need more than 48 KB of shared memory (opt-in, once per handle: bit log2 N of sp_smem_set).
template <int N>
static int spectrum_launch(sb200_handle* h, cudaStream_t st, const SpArgs& a) {
    using Sh = SpShape<N>;
    if (!(h->sp_smem_set & (1u << (31 - __builtin_clz(N))))) {
        CK(cudaFuncSetAttribute(k_spectrum<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Sh::SMEM));
        h->sp_smem_set |= 1u << (31 - __builtin_clz(N));
    }
    if (!h->sms) CK(cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, h->device));
    int per_sm = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_spectrum<N>, Sh::TB, Sh::SMEM));
    const uint64_t units = (a.total + Sh::S - 1) / Sh::S, cap = (uint64_t)h->sms * (uint64_t)(per_sm > 0 ? per_sm : 1);
    CK(cudaEventRecord(h->ev0, st));
    k_spectrum<N><<<(unsigned)(units < cap ? units : cap), Sh::TB, Sh::SMEM, st>>>(a);
    return SB200_OK;
}

// Spectrum meter (k_spectrum<N>): frames of N = fft_len samples every hop samples of each row, optionally windowed, through FFT<N>,
// SquaredNorm per bin with bin 0 cleared, summed over groups of avg frames into int64 out[(r ngroups + g) N + k].
extern "C" int sb200_spectrum(sb200_handle* h, const int16_t* iq, uint64_t row_stride, uint32_t nrows, uint64_t n_in, uint32_t fft_len,
                              uint64_t hop, uint32_t avg, const int16_t* window, int64_t* out, void* cuda_stream) {
    if (!h) return SB200_E_INVALID;
    if (!iq || !out) return h->fail(SB200_E_INVALID, "null argument");
    const uint32_t N = fft_len;
    if (N < SB_SP_MINN || N > SB_SP_MAXN || (N & (N - 1))) return h->fail(SB200_E_INVALID, "fft_len must be a power of two, 4 .. 32768");
    if (hop < 1 || hop > (1ull << 32)) return h->fail(SB200_E_INVALID, "hop_samples must be 1 .. 2^32");
    if (avg < 1 || avg > (1u << 31)) return h->fail(SB200_E_INVALID, "avg must be 1 .. 2^31");
    int rc = check_meter_rows(h, row_stride, nrows, n_in);
    if (rc != SB200_OK) return rc;
    if (window)
        for (uint32_t n = 0; n < N; n++)
            if (window[n] < 0) return h->fail(SB200_E_INVALID, "window entries must be 0 .. 32767");
    const uint64_t nframes = n_in >= N ? (n_in - N) / hop + 1 : 0, ngroups = nframes / avg;
    if (ngroups == 0) return SB200_OK;
    const uint64_t used = (ngroups * avg - 1) * hop + N;   // samples of each row the used frames cover
    return meter_run(h, iq, row_stride, nrows, used, out, (uint64_t)nrows * ngroups * N, cuda_stream,
                     [&](cudaStream_t st, const uint32_t* d_in, uint64_t d_stride, int64_t* d_out) {
        const int trc = upload_sptab(h);
        if (trc != SB200_OK) return trc;
        SpArgs a; memset(&a, 0, sizeof a);
        a.x = d_in; a.stride = d_stride; a.tw = (const uint32_t*)h->sptab.p; a.hop = hop; a.avg = avg;
        a.ngroups = ngroups; a.total = (uint64_t)nrows * ngroups; a.out = d_out;
        if (window) { CK(to_device(h->spwin, window, false, N * 2ull, st, &a.win)); }
        int lrc = SB200_OK;
        with_fft_len(N, [&](auto n) { lrc = spectrum_launch<decltype(n)::value>(h, st, a); });
        return lrc;
    });
}

// Power meter (k_power_meter): TPowerMeter<N> over the blocks of N = block_len samples of each row, uint32 out[r (n_in / N) + b].
extern "C" int sb200_power_meter(sb200_handle* h, const int16_t* iq, uint64_t row_stride, uint32_t nrows, uint64_t n_in, uint32_t block_len,
                                 uint32_t* out, void* cuda_stream) {
    if (!h) return SB200_E_INVALID;
    if (!iq || !out) return h->fail(SB200_E_INVALID, "null argument");
    const uint32_t N = block_len;
    if (N < 1 || N > SB_PM_MAXN) return h->fail(SB200_E_INVALID, "block_len must be 1 .. 65536");
    const int rc = check_meter_rows(h, row_stride, nrows, n_in);
    if (rc != SB200_OK) return rc;
    const uint64_t nblocks = n_in / N;
    if (nblocks == 0) return SB200_OK;
    return meter_run(h, iq, row_stride, nrows, nblocks * N, out, (uint64_t)nrows * nblocks, cuda_stream,
                     [&](cudaStream_t st, const uint32_t* d_in, uint64_t d_stride, uint32_t* d_out) {
        if (!h->sms) CK(cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, h->device));
        const uint64_t total = (uint64_t)nrows * nblocks, threads = N < 128 ? total : 32 * total, cap = 16ull * 256 * (uint64_t)h->sms;
        const uint64_t ctas = ((threads < cap ? threads : cap) + 255) / 256;
        CK(cudaEventRecord(h->ev0, st));
        k_power_meter<<<(unsigned)ctas, 256, 0, st>>>(d_in, d_stride, nblocks, total, N, d_out);
        return SB200_OK;
    });
}
