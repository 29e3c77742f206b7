// sora_b200 — the wideband filters and the radio channel simulator: sb200_fir_decimate2, the channelizer and the combiner (fir_kernels.cuh),
// the filter-bank channelizer and combiner (bank_kernels.cuh), the arbitrary-rate channelizer and combiner (arb_kernels.cuh),
// sb200_channel_sim (sim_kernels.cuh).
#include "handle.cuh"
#include "fir_kernels.cuh"
#include "bank_kernels.cuh"
#include "arb_kernels.cuh"
#include "sim_kernels.cuh"

// Lets `kernel` use `bytes` of dynamic shared memory on this device, once per handle: bit `bit` of `set` records that it has.
template <class Mask, class Kernel>
static cudaError_t smem_once(Mask& set, uint64_t bit, Kernel kernel, int bytes) {
    if (set & bit) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) set |= (Mask)bit;
    return e;
}

// One launch of k_channelize (fir_kernels.cuh) over device buffers, between ev0 and the caller's finish_call.  Outputs per thread from D;
// channels split into groups (the input then read once per group) only as far as needed for four CTAs per multiprocessor.  ChTaps
// launches the U = 1 specialisation, BrTaps the rational one.
template <int J, class Taps>
static int channelize_launch_j(sb200_handle* h, cudaStream_t st, dim3 grid, const uint32_t* d_in, uint64_t n_in, const ChChannels& ch, uint32_t cpg,
                               uint32_t D, const Taps& T, uint32_t* d_out, uint64_t stride, uint64_t n_out) {
    constexpr bool RAT = std::is_same<Taps, BrTaps>::value;
    CK(smem_once(h->ch_smem_set, 1ull << (J + (RAT ? 32 : 0)), k_channelize<J, RAT>, SB_CH_SMEM));
    CK(cudaEventRecord(h->ev0, st));
    k_channelize<J, RAT><<<grid, SB_FIR_THREADS, SB_CH_SMEM, st>>>(d_in, n_in, (const uint32_t*)h->nco.p, ch, cpg, D, T, d_out, stride, n_out);
    return SB200_OK;
}
template <class Taps>
static int channelize_launch(sb200_handle* h, cudaStream_t st, const uint32_t* d_in, uint64_t n_in, const ChChannels& ch, uint32_t D, const Taps& T,
                             uint32_t* d_out, uint64_t stride, uint64_t n_out) {
    if (!h->sms) CK(cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, h->device));
    const uint64_t tiles = (n_in + SB_FIR_TILE - 1) / SB_FIR_TILE;
    uint32_t groups = 1;
    while (groups < ch.n && tiles * groups < 4ull * (uint64_t)h->sms) groups++;
    const uint32_t cpg = (ch.n + groups - 1) / groups; groups = (ch.n + cpg - 1) / cpg;
    const dim3 grid((unsigned)tiles, groups);
    const uint32_t need = ((SB_FIR_TILE + D - 1) / D + SB_FIR_THREADS - 1) / SB_FIR_THREADS;     // outputs per thread of a tile (and phase)
    if (need <= 1) return channelize_launch_j<1>(h, st, grid, d_in, n_in, ch, cpg, D, T, d_out, stride, n_out);
    if (need <= 2) return channelize_launch_j<2>(h, st, grid, d_in, n_in, ch, cpg, D, T, d_out, stride, n_out);
    if (need <= 4) return channelize_launch_j<4>(h, st, grid, d_in, n_in, ch, cpg, D, T, d_out, stride, n_out);
    if (need <= 8) return channelize_launch_j<8>(h, st, grid, d_in, n_in, ch, cpg, D, T, d_out, stride, n_out);
    if constexpr (std::is_same<Taps, ChTaps>::value) return channelize_launch_j<16>(h, st, grid, d_in, n_in, ch, cpg, D, T, d_out, stride, n_out);
    return h->fail(SB200_E_INVALID, "decim must be at least 3 when interp > 1");     // unreachable: D > U >= 2
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

// The Q14 NCO table of fir_kernels.cuh and sim_kernels.cuh, SB_CH_NCO words: (C, S) = (rint(2^14 cos 2 pi i / 4096), rint(2^14 sin 2 pi i / 4096)), packed like cs16.
static void fill_nco(uint32_t* t) {
    for (int i = 0; i < SB_CH_NCO; i++) { const double a = 2.0 * M_PI * i / 4096.0; t[i] = pack(mk((int)nearbyint(16384.0 * cos(a)), (int)nearbyint(16384.0 * sin(a)))); }
}
// The NCO table of the channelizers and the combiners, uploaded on first use.
static int upload_nco(sb200_handle* h) {
    if (h->nco.p) return SB200_OK;
    std::vector<uint32_t> t(SB_CH_NCO);
    fill_nco(t.data());
    TableArena ar; ar.add(t.data(), SB_CH_NCO * 4);
    return ar.upload(h, h->nco, "cudaMalloc NCO table", "NCO table upload");
}

// Checks of the channelizers' and the combiners' calls, which pass the messages in their own parameter names.  The rate pair of the
// rational-rate calls: the smaller factor 1 .. 16, the larger from it to 64, coprime.
static_assert(SB_CH_MAXINTERP == SB_CH_MAXDECIM && SB_CH_MAXRDECIM == SB_CBR_MAXINTERP, "the rational channelizer and combiner share their rate limits");
static int check_rate_pair(sb200_handle* h, uint32_t lo, uint32_t hi, const char* lo_msg, const char* hi_msg) {
    if (lo < 1 || lo > SB_CH_MAXINTERP) return h->fail(SB200_E_INVALID, lo_msg);
    if (hi < lo || hi > SB_CH_MAXRDECIM) return h->fail(SB200_E_INVALID, hi_msg);
    uint32_t a = lo, b = hi; while (b) { const uint32_t t = a % b; a = b; b = t; }
    return a == 1 ? SB200_OK : h->fail(SB200_E_INVALID, "interp and decim must be coprime");
}
// The |tap| sum of each branch (taps r, r + interp, ...) at most 65535, so that the int32 sums over one branch cannot wrap.
static int check_tap_sums(sb200_handle* h, const int16_t* taps, uint32_t ntaps, uint32_t interp) {
    for (uint32_t r = 0; r < interp; r++) {
        uint32_t asum = 0; for (uint32_t i = r; i < ntaps; i += interp) asum += (uint32_t)abs((int)taps[i]);
        if (asum > 65535u)
            return h->fail(SB200_E_INVALID, interp == 1 ? "sum of |taps| must be at most 65535 (int32 sums must not wrap)"
                                                        : "sum of |taps[k]| over k = r (mod interp) must be at most 65535 for every r (int32 sums must not wrap)");
    }
    return SB200_OK;
}
// The lengths of a channelizer: n_in at most 2^40, rows of n_out = ceil(interp n_in / decim) samples out_stride apart, out_stride at most
// 2^40 and a multiple of 4.
static int check_out_rows(sb200_handle* h, uint64_t n_in, uint32_t interp, uint32_t decim, uint64_t out_stride, uint64_t* n_out) {
    if (n_in > (1ull << 40)) return h->fail(SB200_E_INVALID, "n_in_samples must be at most 2^40");
    *n_out = (interp * n_in + decim - 1) / decim;
    if (out_stride < *n_out || (out_stride & 3u) || out_stride > (1ull << 40))
        return h->fail(SB200_E_INVALID, "out_stride must be at least ceil(interp n_in / decim), at most 2^40 and a multiple of 4");
    return SB200_OK;
}
// The lengths of a combiner: rows row_stride apart, row_stride at least n_in, at most 2^40 and a multiple of 4; n_in and n_out at most 2^40.
static int check_in_rows(sb200_handle* h, uint64_t row_stride, uint64_t n_in, uint64_t n_out) {
    if (row_stride < n_in || (row_stride & 3u) || row_stride > (1ull << 40)) return h->fail(SB200_E_INVALID, "row_stride must be at least n_in, at most 2^40 and a multiple of 4");
    if (n_in > (1ull << 40) || n_out > (1ull << 40)) return h->fail(SB200_E_INVALID, "n_in_samples and n_out_samples (interp n_in_samples) must be at most 2^40");
    return SB200_OK;
}
// The taps by branch for the rational-rate kernels: taps[r + U l] at t[r L + l].
static BrTaps branch_taps(const int16_t* taps, uint32_t ntaps, uint32_t U) {
    static_assert(sizeof(BrTaps) + sizeof(CbChannels) + 64 <= 32764 && sizeof(CbChannels) >= sizeof(ChChannels), "kernel parameters of k_channelize<J, true> and k_combine<J, true>");
    BrTaps T; memset(&T, 0, sizeof T); T.n = ntaps; T.u = U; T.L = (ntaps + U - 1) / U;
    for (uint32_t i = 0; i < ntaps; i++) T.t[(i % U) * T.L + i / U] = taps[i];
    return T;
}
// f(std::integral_constant<int, M>()) for a bank size M of 2 .. 64 (a power of two, checked by the caller): the kernels of bank_kernels.cuh
// take M as a template parameter.
template <class F>
static void with_bank_size(uint32_t M, F f) {
    switch (M) {
        case 2:  f(std::integral_constant<int, 2>()); break;
        case 4:  f(std::integral_constant<int, 4>()); break;
        case 8:  f(std::integral_constant<int, 8>()); break;
        case 16: f(std::integral_constant<int, 16>()); break;
        case 32: f(std::integral_constant<int, 32>()); break;
        default: f(std::integral_constant<int, 64>()); break;
    }
}

// Residency and staging of the channelizers (channelize_call, sb200_channelize_bank), after their own checks: a host capture goes up into
// the workspace, a host `out` is bound to the workspace with rows n_out (rounded to 4) apart, copied into the caller's rows at the end;
// then launch(st, d_in, d_out, d_stride) launches the kernel between ev0 and finish_call.
template <class Launch>
static int channelize_run(sb200_handle* h, const int16_t* iq, uint64_t n_in, uint32_t nrows, int16_t* out, uint64_t out_stride, uint64_t n_out,
                          void* cuda_stream, Launch launch) {
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    const bool in_dev = is_device_ptr(iq), out_dev = is_device_ptr(out);
    if ((in_dev && ((uintptr_t)iq & 15u)) || (out_dev && ((uintptr_t)out & 15u))) return h->fail(SB200_E_INVALID, "device input and output must be 16-byte aligned");
    CallScope call(h, st); CK(call.begin()); call.reads(iq);
    const int nrc = upload_nco(h);
    if (nrc != SB200_OK) return nrc;
    const uint32_t* d_in; uint32_t* d_out = (uint32_t*)out; uint64_t d_stride = out_stride; Returns ret;
    CK(to_device(h->iq, (const uint32_t*)iq, in_dev, n_in * 4ull, st, &d_in, 16));
    if (!out_dev) {
        d_stride = (n_out + 3u) & ~3ull; CK(h->iq40.need(nrows * d_stride * 4ull)); d_out = (uint32_t*)h->iq40.p;
        ret.bind2d(out, out_stride * 4ull, d_out, d_stride * 4ull, n_out * 4ull, nrows);
    }
    const int rc = launch(st, d_in, d_out, d_stride);
    return rc != SB200_OK ? rc : finish_call(h, st, ret, 0, 1);
}

// Wideband channelizer (fir_kernels.cuh): every channel shifted by its NCO, filtered and decimated by `decim`; channel c in row c of `out`.
// sb200_channelize is the interp = 1 case of sb200_channelize_rational with its own limits; both share the checks, staging and launch
// here (rational = false: sb200_channelize).
static int channelize_call(sb200_handle* h, const int16_t* iq, uint64_t n_in, const sb200_ddc_channel* channels, uint32_t nchannels, uint32_t interp,
                           uint32_t decim, const int16_t* taps, uint32_t ntaps, int16_t* out, uint64_t out_stride, void* cuda_stream, bool rational) {
    if (!h) return SB200_E_INVALID;
    if (!iq || !channels || !taps || !out) return h->fail(SB200_E_INVALID, "null argument");
    if (nchannels < 1 || nchannels > SB_CH_MAXCH) return h->fail(SB200_E_INVALID, "nchannels must be 1 .. 16");
    if (!rational && (decim < 1 || decim > SB_CH_MAXDECIM)) return h->fail(SB200_E_INVALID, "decim must be 1 .. 16");
    int rc = rational ? check_rate_pair(h, interp, decim, "interp must be 1 .. 16", "decim must be interp .. 64") : SB200_OK;
    if (rc != SB200_OK) return rc;
    if ((ntaps & 1u) == 0 || ntaps > interp * SB_CH_MAXTAPS)       // no limit on ntaps beyond the branch length
        return h->fail(SB200_E_INVALID, rational ? "ntaps must be odd and ceil(ntaps / interp) at most 255" : "ntaps must be odd and at most 255");
    uint64_t n_out;
    if ((rc = check_tap_sums(h, taps, ntaps, interp)) != SB200_OK || (rc = check_out_rows(h, n_in, interp, decim, out_stride, &n_out)) != SB200_OK) return rc;
    if (n_in == 0) return SB200_OK;
    return channelize_run(h, iq, n_in, nchannels, out, out_stride, n_out, cuda_stream, [&](cudaStream_t st, const uint32_t* d_in, uint32_t* d_out, uint64_t d_stride) {
        ChChannels ch; memset(&ch, 0, sizeof ch); ch.n = nchannels;
        for (uint32_t i = 0; i < nchannels; i++) { ch.inc[i] = channels[i].phase_inc; ch.phase0[i] = channels[i].phase0; }
        if (interp > 1) return channelize_launch(h, st, d_in, n_in, ch, decim, branch_taps(taps, ntaps, interp), d_out, d_stride, n_out);
        ChTaps T; memset(&T, 0, sizeof T); T.n = ntaps; for (uint32_t i = 0; i < ntaps; i++) T.t[i] = taps[i];
        return channelize_launch(h, st, d_in, n_in, ch, decim, T, d_out, d_stride, n_out);
    });
}
extern "C" int sb200_channelize(sb200_handle* h, const int16_t* iq, uint64_t n_in, const sb200_ddc_channel* channels, uint32_t nchannels, uint32_t decim,
                                const int16_t* taps, uint32_t ntaps, int16_t* out, uint64_t out_stride, void* cuda_stream) {
    return channelize_call(h, iq, n_in, channels, nchannels, 1, decim, taps, ntaps, out, out_stride, cuda_stream, false);
}
// Rational-rate channelizer: every channel shifted by its NCO, zero-stuffed by `interp`, filtered and decimated by `decim`.
extern "C" int sb200_channelize_rational(sb200_handle* h, const int16_t* iq, uint64_t n_in, const sb200_ddc_channel* channels, uint32_t nchannels,
                                         uint32_t interp, uint32_t decim, const int16_t* taps, uint32_t ntaps, int16_t* out, uint64_t out_stride, void* cuda_stream) {
    return channelize_call(h, iq, n_in, channels, nchannels, interp, decim, taps, ntaps, out, out_stride, cuda_stream, true);
}

// Polyphase filter-bank channelizer (bank_kernels.cuh): all M = nchannels channels of the uniform grid centred at (k + odd / 2) fs / M,
// filtered and decimated by `decim`, in one launch; channel k in row k of `out`.
extern "C" int sb200_channelize_bank(sb200_handle* h, const int16_t* iq, uint64_t n_in, uint32_t nchannels, uint32_t decim, uint32_t odd_stacking,
                                     const int16_t* taps, uint32_t ntaps, int16_t* out, uint64_t out_stride, void* cuda_stream) {
    if (!h) return SB200_E_INVALID;
    if (!iq || !taps || !out) return h->fail(SB200_E_INVALID, "null argument");
    const uint32_t M = nchannels, D = decim;
    if (M < 2 || M > SB_BK_MAXCH || (M & (M - 1))) return h->fail(SB200_E_INVALID, "nchannels must be a power of two, 2 .. 64");
    if (D < 1 || M % D) return h->fail(SB200_E_INVALID, "decim must divide nchannels");
    if (odd_stacking > 1u) return h->fail(SB200_E_INVALID, "odd_stacking must be 0 or 1");
    if ((ntaps & 1u) == 0 || ntaps > SB_BK_MAXTAPS) return h->fail(SB200_E_INVALID, "ntaps must be odd and at most 1023");
    uint64_t n_out; int rc;
    if ((rc = check_tap_sums(h, taps, ntaps, 1)) != SB200_OK || (rc = check_out_rows(h, n_in, 1, D, out_stride, &n_out)) != SB200_OK) return rc;
    if (n_in == 0) return SB200_OK;
    return channelize_run(h, iq, n_in, M, out, out_stride, n_out, cuda_stream, [&](cudaStream_t st, const uint32_t* d_in, uint32_t* d_out, uint64_t d_stride) {
        const BrTaps T = branch_taps(taps, ntaps, 1);  // the taps in their own order
        CK(cudaEventRecord(h->ev0, st));
        with_bank_size(M, [&](auto m) {
            k_channelize_bank<decltype(m)::value><<<(unsigned)((n_in + SB_FIR_TILE - 1) / SB_FIR_TILE), SB_FIR_THREADS, 0, st>>>(
                d_in, n_in, (const uint32_t*)h->nco.p, D, odd_stacking, T, d_out, d_stride, n_out);
        });
        return SB200_OK;
    });
}

// The checks of both arbitrary-rate calls on their resampler: the step range, t_(n_out - 1) = tau0 + (n_out - 1) step below 2^63, and
// the |tap| sum of every row of H.
static int check_arbitrary(sb200_handle* h, uint64_t tau0, uint64_t step, const int16_t* taps, uint32_t ntaps, uint64_t n_out) {
    if (step < SB_ARB_MINSTEP || step > SB_ARB_MAXSTEP) return h->fail(SB200_E_INVALID, "step must be within 2^28 .. 2^34");
    if (n_out && (tau0 >> 63 || (n_out - 1) > ((1ull << 63) - 1 - tau0) / step)) return h->fail(SB200_E_INVALID, "tau0 + (n_out - 1) step must be below 2^63");
    for (uint32_t p = 0; p < SB_ARB_ROWS; p++) {
        const int rc = check_tap_sums(h, taps + (uint64_t)p * ntaps, ntaps, 1);     // every row of H
        if (rc != SB200_OK) return rc;
    }
    return SB200_OK;
}
// The table of both arbitrary-rate kernels, staged per call into h->arbtab on `st`: the NCO (one device-to-device copy), then H packed in
// tap pairs, row p at word p * arb_row_words(ntaps) with taps 2q (low half) and 2q + 1 (high half) in word q, so that one bulk copy per
// CTA brings both in.  Calls on one handle run in order (CallScope), so a call never rewrites the table under another's kernel.
static int upload_arbtab(sb200_handle* h, cudaStream_t st, const int16_t* taps, uint32_t ntaps) {
    const uint32_t rs = arb_row_words(ntaps);
    std::vector<uint32_t> H((size_t)SB_ARB_ROWS * rs, 0u);
    for (uint32_t p = 0; p < SB_ARB_ROWS; p++)
        for (uint32_t k = 0; k < ntaps; k++) H[p * rs + k / 2] |= (uint32_t)(uint16_t)taps[(uint64_t)p * ntaps + k] << (16 * (k & 1));
    CK(h->arbtab.need((SB_CH_NCO + H.size()) * 4));
    CK(cudaMemcpyAsync(h->arbtab.p, h->nco.p, SB_CH_NCO * 4, cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync((uint32_t*)h->arbtab.p + SB_CH_NCO, H.data(), H.size() * 4, cudaMemcpyHostToDevice, st));
    return SB200_OK;
}

// Arbitrary-rate channelizer (arb_kernels.cuh): every channel shifted by its NCO and resampled at input times (tau0 + m step) / 2^32
// through the 256-phase table H; channel c in row c of `out`.  The table goes up per call (upload_arbtab).  Channels split into groups as
// in channelize_launch.
extern "C" int sb200_channelize_arbitrary(sb200_handle* h, const int16_t* iq, uint64_t n_in, const sb200_ddc_channel* channels, uint32_t nchannels,
                                          uint64_t tau0, uint64_t step, const int16_t* taps, uint32_t ntaps, int16_t* out, uint64_t out_stride,
                                          uint64_t n_out, void* cuda_stream) {
    if (!h) return SB200_E_INVALID;
    if (!iq || !channels || !taps || !out) return h->fail(SB200_E_INVALID, "null argument");
    if (nchannels < 1 || nchannels > SB_CH_MAXCH) return h->fail(SB200_E_INVALID, "nchannels must be 1 .. 16");
    if (ntaps < 1 || ntaps > SB_ARB_MAXTAPS) return h->fail(SB200_E_INVALID, "ntaps must be 1 .. 64");
    const int crc = check_arbitrary(h, tau0, step, taps, ntaps, n_out);
    if (crc != SB200_OK) return crc;
    if (n_in > (1ull << 40)) return h->fail(SB200_E_INVALID, "n_in_samples must be at most 2^40");
    if (out_stride < n_out || (out_stride & 3u) || out_stride > (1ull << 40))
        return h->fail(SB200_E_INVALID, "out_stride must be at least n_out, at most 2^40 and a multiple of 4");
    if (n_out == 0) return SB200_OK;
    return channelize_run(h, iq, n_in, nchannels, out, out_stride, n_out, cuda_stream, [&](cudaStream_t st, const uint32_t* d_in, uint32_t* d_out, uint64_t d_stride) {
        ArbArgs a; memset(&a, 0, sizeof a);
        a.ch.n = nchannels;
        bool rot = false;
        for (uint32_t i = 0; i < nchannels; i++) {
            a.ch.inc[i] = channels[i].phase_inc; a.ch.phase0[i] = channels[i].phase0;
            rot |= channels[i].phase_inc != 0u || (channels[i].phase0 >> 20) != 0u;
        }
        a.rs = arb_row_words(ntaps);
        const int trc = upload_arbtab(h, st, taps, ntaps);
        if (trc != SB200_OK) return trc;
        a.x = d_in; a.n_in = n_in; a.tab = (const uint32_t*)h->arbtab.p;
        a.tau0 = tau0; a.step = step; a.ntaps = ntaps; a.win = arb_win(step, ntaps); a.nco_words = rot ? SB_CH_NCO : 0u;
        a.y = d_out; a.stride = d_stride; a.n_out = n_out;
        if (!h->sms) CK(cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, h->device));
        const uint64_t tiles = (n_out + SB_ARB_TM - 1) / SB_ARB_TM;
        uint32_t groups = 1;
        while (groups < nchannels && tiles * groups < 4ull * (uint64_t)h->sms) groups++;
        a.chan_per_group = (nchannels + groups - 1) / groups; groups = (nchannels + a.chan_per_group - 1) / a.chan_per_group;
        CK(smem_once(h->arb_smem_set, 1u, k_channelize_arbitrary, SB_ARB_SMEM_MAX));
        CK(cudaEventRecord(h->ev0, st));
        k_channelize_arbitrary<<<dim3((unsigned)tiles, groups), SB_FIR_THREADS, arb_smem(step, ntaps, rot), st>>>(a);
        return SB200_OK;
    });
}

// The grid of k_combine<J, true>, k_combine_bank<M> and k_combine_arbitrary<J>, which take tile x + gx y of `tiles`.  A tile holds at
// least 16 outputs (32 W J per phase of k_combine, U 1024 / M of the bank, 256 J of the arbitrary-rate combiner), so n_out <= 2^40 gives
// at most 2^36 tiles: gy = ceil(tiles / (2^31 - 1)) <= 33 and
// gx = ceil(tiles / gy) < 2^31 stay within the grid limits.
static dim3 tile_grid(uint64_t tiles) {
    const uint64_t gy = (tiles + 0x7FFFFFFEull) / 0x7FFFFFFFull, gx = (tiles + gy - 1) / gy;
    return dim3((unsigned)gx, (unsigned)gy);
}

// One launch of k_combine<J, RAT> (fir_kernels.cuh) over device buffers, between ev0 and the caller's finish_call.  ChTaps launches the
// sb200_combine specialisation (D = 1, eight warps per phase, tile = x), BrTaps the rational one with W warps per phase on tile_grid;
// tiles of 32 W J outputs per phase.
template <int J, class Taps>
static int combine_launch_j(sb200_handle* h, cudaStream_t st, const uint32_t* d_in, uint64_t stride, uint64_t n_in, const CbChannels& ch, uint32_t U,
                            uint32_t D, uint32_t W, const Taps& T, uint32_t* d_out, uint64_t n_out, uint32_t accumulate) {
    constexpr bool RAT = std::is_same<Taps, BrTaps>::value;
    CK(smem_once(h->cb_smem_set, 1u << (J + (RAT ? 16 : 0)), k_combine<J, RAT>, RAT ? SB_CBR_SMEM_MAX : SB_CB_SMEM));
    const uint64_t tq = 32ull * W * J, tiles = (n_out + U * tq - 1) / (U * tq);
    const uint32_t smem = RAT ? combine_smem_r(ch.n, U, D, T.n, (uint32_t)tq) : combine_smem(ch.n, U, T.n, (uint32_t)tq);
    CK(cudaEventRecord(h->ev0, st));
    k_combine<J, RAT><<<RAT ? tile_grid(tiles) : dim3((unsigned)tiles), SB_FIR_THREADS, smem, st>>>(d_in, stride, n_in, (const uint32_t*)h->nco.p, ch, U, D, W, T, d_out, n_out, accumulate);
    return SB200_OK;
}

// Residency and staging of the combiners (combine_call, sb200_combine_bank), after their own checks: host rows go up into the workspace
// n_in (rounded to 4) apart, a host `out` is bound to the workspace (its samples uploaded first when `accumulate`), then
// launch(st, d_in, d_stride, d_out) launches the kernel between ev0 and finish_call.
template <class Launch>
static int combine_run(sb200_handle* h, const int16_t* rows, uint64_t row_stride, uint64_t n_in, uint32_t nrows, int16_t* out, uint64_t n_out,
                       uint32_t accumulate, void* cuda_stream, Launch launch) {
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    const bool in_dev = is_device_ptr(rows), out_dev = is_device_ptr(out);
    if ((in_dev && ((uintptr_t)rows & 15u)) || (out_dev && ((uintptr_t)out & 15u))) return h->fail(SB200_E_INVALID, "device rows and output must be 16-byte aligned");
    CallScope call(h, st); CK(call.begin()); call.reads(rows);
    const int nrc = upload_nco(h);
    if (nrc != SB200_OK) return nrc;
    const uint32_t* d_in = (const uint32_t*)rows; uint64_t d_stride = row_stride; uint32_t* d_out; Returns ret;
    if (!in_dev && n_in) {                             // rows n_in (rounded to 4) apart in the workspace
        d_stride = (n_in + 3u) & ~3ull; CK(h->iq.need(nrows * d_stride * 4ull + 16)); d_in = (const uint32_t*)h->iq.p;
        CK(cudaMemcpy2DAsync(h->iq.p, d_stride * 4ull, rows, row_stride * 4ull, n_in * 4ull, nrows, cudaMemcpyHostToDevice, st));
    }
    CK(ret.bind(h->iq40, (uint32_t*)out, n_out * 4ull, &d_out, 16));
    if (accumulate && !out_dev) {                      // the caller's samples go up into the workspace before the launch adds onto them
        call.reads(out); CK(cudaMemcpyAsync(d_out, out, n_out * 4ull, cudaMemcpyHostToDevice, st));
    }
    const int rc = launch(st, d_in, d_stride, d_out);
    return rc != SB200_OK ? rc : finish_call(h, st, ret, 0, 1);
}

// Wideband combiner (fir_kernels.cuh): every row zero-stuffed by `interp`, filtered (and decimated by `decim`), shifted up by its NCO,
// scaled and summed into `out` (or onto it).  sb200_combine is the decim = 1, n_out = interp n_in case of sb200_combine_rational with its
// own limits and kernel specialisation; both share the checks, staging and launch here (rational = false: sb200_combine).
static int combine_call(sb200_handle* h, const int16_t* rows, uint64_t row_stride, uint64_t n_in, const sb200_duc_channel* channels, uint32_t nchannels,
                        uint32_t interp, uint32_t decim, const int16_t* taps, uint32_t ntaps, int16_t* out, uint64_t n_out, uint32_t accumulate,
                        void* cuda_stream, bool rational) {
    if (!h) return SB200_E_INVALID;
    if (!rows || !channels || !taps || !out) return h->fail(SB200_E_INVALID, "null argument");
    if (nchannels < 1 || nchannels > SB_CH_MAXCH) return h->fail(SB200_E_INVALID, "nchannels must be 1 .. 16");
    if (!rational && (interp < 1 || interp > SB_CH_MAXDECIM)) return h->fail(SB200_E_INVALID, "interp must be 1 .. 16");
    int rc = rational ? check_rate_pair(h, decim, interp, "decim must be 1 .. 16", "interp must be decim .. 64") : SB200_OK;
    if (rc != SB200_OK) return rc;
    if ((ntaps & 1u) == 0 || ntaps > (rational ? SB_CBR_MAXTAPS : SB_CH_MAXTAPS) || (ntaps + interp - 1) / interp > SB_CH_MAXTAPS)
        return h->fail(SB200_E_INVALID, rational ? "ntaps must be odd, at most 4095 and ceil(ntaps / interp) at most 255" : "ntaps must be odd and at most 255");
    if ((rc = check_tap_sums(h, taps, ntaps, interp)) != SB200_OK) return rc;
    if (accumulate > 1u) return h->fail(SB200_E_INVALID, "accumulate must be 0 or 1");
    for (uint32_t i = 0; i < nchannels; i++)
        if (channels[i].gain > 65535u) return h->fail(SB200_E_INVALID, "gain must be at most 65535");
    if ((rc = check_in_rows(h, row_stride, n_in, n_out)) != SB200_OK) return rc;
    if (n_out == 0) return SB200_OK;
    return combine_run(h, rows, row_stride, n_in, nchannels, out, n_out, accumulate, cuda_stream,
                       [&](cudaStream_t st, const uint32_t* d_in, uint64_t d_stride, uint32_t* d_out) {
        CbChannels ch; memset(&ch, 0, sizeof ch); ch.n = nchannels;
        for (uint32_t i = 0; i < nchannels; i++) { ch.inc[i] = channels[i].phase_inc; ch.phase0[i] = channels[i].phase0; ch.gain[i] = channels[i].gain; }
        if (!rational) {                               // tiles of 1024, 512 or 256 input samples: the largest whose shared memory fits SB_CB_SMEM (256 always does)
            ChTaps T; memset(&T, 0, sizeof T); T.n = ntaps; for (uint32_t i = 0; i < ntaps; i++) T.t[i] = taps[i];
            if (combine_smem(nchannels, interp, ntaps, 4 * SB_FIR_THREADS) <= SB_CB_SMEM) return combine_launch_j<4>(h, st, d_in, d_stride, n_in, ch, interp, 1, 8, T, d_out, n_out, 0);
            if (combine_smem(nchannels, interp, ntaps, 2 * SB_FIR_THREADS) <= SB_CB_SMEM) return combine_launch_j<2>(h, st, d_in, d_stride, n_in, ch, interp, 1, 8, T, d_out, n_out, 0);
            return combine_launch_j<1>(h, st, d_in, d_stride, n_in, ch, interp, 1, 8, T, d_out, n_out, 0);
        }
        const BrTaps T = branch_taps(taps, ntaps, interp);
        // 32 W J outputs per phase: the largest of 1024 .. 32 whose shared memory fits SB_CBR_SMEM, else 32 (within SB_CBR_SMEM_MAX)
        static const uint32_t kj[6] = {4, 2, 1, 1, 1, 1}, kw[6] = {8, 8, 8, 4, 2, 1};
        int p = 0;
        while (p < 5 && combine_smem_r(nchannels, interp, decim, ntaps, 32u * kw[p] * kj[p]) > SB_CBR_SMEM) p++;
        if (kj[p] == 4) return combine_launch_j<4>(h, st, d_in, d_stride, n_in, ch, interp, decim, kw[p], T, d_out, n_out, accumulate);
        if (kj[p] == 2) return combine_launch_j<2>(h, st, d_in, d_stride, n_in, ch, interp, decim, kw[p], T, d_out, n_out, accumulate);
        return combine_launch_j<1>(h, st, d_in, d_stride, n_in, ch, interp, decim, kw[p], T, d_out, n_out, accumulate);
    });
}
extern "C" int sb200_combine(sb200_handle* h, const int16_t* rows, uint64_t row_stride, uint64_t n_in, const sb200_duc_channel* channels, uint32_t nchannels,
                             uint32_t interp, const int16_t* taps, uint32_t ntaps, int16_t* out, void* cuda_stream) {
    return combine_call(h, rows, row_stride, n_in, channels, nchannels, interp, 1, taps, ntaps, out, interp * n_in, 0, cuda_stream, false);
}
// Rational-rate combiner: every row zero-stuffed by `interp`, filtered, decimated by `decim`, shifted up by its NCO, scaled and summed into
// n_out outputs, added onto out's samples when `accumulate`.
extern "C" int sb200_combine_rational(sb200_handle* h, const int16_t* rows, uint64_t row_stride, uint64_t n_in, const sb200_duc_channel* channels,
                                      uint32_t nchannels, uint32_t interp, uint32_t decim, const int16_t* taps, uint32_t ntaps, int16_t* out,
                                      uint64_t n_out, uint32_t accumulate, void* cuda_stream) {
    return combine_call(h, rows, row_stride, n_in, channels, nchannels, interp, decim, taps, ntaps, out, n_out, accumulate, cuda_stream, true);
}

// Polyphase filter-bank combiner (bank_kernels.cuh): the M = nchannels rows onto the uniform grid centred at (k + odd / 2) fs / M,
// interpolated by `interp`, summed into n_out outputs (added onto out's samples when `accumulate`) in one launch, on tile_grid's grid of
// tiles of U 1024 / M outputs.
extern "C" int sb200_combine_bank(sb200_handle* h, const int16_t* rows, uint64_t row_stride, uint64_t n_in, uint32_t nchannels, uint32_t interp,
                                  uint32_t odd_stacking, const int16_t* taps, uint32_t ntaps, int16_t* out, uint64_t n_out, uint32_t accumulate,
                                  void* cuda_stream) {
    if (!h) return SB200_E_INVALID;
    if (!rows || !taps || !out) return h->fail(SB200_E_INVALID, "null argument");
    const uint32_t M = nchannels, U = interp;
    if (M < 2 || M > SB_BK_MAXCH || (M & (M - 1))) return h->fail(SB200_E_INVALID, "nchannels must be a power of two, 2 .. 64");
    if (U < 1 || M % U) return h->fail(SB200_E_INVALID, "interp must divide nchannels");
    if (odd_stacking > 1u) return h->fail(SB200_E_INVALID, "odd_stacking must be 0 or 1");
    if ((ntaps & 1u) == 0 || ntaps > SB_BK_MAXTAPS || ntaps > 2 * SB_CBK_SPAN / M * U)
        return h->fail(SB200_E_INVALID, "ntaps must be odd, at most 1023 and at most 2048 interp / nchannels");
    if (accumulate > 1u) return h->fail(SB200_E_INVALID, "accumulate must be 0 or 1");
    const int rc = check_in_rows(h, row_stride, n_in, n_out);
    if (rc != SB200_OK) return rc;
    if (n_out == 0) return SB200_OK;
    return combine_run(h, rows, row_stride, n_in, M, out, n_out, accumulate, cuda_stream,
                       [&](cudaStream_t st, const uint32_t* d_in, uint64_t d_stride, uint32_t* d_out) {
        const BrTaps T = branch_taps(taps, ntaps, 1);  // the taps in their own order
        const uint64_t to = U * (SB_CBK_SPAN / M), tiles = (n_out + to - 1) / to;
        CK(cudaEventRecord(h->ev0, st));
        with_bank_size(M, [&](auto m) {
            k_combine_bank<decltype(m)::value><<<tile_grid(tiles), SB_FIR_THREADS, 0, st>>>(d_in, d_stride, n_in, (const uint32_t*)h->nco.p, U, odd_stacking, T,
                                                                                           d_out, n_out, accumulate);
        });
        return SB200_OK;
    });
}

// One launch of k_combine_arbitrary<J> (arb_kernels.cuh) on tile_grid's grid of tiles of 256 J outputs, between ev0 and the caller's
// finish_call.  Bit J of arb_smem_set (bit 0 is k_channelize_arbitrary's).
template <int J>
static int combine_arbitrary_launch_j(sb200_handle* h, cudaStream_t st, ArbCbArgs& a) {
    constexpr uint32_t TM = SB_FIR_THREADS * J;
    CK(smem_once(h->arb_smem_set, 1u << J, k_combine_arbitrary<J>, J == 1 ? SB_ARB_CB_SMEM_MAX : SB_CBR_SMEM));
    a.win = arb_win(a.step, a.ntaps, TM);
    CK(cudaEventRecord(h->ev0, st));
    k_combine_arbitrary<J><<<tile_grid((a.n_out + TM - 1) / TM), SB_FIR_THREADS, arb_combine_smem(a.ch.n, a.step, a.ntaps, a.nco_words != 0, TM), st>>>(a);
    return SB200_OK;
}

// Arbitrary-rate combiner (arb_kernels.cuh): every row resampled at row times (tau0 + n step) / 2^32 through the 256-phase table H, shifted
// up by its NCO, scaled and summed into n_out outputs (added onto out's samples when `accumulate`) in one launch.  Tiles of 1024, 512 or 256
// outputs: the largest whose shared memory fits SB_CBR_SMEM (256 fits SB_ARB_CB_SMEM_MAX at every limit).  The table goes up per call
// (upload_arbtab), residency and staging are combine_run's.
extern "C" int sb200_combine_arbitrary(sb200_handle* h, const int16_t* rows, uint64_t row_stride, uint64_t n_in, const sb200_duc_channel* channels,
                                       uint32_t nchannels, uint64_t tau0, uint64_t step, const int16_t* taps, uint32_t ntaps, int16_t* out,
                                       uint64_t n_out, uint32_t accumulate, void* cuda_stream) {
    if (!h) return SB200_E_INVALID;
    if (!rows || !channels || !taps || !out) return h->fail(SB200_E_INVALID, "null argument");
    if (nchannels < 1 || nchannels > SB_CH_MAXCH) return h->fail(SB200_E_INVALID, "nchannels must be 1 .. 16");
    if (ntaps < 1 || ntaps > SB_ARB_MAXTAPS) return h->fail(SB200_E_INVALID, "ntaps must be 1 .. 64");
    int rc = check_arbitrary(h, tau0, step, taps, ntaps, n_out);
    if (rc != SB200_OK) return rc;
    if (accumulate > 1u) return h->fail(SB200_E_INVALID, "accumulate must be 0 or 1");
    for (uint32_t i = 0; i < nchannels; i++)
        if (channels[i].gain > 65535u) return h->fail(SB200_E_INVALID, "gain must be at most 65535");
    if ((rc = check_in_rows(h, row_stride, n_in, n_out)) != SB200_OK) return rc;
    if (n_out == 0) return SB200_OK;
    return combine_run(h, rows, row_stride, n_in, nchannels, out, n_out, accumulate, cuda_stream,
                       [&](cudaStream_t st, const uint32_t* d_in, uint64_t d_stride, uint32_t* d_out) {
        ArbCbArgs a; memset(&a, 0, sizeof a);
        a.ch.n = nchannels;
        bool rot = false;
        for (uint32_t i = 0; i < nchannels; i++) {
            a.ch.inc[i] = channels[i].phase_inc; a.ch.phase0[i] = channels[i].phase0; a.ch.gain[i] = channels[i].gain;
            rot |= channels[i].phase_inc != 0u || (channels[i].phase0 >> 20) != 0u;
        }
        const int trc = upload_arbtab(h, st, taps, ntaps);
        if (trc != SB200_OK) return trc;
        a.x = d_in; a.stride = d_stride; a.n_in = n_in; a.tab = (const uint32_t*)h->arbtab.p;
        a.tau0 = tau0; a.step = step; a.ntaps = ntaps; a.rs = arb_row_words(ntaps); a.nco_words = rot ? SB_CH_NCO : 0u;
        a.y = d_out; a.n_out = n_out; a.accumulate = accumulate;
        if (arb_combine_smem(nchannels, step, ntaps, rot, 4 * SB_FIR_THREADS) <= SB_CBR_SMEM) return combine_arbitrary_launch_j<4>(h, st, a);
        if (arb_combine_smem(nchannels, step, ntaps, rot, 2 * SB_FIR_THREADS) <= SB_CBR_SMEM) return combine_arbitrary_launch_j<2>(h, st, a);
        return combine_arbitrary_launch_j<1>(h, st, a);
    });
}

// The table of sb200_channel_sim (sim_kernels.cuh), uploaded on first use: the NCO of fill_nco, then H (256 rows of 8 Q14 taps, packed in
// pairs like cs16) and LNT, from the closed forms of include/sora_b200.h.  I0 is its power series (tests/sim_model.py sums the same one).
static double sim_i0(double x) {
    double s = 1.0, t = 1.0; const double q = x * x / 4.0;
    for (int k = 1; k < 32; k++) { t = t * (q / ((double)k * k)); s = s + t; }
    return s;
}
static int upload_simtab(sb200_handle* h) {
    if (h->simtab.p) return SB200_OK;
    std::vector<uint32_t> t(SB_SIM_TAB);
    fill_nco(t.data());
    const double i05 = sim_i0(5.0);
    for (int p = 0; p < 256; p++) {
        int hv[8];
        for (int k = 0; k < 8; k++) {
            const double d = k - 3 - p / 256.0, sinc = d == 0.0 ? 1.0 : sin(M_PI * d) / (M_PI * d);
            hv[k] = (int)nearbyint(16384.0 * sinc * sim_i0(5.0 * sqrt(1.0 - (d / 4.0) * (d / 4.0))) / i05);
        }
        for (int k = 0; k < 4; k++) t[SB_CH_NCO + 4 * p + k] = pack(mk(hv[2 * k], hv[2 * k + 1]));
    }
    for (int j = 0; j < SB_SIM_LNT; j++) t[SB_CH_NCO + SB_SIM_H + j] = (uint32_t)nearbyint(-log((2048.0 + j + 0.5) / 4096.0) * 16777216.0);
    TableArena ar; ar.add(t.data(), SB_SIM_TAB * 4);
    return ar.upload(h, h->simtab, "cudaMalloc channel simulator table", "channel simulator table upload");
}

// Rows of length n at l * A + r * B (l < N, r < R) are pairwise disjoint: |dl A + dr B| >= n for every (dl, dr) != 0, |dl| < N, |dr| < R.
// For each dr > 0 only the dl nearest -dr B / A (clamped) can come closest.
static bool rows_disjoint(uint64_t A, uint64_t B, uint32_t N, uint32_t R, uint64_t n) {
    if (N > 1 && A < n) return false;                  // dr = 0, dl = 1
    for (uint32_t dr = 1; dr < R; dr++) {
        const double b = (double)dr * (double)B;
        const long long c = N > 1 ? (long long)floor(-b / (double)A) : 0;
        for (long long dl = c - 1; dl <= c + 2; dl++) {
            if (dl <= -(long long)N || dl >= (long long)N) continue;
            const __int128 v = (__int128)dl * (__int128)A + (__int128)dr * (__int128)B;
            if ((v < 0 ? -v : v) < (__int128)n) return false;
        }
    }
    return true;
}

// One launch of k_channel_sim<J> (sim_kernels.cuh), between ev0 and the caller's finish_call.
template <int J>
static int sim_launch_j(sb200_handle* h, cudaStream_t st, SimArgs& a) {
    const uint32_t tm = SB_FIR_THREADS * J;
    CK(smem_once(h->sim_smem_set, 1u << J, k_channel_sim<J>, sim_smem(SB_SIM_MAXROWS, SB_SIM_MAXROWS, SB_SIM_MAXTAPS, tm)));
    a.ntiles = (uint32_t)((a.n_out + tm - 1) / tm);
    CK(cudaEventRecord(h->ev0, st));
    k_channel_sim<J><<<(unsigned)((uint64_t)a.ntiles * a.nlinks), SB_FIR_THREADS, sim_smem(a.T, a.R, a.L, tm), st>>>(a);
    return SB200_OK;
}

// Radio channel simulator (sim_kernels.cuh): every link's input rows through its clock offset, taps, carrier offset and noise.  Tiles of 2048
// outputs for T <= 2 and of 1024 for T = 4, which keeps the shared memory at most 68 KB.
extern "C" int sb200_channel_sim(sb200_handle* h, const int16_t* x, uint64_t in_link_stride, uint64_t in_row_stride, uint32_t ntx, uint64_t n_in,
                                 const sb200_link* links, const int16_t* taps, uint32_t ntaps, uint32_t nlinks,
                                 uint64_t seed, int16_t* y, uint64_t out_link_stride, uint64_t out_row_stride, uint32_t nrx, uint64_t n_out, void* cuda_stream) {
    if (!h) return SB200_E_INVALID;
    if (!x || !links || !taps || !y) return h->fail(SB200_E_INVALID, "null argument");
    if (ntx < 1 || ntx > SB_SIM_MAXROWS || nrx < 1 || nrx > SB_SIM_MAXROWS) return h->fail(SB200_E_INVALID, "ntx and nrx must be 1 .. 4");
    if (ntaps < 1 || ntaps > SB_SIM_MAXTAPS) return h->fail(SB200_E_INVALID, "ntaps must be 1 .. 64");
    if (n_in > (1ull << 30) || n_out > (1ull << 30)) return h->fail(SB200_E_INVALID, "n_in and n_out must be at most 2^30");
    if ((in_link_stride | in_row_stride | out_link_stride | out_row_stride) & 3u) return h->fail(SB200_E_INVALID, "strides must be multiples of 4");
    if ((in_link_stride | in_row_stride | out_link_stride | out_row_stride) >> 40) return h->fail(SB200_E_INVALID, "strides must be below 2^40");
    if (!rows_disjoint(out_link_stride, out_row_stride, nlinks, nrx, n_out)) return h->fail(SB200_E_INVALID, "output rows overlap");
    if (nlinks == 0 || n_out == 0) return SB200_OK;
    const uint32_t T = ntx, R = nrx, L = ntaps;
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaSetDevice(h->device));
    const bool x_dev = is_device_ptr(x), y_dev = is_device_ptr(y), l_dev = is_device_ptr(links), t_dev = is_device_ptr(taps);
    if ((x_dev && ((uintptr_t)x & 15u)) || (y_dev && ((uintptr_t)y & 15u))) return h->fail(SB200_E_INVALID, "device x and y must be 16-byte aligned");
    if ((t_dev && ((uintptr_t)taps & 3u)) || (l_dev && ((uintptr_t)links & 7u))) return h->fail(SB200_E_INVALID, "device taps must be 4-byte and device links 8-byte aligned");
    const uint64_t ntap_words = (uint64_t)nlinks * R * T * L;
    if (!l_dev && !t_dev) {                            // host tables: checked here
        for (uint32_t l = 0; l < nlinks; l++) {
            const sb200_link& k = links[l];
            if (k.step < (1ull << 32) - (1ull << 24) || k.step > (1ull << 32) + (1ull << 24)) return h->fail(SB200_E_INVALID, "step must be within 2^32 +- 2^24");
            if (k.tau0 >= (1ull << 62)) return h->fail(SB200_E_INVALID, "tau0 must be below 2^62");
            if (k.noise_q8 >= (1u << 24)) return h->fail(SB200_E_INVALID, "noise_q8 must be below 2^24");
        }
        for (uint64_t i = 0; i < (uint64_t)nlinks * R; i++) {
            uint32_t sum = 0; const int16_t* g = taps + i * T * L * 2;
            for (uint32_t q = 0; q < 2 * T * L; q++) sum += (uint32_t)abs((int)g[q]);
            if (sum > 65535u) return h->fail(SB200_E_INVALID, "sum of |g.re| + |g.im| over t and j must be at most 65535 for every link and output row");
        }
    }
    CallScope call(h, st); CK(call.begin()); call.reads(x); call.reads(links); call.reads(taps);
    const sb200_link* d_links; const uint32_t* d_taps;
    CK(to_device(h->simlink, links, l_dev, nlinks * sizeof(sb200_link), st, &d_links));
    CK(to_device(h->simtap, (const uint32_t*)taps, t_dev, ntap_words * 4ull, st, &d_taps));
    if (l_dev || t_dev) {                              // a table on the device: its limits checked there, one 4-byte read-back
        CK(h->slotchk.need(8));
        CK(cudaMemsetAsync(h->slotchk.p, 0, 4, st));
        const uint64_t nt = (uint64_t)nlinks * R;
        k_sim_check<<<(unsigned)((nt + 255) / 256), 256, 0, st>>>(d_links, (const int16_t*)d_taps, nlinks, R, T, L, (uint32_t*)h->slotchk.p);
        uint32_t bad = 0;
        CK(cudaMemcpyAsync(&bad, h->slotchk.p, 4, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (bad) return h->fail(SB200_E_INVALID, "a link record or tap sum is out of its limits (step, tau0, noise_q8 or sum of |g| > 65535)");
    }
    const int trc = upload_simtab(h);
    if (trc != SB200_OK) return trc;
    SimArgs a; memset(&a, 0, sizeof a);
    a.T = T; a.R = R; a.L = L; a.nlinks = nlinks; a.n_in = n_in; a.n_out = n_out; a.seed = seed;
    a.links = d_links; a.taps = d_taps; a.tab = (const uint32_t*)h->simtab.p;
    a.in_link = in_link_stride; a.in_row = in_row_stride; a.out_link = out_link_stride; a.out_row = out_row_stride;
    if (x_dev) a.x = (const uint32_t*)x;
    else {                                             // the whole span of the rows, strides kept (rows may share samples: a stride may be 0)
        const uint64_t span = (uint64_t)(nlinks - 1) * in_link_stride + (uint64_t)(T - 1) * in_row_stride + n_in;
        CK(to_device(h->iq, (const uint32_t*)x, false, span * 4ull, st, &a.x, 16));
    }
    Returns ret;
    if (y_dev) a.y = (uint32_t*)y;
    else {                                             // rows n_out (rounded to 4) apart in the workspace, copied into the caller's rows row by row
        const uint64_t no4 = (n_out + 3) & ~3ull;
        CK(h->iq40.need((uint64_t)nlinks * R * no4 * 4ull + 16)); a.y = (uint32_t*)h->iq40.p; a.out_row = no4; a.out_link = R * no4;
        for (uint32_t r = 0; r < R; r++)
            ret.bind2d(y + 2 * r * out_row_stride, (nlinks > 1 ? out_link_stride : n_out) * 4ull, a.y + r * no4, R * no4 * 4ull, n_out * 4ull, nlinks);
    }
    const int rc = T <= 2 ? sim_launch_j<8>(h, st, a) : sim_launch_j<4>(h, st, a);
    return rc != SB200_OK ? rc : finish_call(h, st, ret, 0, 1);
}
