/* sora_b200 — C ABI of the Hopper (sm_90a) 802.11 receive baseband.
 *
 * This is the drop-in boundary for Sora's dot11 RX hot path.  Every entry point states which reference
 * interface it stands behind (paths relative to the reference tree):
 *
 *   sb200_create / sb200_destroy   <->  BB11ARxContextInit            kernel/inc/bb/bba.h:191-201
 *                                       BB11aDemodContext::Init       kernel/bb/demod11/fb11ademod_config.hpp:105-121
 *   sb200_rx11a_batch              <->  the sub-graph ds2 .. fsink of CreateDemodGraph11a_40M
 *                                       kernel/bb/demod11/fb11ademod_config.hpp:169-242, driven like RxThread
 *                                       kernel/bb/demod11/fb11a_demod.cpp:29-81; legacy shape BB11ARxCarrierSense +
 *                                       BB11ARxFrameDemod, kernel/inc/bb/bba.h:203-262
 *   sb200_rx11b_batch              <->  the whole graph behind TMemSamples of CreateDemodGraph (802.11b)
 *                                       kernel/bb/demod11/fb11bdemod_config.hpp:123-180, driven like MAC11b_Receive
 *                                       kernel/bb/demod11/fb11b_demod.cpp:26-79; legacy shape BB11BSpd + BB11BRx,
 *                                       kernel/inc/bb/bbb.h:176-248
 *   sb200_viterbi_k7               <->  T11aViterbi<TR_MAX,N_IN,DEPTH,LOOKAHEAD>::Filter
 *                                       kernel/bb/Brick11/src/viterbi.hpp:104-237 (BASELINE config #5)
 *   sb200_rx11a_taps               <->  BB_DEBUG `_dump_symbol` taps  kernel/brick/inc/bb_debug.h:5-41
 *
 * Conventions: plain pointers and sizes only; every function returns 0 on success or a negative SB200_E_* code
 * and never throws.  Sample and result buffers may live in host or device memory (detected per pointer); host
 * buffers are staged through the handle's pinned/device workspaces on `stream`.  When a call touches memory:
 *   - a call returns once it no longer needs any host buffer of the caller: it synchronises `stream` before
 *     returning when a result buffer is host memory, or when an input it copies is page-locked host memory
 *     (sb200_host_alloc, cudaHostRegister); pageable inputs are copied out before the call returns;
 *   - with device buffers and host-resident tables a call does not wait for `stream`: its work stays queued;
 *   - device-resident slot or payload tables cost a read-back (one stream synchronisation), except a repeated
 *     receive call on the same slot table under the option slot_table_immutable; sb200_rx11a_batch_ex at 44 Msps
 *     checks the slot table of its resampled captures the same way;
 *   - calls on one handle execute in the order they were made, whatever streams they are given (a call on another
 *     stream than the previous one waits for it on the device, not on the host).
 * One handle may be used by one host thread at a time; separate handles may run concurrently.
 * There is NO CPU fallback: if no CUDA device is usable the create call fails.
 */
#ifndef SORA_B200_H
#define SORA_B200_H
#include <stdint.h>
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

#define SB200_OK              0
#define SB200_E_INVALID      (-1)
#define SB200_E_CUDA         (-2)
#define SB200_E_NOMEM        (-3)
#define SB200_E_NODEVICE     (-4)

/* Frame status values = CF_Error::error_code of the reference (brick/inc/stdfacade.h:10-12,
 * Brick11/src/ieee80211facade.hpp:10-19) plus one engine-only code. */
#define SB200_FRAME_OK            0x00000001u  /* E_ERROR_FRAME_OK */
#define SB200_FRAME_FAILED        0x8000FFFFu  /* E_ERROR_FAILED */
#define SB200_FRAME_PLCP_FAIL     0x80000005u  /* E_ERROR_PLCP_HEADER_FAIL */
#define SB200_FRAME_CRC32_FAIL    0x80000006u  /* E_ERROR_CRC32_FAIL */
#define SB200_FRAME_SFD_FAIL      0x80000004u  /* E_ERROR_SFD_FAIL */
#define SB200_FRAME_SFD_TIMEOUT   0x80000008u  /* E_ERROR_SFD_TIMEOUT */
#define SB200_FRAME_SYNC_TIMEOUT  0x80000009u  /* E_ERROR_SYNC_TIMEOUT */
#define SB200_FRAME_NONE          0x8000F001u  /* slot exhausted before any frame event (the reference just runs out of samples) */

#define SB200_CR_12 0   /* Brick11/src/ieee80211const.h:13-18 */
#define SB200_CR_23 1
#define SB200_CR_34 2

typedef struct sb200_handle sb200_handle;

typedef struct sb200_cfg {
    uint32_t cca_pwr_threshold;   /* CF_11CCA::cca_pwr_threshold, 0 = reference default 1000*1000 (fb11ademod_config.hpp:107) */
    uint32_t reserved[7];
} sb200_cfg;

typedef struct sb200_frame_result {   /* CF_11aRxVector + CF_Error + CF_11CCA + CF_CFOffset after the first event of a slot */
    uint32_t status;       /* SB200_FRAME_* */
    uint32_t rate_kbps;    /* CF_11aRxVector::data_rate_kbps */
    uint32_t length;       /* CF_11aRxVector::frame_length (PSDU bytes incl. FCS) */
    uint32_t crc32;        /* CF_11aRxVector::crc32: the received FCS */
    uint32_t nsym;         /* CF_11aRxVector::total_symbols (SIGNAL + data) */
    uint32_t detect_index; /* 20 Msps sample index, relative to the slot, of the first sample routed to the demod branch */
    int16_t  cfo_est;      /* CF_CFOffset::CFO_est (FP_RAD per 20 Msps sample) */
    uint16_t peak_index;   /* CF_11CCA::cca_peak_index */
} sb200_frame_result;

int  sb200_create(int device, const sb200_cfg* cfg, sb200_handle** out);
void sb200_destroy(sb200_handle* h);
const char* sb200_last_error(const sb200_handle* h);
/* number of kernels this handle has launched so far (bench.py's gpu_launches) */
uint64_t sb200_launch_count(const sb200_handle* h);
/* what the most recent sb200_rx11a_batch call with a HOST iq buffer really sent over the link: sample bytes copied host -> device, the number
 * of pipeline chunks and how many of them the host threads gathered first (option host_decimate); bench.py's e2e.h2d_bytes_per_step */
int sb200_last_transfer(const sb200_handle* h, uint64_t* h2d_bytes, uint32_t* chunks, uint32_t* chunks_gathered);
/* name of the Viterbi kernel the most recent launch used ("k_viterbi_lane": one lane per code block, large batches; "k_viterbi_re": four
 * lanes per code block; option "viterbi_lane_min" = smallest launch, in code blocks, the first one takes) — bench.py's roofline.kernel */
const char* sb200_last_viterbi_kernel(const sb200_handle* h);
/* device time (ms) of the kernels of the most recent *_batch / viterbi call, measured with CUDA events on `stream` */
float sb200_last_kernel_ms(sb200_handle* h);
/* per-kernel device times (ms) of the most recent sb200_rx11a_batch: [0] carrier sense, [1] OFDM front end,
 * [2] Viterbi+descramble+CRC, [3] result pack */
int sb200_last_kernel_times(sb200_handle* h, float* ms4);
/* Tunables.  "chunk_frames" (default 4096): when the IQ buffer is HOST memory, calls with more slots are cut into chunks whose
 * host->device copy, OFDM front end and Viterbi overlap on three streams; 0 = one pass on the caller's stream.
 * "chunk_frames_device" (default 0 = off): the same for device-resident IQ.  sb200_last_kernel_times needs an un-chunked call.
 * "ht_mcs_limit" (default 11): the first 802.11n MCS index the HT-SIG parser refuses.  11 is the reference as it ships (PHY_11n.hpp:496-501:
 *   MCS 8..10 decode, anything else ends with E_ERROR_PLCP_HEADER_FAIL); 15 sends MCS 11..14 through the 16-QAM / 64-QAM branches the
 *   reference's receive graph already carries (fb11ndemod_config.hpp:196-236, demapper11n.hpp:199-309, deinterleaver_11n.hpp) — rate 1/2,
 *   3/4 and 2/3 Viterbi, stream parser blocks of 2 / 3 bits.  Values 9 .. 15.
 * "host_decimate" (default 0 = off): number of host threads (the caller's included) that gather the even samples of every slot of a chunk
 * into pinned staging memory before the copy — TDownSample2 (Brick11/src/samples.hpp:27-49) keeps samples 0 and 2 of every 4, so the
 * 802.11a chain never reads the odd ones and only half of a host-resident 40 Msps capture has to cross PCIe.  Results are identical.
 * "host_decimate_mix" (default 1): with host_decimate on, 1 = per chunk the call either gathers on the host threads or — when the copies
 *   already queued would run out before a gather could finish — sends the chunk as it is, so that the link and the host cores are both kept
 *   busy (link rate and gather cost are estimated from the call's own events); 0 = every chunk is gathered; 2 = alternate (tests).
 * "viterbi_lane_min" (default 16384), "viterbi_lane_max" (default 49152): launches of lane_min .. lane_max code blocks are decoded by the
 *   one-lane-per-code-block Viterbi kernel (32 code blocks per warp, history ring in global memory: the fewest instructions, but it needs a
 *   large batch to fill the machine, and its ring traffic costs more than it saves on the largest ones), the others by the
 *   four-lanes-per-code-block kernel (ring in shared memory).  Results are identical.  lane_min 0 and lane_max 0xFFFFFFFF = always,
 *   lane_min 0xFFFFFFFF = never.
 * Slot tables (frame_off/frame_len) are bounds-checked against iq_total_samples on EVERY call, host- or device-resident (a device table costs one
 * small reduction kernel and an 8-byte read-back).  "slot_table_immutable" (default 0): set to 1 to promise that a device-resident table is not
 * rewritten while the same pointers, count and total are passed again; only then is the check (and the host copy the chunked path needs) cached. */
int sb200_set_option(sb200_handle* h, const char* name, uint64_t value);

/* Decode `nframes` independent capture slots.  Slot i is iq[2*frame_off[i] .. 2*(frame_off[i]+frame_len[i])) int16
 * (interleaved I,Q; 40 Msps COMPLEX16 stream as TMemSamples would feed it), processed from a fresh context exactly as
 * the reference graph processes a dump file, up to its first frame event.  out_bytes row i (out_stride bytes) receives
 * the PSDU (FCS included), res[i] the verdict.  iq_total_samples bounds the iq buffer. */
int sb200_rx11a_batch(sb200_handle* h, const int16_t* iq, uint64_t iq_total_samples,
                      const uint64_t* frame_off, const uint32_t* frame_len, uint32_t nframes,
                      uint8_t* out_bytes, uint32_t out_stride, sb200_frame_result* res, void* cuda_stream);

/* One continuous capture holding any number of frames (SURVEY.md §8(f) rank 1): frames are reported in order exactly as the
 * reference's RxThread finds them (fb11a_demod.cpp:29-81) — after each event the graph restarts on the next 28-sample block and
 * only the DC estimate carries over.  res / out_bytes / sample_index are HOST arrays of max_frames entries; sample_index[i] =
 * CF_MemSamples::mem_sample_index (40 Msps samples consumed) when event i was seen; detect_index is relative to the restart. */
int sb200_rx11a_stream(sb200_handle* h, const int16_t* iq, uint64_t nsamples, uint32_t max_frames, uint8_t* out_bytes, uint32_t out_stride,
                       sb200_frame_result* res, uint32_t* sample_index, uint32_t* nframes_out, void* cuda_stream);

/* Many continuous captures in one call: capture s = samples [stream_off[s], stream_off[s] + stream_len[s]); results of capture s sit in
 * res / out_bytes / sample_index rows s * max_frames .. (+ nframes_out[s]).  Every pass decodes the next frame of all captures that still
 * have samples, so the device works on a full batch while each capture keeps RxThread's sequential semantics.  Tables and results are
 * host memory; iq may be host or device. */
int sb200_rx11a_streams(sb200_handle* h, const int16_t* iq, uint64_t iq_total_samples, const uint64_t* stream_off, const uint32_t* stream_len,
                        uint32_t nstreams, uint32_t max_frames, uint8_t* out_bytes, uint32_t out_stride, sb200_frame_result* res,
                        uint32_t* sample_index, uint32_t* nframes_out, void* cuda_stream);

/* 2:1 anti-alias FIR decimator for a COMPLEX16 capture — the "FIR decimation / channel-select" stage; an extension: the reference's 802.11a
 * graph only drops every other sample (TDownSample2, Brick11/src/samples.hpp:27-49).  out[m] = sat16((sum_k taps[k] * x[2m + k - (ntaps-1)/2]
 * + 2^14) >> 15), x = 0 outside the buffer, re and im independently; taps Q15, ntaps odd <= 63, taps = NULL: built-in 31-tap half-band low-pass.
 * out receives (n_in + 1) / 2 samples and is what sb200_rx11a_batch_ex(sample_rate_mhz = 20) takes.  Host or device pointers (device: 16-byte aligned).
 * It computes what sb200_channelize below computes for channel (0, 0) and decim 2, without that call's tap-sum and stride checks. */
int sb200_fir_decimate2(sb200_handle* h, const int16_t* iq, uint64_t n_in_samples, const int16_t* taps, uint32_t ntaps, int16_t* out, void* cuda_stream);

/* Wideband channelizer: several channels of one COMPLEX16 capture x[0 .. n_in) (x = 0 outside it) shifted to 0 Hz, low-pass filtered and
 * decimated by D = decim, in one call; an extension without a reference counterpart.  For channel (phase_inc, phase0) and every output
 * m in 0 .. n_out = ceil(n_in / D):
 *     phi(n)  = (phase0 + (uint32)n * phase_inc) mod 2^32             n = absolute input index: stateless, no serial NCO
 *     (C, S)  = NCO[phi(n) >> 20]                                      4096 entries, Q14: C = rint(16384 cos(2 pi i / 4096)), S = rint(16384 sin(2 pi i / 4096))
 *     v(n).re = sat16((x.re * C + x.im * S + 2^13) >> 14)            x * e^{-j theta}: moves +f_c to 0 Hz
 *     v(n).im = sat16((x.im * C - x.re * S + 2^13) >> 14)
 *     y[m]    = sat16((sum_k taps[k] * v(D m + k - c) + 2^14) >> 15)   c = (ntaps - 1) / 2, int32 accumulator, re and im independently
 * The NCO is Q14 so that phase_inc = phase0 = 0 is the identity bit for bit; with D = 2 that channel is sb200_fir_decimate2.  A channel
 * centred at f_c in a capture at f_s takes phase_inc = round(f_c / f_s * 2^32) mod 2^32 (negative f_c wraps).
 * Channel c goes to out[c * out_stride .. + n_out) (samples), so stream_off[c] = c * out_stride and stream_len[c] = n_out hand the rows
 * to sb200_rx11a_streams / sb200_rx11b_streams / sb200_rx11n_streams as they are.  iq and out may be host or device pointers (device:
 * 16-byte aligned, and the call is then asynchronous on the stream); channels and taps are host arrays.  Limits (SB200_E_INVALID):
 * 1 <= nchannels <= 16, 1 <= decim <= 16, ntaps odd and <= 255, sum |taps| <= 65535 (the accumulator cannot wrap), out_stride >= n_out,
 * a multiple of 4 and <= 2^40, n_in <= 2^40.  One kernel launch; sb200_last_kernel_ms times it. */
typedef struct sb200_ddc_channel { uint32_t phase_inc; uint32_t phase0; } sb200_ddc_channel;
int sb200_channelize(sb200_handle* h, const int16_t* iq, uint64_t n_in_samples, const sb200_ddc_channel* channels, uint32_t nchannels, uint32_t decim,
                     const int16_t* taps, uint32_t ntaps, int16_t* out, uint64_t out_stride_samples, void* cuda_stream);

/* Rational-rate channelizer: sb200_channelize with the rate changed by U / D (U = interp, D = decim) instead of 1 / D, so that one capture
 * feeds receivers of rates that no whole-number D reaches from it (802.11b at 44 Msps and OFDM at 40 Msps out of 160 or 176 Msps);
 * an extension without a reference counterpart.  For channel (phase_inc, phase0), c = (ntaps - 1) / 2 and every output
 * m in 0 .. n_out = ceil(U n_in / D):
 *     v(n)  = the Q14 NCO rotation of x(n) by sb200_channelize, with the phase of the absolute INPUT index n
 *     z(i)  = v(i / U) if i mod U == 0 and 0 <= i / U < n_in, else 0          zero-stuffing
 *     y[m]  = sat16((sum_k taps[k] * z(D m + k - c) + 2^14) >> 15)             int32 accumulator, re and im independently
 * Output m stands at input time D m / U: output 0 lines up with input 0.  Only the taps k = c - D m (mod U) meet a non-zero z, so an
 * interpolation filter has a DC gain of U (each branch near unity) and the accumulator limit is per branch, as in sb200_combine.  With
 * interp = 1 this is sb200_channelize, bit for bit, with decim up to 64.  Rows, residency, alignment and staging as in sb200_channelize;
 * the rows go to sb200_rx11a_streams / sb200_rx11b_streams / sb200_rx11n_streams as they are.  Limits (SB200_E_INVALID, nothing launched):
 * 1 <= interp <= 16, interp <= decim <= 64, gcd(interp, decim) = 1 (rate reduction only), ntaps odd with ceil(ntaps / interp) <= 255, for
 * every residue r mod interp the sum of |taps[k]| over k = r (mod interp) <= 65535, 1 <= nchannels <= 16, out_stride >= n_out, a multiple
 * of 4 and <= 2^40, n_in <= 2^40.  One kernel launch; sb200_last_kernel_ms times it. */
int sb200_channelize_rational(sb200_handle* h, const int16_t* iq, uint64_t n_in_samples, const sb200_ddc_channel* channels, uint32_t nchannels,
                              uint32_t interp, uint32_t decim, const int16_t* taps, uint32_t ntaps, int16_t* out, uint64_t out_stride_samples,
                              void* cuda_stream);

/* Arbitrary-rate channelizer: sb200_channelize with the rate changed by any factor between x16 and /4, so that captures at rates derived
 * from 30.72 MHz (30.72, 61.44, 122.88 Msps) reach the receivers at 40 and 44 Msps; an extension without a reference counterpart.  For
 * channel (phase_inc, phase0), c = floor((ntaps - 1) / 2) and every output m in 0 .. n_out = n_out_samples:
 *     v(n)    = the Q14 NCO rotation of x(n) by sb200_channelize, at the phase of the absolute INPUT index n   (x = 0 outside [0, n_in))
 *     t_m     = tau0 + m * step                                  exact, uint64 (Q32.32 input samples); the limits keep it below 2^63
 *     t'      = t_m + 2^23,  i = t' >> 32,  p = (t' >> 24) & 255
 *     y[m]    = sat16((sum_{k < ntaps} H[p][k] * v(i - c + k) + 2^13) >> 14)     int32, re and im independently
 *     H[p][k] = taps[p * ntaps + k]                               256 rows of ntaps Q14 taps; row p is the fractional delay p / 256
 * Output m stands at input time t_m / 2^32, rounded to 1/256 of an input sample.  The table is Q14, not the channelizers' Q15, as in
 * sb200_channel_sim, so that a unit impulse is representable: with step = 2^32, tau0 = d 2^32, phase_inc = phase0 = 0 and row 0 the unit
 * impulse at k = c, y[m] = x[m + d] bit for bit; with ntaps = 8 and sb200_channel_sim's H this is that call's stage 1.  A capture at fs_in
 * to fs_out takes step = round(2^32 fs_in / fs_out) (api.arbitrary_step) and a low-pass table cut by the lower of the two rates
 * (api.arbitrary_taps).  There is one (tau0, step) and one table per call: rows of two rates (802.11b at 44 Msps beside OFDM at 40 Msps)
 * take two calls, as with sb200_channelize_rational.  n_out is the caller's choice; outputs past the input read zeros.  Larger decimations
 * go through sb200_channelize or sb200_channelize_bank with a whole decim first (245.76 -> 122.88 Msps, then this call).  Channel c goes
 * to out[c * out_stride .. + n_out) (samples): the rows go to sb200_rx11a_streams / sb200_rx11b_streams / sb200_rx11n_streams as they are.
 * iq and out may be host or device pointers (device: 16-byte aligned, and the call is then asynchronous on the stream); channels and taps
 * are host arrays.  Limits (SB200_E_INVALID, nothing launched): 1 <= nchannels <= 16, 1 <= ntaps <= 64, 2^28 <= step <= 2^34,
 * tau0 + (n_out - 1) step < 2^63, for every row p sum_k |H[p][k]| <= 65535 (the accumulator cannot wrap), n_in <= 2^40, out_stride >=
 * n_out, a multiple of 4 and <= 2^40.  n_out = 0 launches nothing.  One kernel launch; sb200_last_kernel_ms times it. */
int sb200_channelize_arbitrary(sb200_handle* h, const int16_t* iq, uint64_t n_in_samples, const sb200_ddc_channel* channels, uint32_t nchannels,
                               uint64_t tau0, uint64_t step, const int16_t* taps, uint32_t ntaps, int16_t* out, uint64_t out_stride_samples,
                               uint64_t n_out_samples, void* cuda_stream);

/* Polyphase filter-bank channelizer: every channel of a uniform grid of M = nchannels channels, centred at (k + o/2) fs / M for k in
 * 0 .. M-1 (k >= M/2 wraps to negative frequencies), out of one COMPLEX16 capture x[0 .. n_in) (x = 0 outside it), filtered by one set
 * of taps and decimated by D = decim, in one pass; an extension without a reference counterpart.  o = odd_stacking: 0 puts channel 0 at
 * 0 Hz, 1 at fs / 2M.  For channel k, c = (ntaps - 1) / 2 and every output m in 0 .. n_out = ceil(n_in / D):
 *     n_j       = D m + j - c                                                   absolute input index met by tap j
 *     (C, S)    = NCO[((2k + o) n_j (2048 / M)) mod 4096]                       the Q14 table of sb200_channelize
 *     y_k[m].re = sat16((sum_j taps[j] (x.re C + x.im S) + 2^28) >> 29)         int64, one rounding
 *     y_k[m].im = sat16((sum_j taps[j] (x.im C - x.re S) + 2^28) >> 29)
 * This is channel k of sb200_channelize with phase_inc = (2k + o) 2^31 / M and phase0 = 0, except that the rotated sample is kept exact
 * instead of rounded to int16: the two agree within 2 LSB where neither saturates.  The cost grows with ntaps / D + M^2 / D per input
 * sample, not with M ntaps / D.  Channel k goes to out[k * out_stride .. + n_out) (samples): the rows go to sb200_rx11a_streams /
 * sb200_rx11b_streams / sb200_rx11n_streams as they are.  iq and out may be host or device pointers (device: 16-byte aligned, and the
 * call is then asynchronous on the stream); taps is a host array.  Limits (SB200_E_INVALID, nothing launched): nchannels a power of two,
 * 2 .. 64; decim divides nchannels; odd_stacking 0 or 1; ntaps odd, 1 .. 1023; sum |taps| <= 65535 (every branch sum fits int32);
 * out_stride >= n_out, a multiple of 4 and <= 2^40; n_in <= 2^40.  One kernel launch; sb200_last_kernel_ms times it. */
int sb200_channelize_bank(sb200_handle* h, const int16_t* iq, uint64_t n_in_samples, uint32_t nchannels, uint32_t decim, uint32_t odd_stacking,
                          const int16_t* taps, uint32_t ntaps, int16_t* out, uint64_t out_stride_samples, void* cuda_stream);

/* Polyphase filter-bank combiner, the transmit counterpart of sb200_channelize_bank: M = nchannels rows x_k[0 .. n_in) of COMPLEX16 (row k
 * at rows + k * row_stride samples, x_k = 0 outside it) interpolated by U = interp, row k moved to the centre (k + o/2) fs / M of the grid
 * of sb200_channelize_bank (o = odd_stacking; api.bank_centres gives the centres), and summed into one capture y[0 .. n_out) in one pass;
 * an extension without a reference counterpart.  With c = (ntaps - 1) / 2, T[i] = NCO[i 2048 / M] (the Q14 table of sb200_channelize) and
 * sigma(n) = (-1)^(o floor(n / M)), every output n in 0 .. n_out = n_out_samples is, in int64 and exact up to the two roundings:
 *     W_p(i) = (sum_k x_k(i) T[(2k + o) p mod 2M] + 2^13) >> 14        p = 0 .. M-1; rotating up: re = x.re C - x.im S, im = x.im C + x.re S
 *     acc(n) = sum_i taps[c + U i - n] W_{n mod M}(i)                   over 0 <= i < n_in, 0 <= c + U i - n < ntaps
 *     a(n)   = accumulate ? out[n] as it was before the call : 0
 *     y(n)   = sat16(a(n) + ((sigma(n) acc(n) + 2^14) >> 15))
 * Channel k is sb200_combine channel {(2k + o) 2^31 / M, 0, 4096} at the same U, rotated by the phase of the absolute output index as
 * there: for n = M a + p that channel's table entry is NCO[(2k + o) n 2048 / M mod 4096] = sigma(n) T[(2k + o) p mod 2M].  The bank rounds
 * twice in all where sb200_combine rounds after the filter and after every rotation, so where nothing saturates the two differ by at most
 * 1.2072 K + 0.5 B / 32768 + 0.5 per component, K the number of non-zero rows and B the largest per-branch sum of |taps|.  Proof: against
 * the exact value, each of sb200_combine's channels is off by its filter rounding (0.5 per component) carried through the Q14 rotation,
 * 0.5 (|C| + |S|)_max / 16384 = 0.5 * 23170 / 16384 <= 0.7072, plus the rotation's own 0.5; a zero row adds nothing.  The bank's W is off
 * by at most 0.5, which the one branch of taps an output meets scales by at most B / 32768 before the final rounding adds 0.5.
 * A row sent with (M, U, o) comes back from sb200_channelize_bank with (M, D = U, o), aligned at the same index.  With E_p and O_p the
 * even-k and odd-k halves of the sum, W_p = E_p + O_p and W_{p+M/2} = j^o (E_p - O_p), exact in int64 before the rounding
 * (NCO[i + 2048] = -NCO[i], NCO[i + 1024] = j NCO[i]): the kernel computes half the products of the direct sum.
 * Unlike the other wideband calls there is no tap-sum limit: |W| < 2^22 and |acc| < 2^47 at every limit.  There are no per-channel
 * gains: a Q12 gain on x before the IDFT would need a third rounding or more than int64 range; scale the rows instead.
 * n_out is the caller's choice: outputs past the rows' support are a(n) plus the filter's tail.  n_out = 0 launches nothing and n_in = 0
 * means all-zero rows.  rows and out may be host or device pointers (device: 16-byte aligned, and the call is then asynchronous on the
 * stream; a host out is uploaded first when accumulate = 1); taps is a host array.  Limits (SB200_E_INVALID, nothing launched): nchannels a
 * power of two, 2 .. 64; interp divides nchannels; odd_stacking 0 or 1; ntaps odd, 1 .. 1023 and ntaps <= 2048 interp / nchannels (that
 * is, ceil(ntaps / U) M <= 2048); row_stride >= n_in, a multiple of 4 and <= 2^40; n_in <= 2^40; n_out <= 2^40; accumulate 0 or 1.
 * One kernel launch; sb200_last_kernel_ms times it. */
int sb200_combine_bank(sb200_handle* h, const int16_t* rows, uint64_t row_stride_samples, uint64_t n_in_samples,
                       uint32_t nchannels, uint32_t interp, uint32_t odd_stacking, const int16_t* taps, uint32_t ntaps,
                       int16_t* out, uint64_t n_out_samples, uint32_t accumulate, void* cuda_stream);

/* Wideband combiner, the transmit counterpart of sb200_channelize: K = nchannels rows x_k[0 .. n_in) of COMPLEX16 at the channel rate
 * (row k at rows + k * row_stride samples) interpolated by U = interp, each moved to its centre frequency, scaled and summed into one
 * capture y[0 .. U n_in) at the wideband rate; an extension without a reference counterpart.  For channel k = {phase_inc, phase0, gain}
 * and every output n:
 *     z_k(i)    = x_k(i / U) if i mod U == 0 and 0 <= i / U < n_in, else 0        zero-stuffing
 *     u_k(n)    = sat16((sum_j taps[j] * z_k(n + j - c) + 2^14) >> 15)          c = (ntaps - 1) / 2, int32, re and im independently
 *     phi(n)    = (phase0 + (uint32)n * phase_inc) mod 2^32, (C, S) = NCO[phi >> 20]   the Q14 table of sb200_channelize, n = absolute output index
 *     v_k(n).re = sat16((u.re * C - u.im * S + 2^13) >> 14)                     u * e^{+j theta}: moves 0 Hz to +f_c
 *     v_k(n).im = sat16((u.im * C + u.re * S + 2^13) >> 14)
 *     y(n)      = sat16(sum_k ((v_k(n) * gain_k + 2^11) >> 12))                 gain in Q12 (4096 = unity), int32, re and im independently
 * The NCO convention is the channelizer's with the opposite sign: a channel sent with (phase_inc, phase0) is recovered by sb200_channelize
 * with the same pair.  Only the taps j = c - n (mod U) meet a non-zero z, so an interpolation filter may have a DC gain of U (each branch
 * near unity); the limit that keeps the accumulator from wrapping is per branch.  The tail of the filter past U n_in is cut, as the
 * channelizer cuts its edges: to keep it, pad the rows with zeros.  rows and out may be host or device pointers (device: 16-byte aligned,
 * and the call is then asynchronous on the stream); channels and taps are host arrays.  Limits (SB200_E_INVALID, nothing launched):
 * 1 <= nchannels <= 16, 1 <= interp <= 16, ntaps odd and <= 255, for every residue r mod U the sum of |taps[j]| over j = r (mod U) <= 65535,
 * gain <= 65535, row_stride >= n_in, a multiple of 4 and <= 2^40, interp * n_in <= 2^40.  One kernel launch; sb200_last_kernel_ms times it.
 * Input is COMPLEX16 only: COMPLEX8 rows (the 802.11b and legacy transmitters) are widened first, for example x << 7. */
typedef struct sb200_duc_channel { uint32_t phase_inc; uint32_t phase0; uint32_t gain; } sb200_duc_channel;
int sb200_combine(sb200_handle* h, const int16_t* rows, uint64_t row_stride_samples, uint64_t n_in_samples, const sb200_duc_channel* channels,
                  uint32_t nchannels, uint32_t interp, const int16_t* taps, uint32_t ntaps, int16_t* out, void* cuda_stream);

/* Rational-rate combiner, the transmit counterpart of sb200_channelize_rational: sb200_combine with the rate changed by U / D (U = interp,
 * D = decim) instead of U, so that rows of rates that no whole-number U reaches go into one capture (802.11b at 44 Msps into 160 Msps with
 * (40, 11), OFDM at 40 Msps into 176 Msps with (22, 5)); an extension without a reference counterpart.  For channel k = {phase_inc, phase0,
 * gain}, c = (ntaps - 1) / 2 and every output n in 0 .. n_out = n_out_samples:
 *     z_k(i)  = x_k(i / U) if i mod U == 0 and 0 <= i / U < n_in, else 0              zero-stuffing
 *     u_k(n)  = sat16((sum_j taps[j] * z_k(D n + j - c) + 2^14) >> 15)                int32, re and im independently
 *     v_k(n)  = u_k(n) rotated UP by NCO[(phase0 + (uint32)n * phase_inc) >> 20]      sb200_combine's rotation, n = absolute output index
 *     a(n)    = accumulate ? out[n] as it was before the call : 0
 *     y(n)    = sat16(a(n) + sum_k ((v_k(n) * gain_k + 2^11) >> 12))                  int32, re and im independently
 * Output n stands at input time D n / U: output 0 lines up with input 0, the channelizer's convention, so a row sent with (U, D, phase_inc,
 * phase0) comes back from sb200_channelize_rational with (D, U) and the same pair.  Only the taps j = c - D n (mod U) meet a non-zero z,
 * so the accumulator limit is per branch.  n_out is the caller's choice: outputs past the rows' support are a(n) plus the filter's tails, so
 * rows need no trailing zeros.  accumulate = 1 adds the call onto out with one saturation per call, so that one capture holds rows of two
 * rates (two calls into one buffer).  With decim = 1, interp <= 16, ntaps <= 255, n_out = U n_in and accumulate = 0 this is sb200_combine,
 * bit for bit.  rows and out may be host or device pointers (device: 16-byte aligned, and the call is then asynchronous on the stream; a
 * host out is uploaded first when accumulate = 1); channels and taps are host arrays.  Limits (SB200_E_INVALID, nothing launched):
 * 1 <= decim <= 16, decim <= interp <= 64, gcd(interp, decim) = 1 (rate increase only), ntaps odd, <= 4095 and ceil(ntaps / interp) <= 255,
 * for every residue r mod interp the sum of |taps[j]| over j = r (mod interp) <= 65535, gain <= 65535, 1 <= nchannels <= 16,
 * row_stride >= n_in, a multiple of 4 and <= 2^40, n_in <= 2^40, n_out <= 2^40, accumulate 0 or 1.  n_out = 0 launches nothing and
 * n_in = 0 means all-zero rows.  One kernel launch; sb200_last_kernel_ms times it. */
int sb200_combine_rational(sb200_handle* h, const int16_t* rows, uint64_t row_stride_samples, uint64_t n_in_samples,
                           const sb200_duc_channel* channels, uint32_t nchannels, uint32_t interp, uint32_t decim,
                           const int16_t* taps, uint32_t ntaps, int16_t* out, uint64_t n_out_samples, uint32_t accumulate,
                           void* cuda_stream);

/* Arbitrary-rate combiner, the transmit counterpart of sb200_channelize_arbitrary: sb200_combine_rational with the rate changed by any
 * factor between x16 and /4, so that rows at 40 and 44 Msps go into captures at rates derived from 30.72 MHz (30.72, 61.44, 122.88 Msps;
 * 44 -> 122.88 Msps is U / D = 768 / 275); an extension without a reference counterpart.  K = nchannels rows x_k[0 .. n_in) of COMPLEX16,
 * row k at rows + k * row_stride samples, x_k = 0 outside [0, n_in).  For channel k = {phase_inc, phase0, gain}, c = floor((ntaps - 1) / 2)
 * and every output n in 0 .. n_out = n_out_samples:
 *     t_n     = tau0 + n * step                                 exact, uint64 (Q32.32 row samples); the limits keep it below 2^63
 *     t'      = t_n + 2^23,  i = t' >> 32,  p = (t' >> 24) & 255
 *     u_k(n)  = sat16((sum_{j < ntaps} H[p][j] * x_k(i - c + j) + 2^13) >> 14)      int32, re and im independently
 *     v_k(n)  = u_k(n) rotated UP by NCO[(phase0 + (uint32)n * phase_inc) >> 20]   sb200_combine's rotation, n = absolute output index
 *     a(n)    = accumulate ? out[n] as it was before the call : 0
 *     y(n)    = sat16(a(n) + sum_k ((v_k(n) * gain_k + 2^11) >> 12))               int32, re and im independently
 *     H[p][j] = taps[p * ntaps + j]                              256 rows of ntaps Q14 taps; row p is the fractional delay p / 256
 * Stage u is sb200_channelize_arbitrary's resampler with the same table; stages v and y are sb200_combine_rational's rotation, gain, sum
 * and accumulate.  Rows at fs_rows into a capture at fs_capture take step = round(2^32 fs_rows / fs_capture) (api.arbitrary_step) and the
 * table api.arbitrary_taps(fs_rows, fs_capture, ntaps, passband), whose default stop band puts the cut at the rows' Nyquist rate, which
 * removes the images.  There is one (tau0, step) and one table per call: rows of two rates (802.11b at 44 Msps beside OFDM at 40 Msps) take
 * two calls into one buffer, the second with accumulate = 1, as with sb200_combine_rational.  Pins:
 *   - with one row, channel {0, 0, 4096} and accumulate = 0 the call is sb200_channelize_arbitrary's channel (0, 0) with the same tau0,
 *     step, table and n_out, bit for bit: NCO[0] = (16384, 0), and the rotation and the Q12 gain of 4096 are then exact identities (so with
 *     sb200_channel_sim's H and 8 taps it is also that call's stage 1);
 *   - with row 0 the unit impulse at j = c, step = 2^32 and tau0 = d 2^32 it is a pure shift, y[n] = x[n + d];
 *   - a row sent with (phase_inc, phase0), tau0 = 0 and step s comes back from sb200_channelize_arbitrary with the same pair and step
 *     ~ 2^64 / s; not bit for bit (two filters, two roundings), but the receivers decode it.
 * rows and out may be host, page-locked or device pointers (device: 16-byte aligned, and the call is then asynchronous on the stream; a
 * host out is uploaded first when accumulate = 1); channels and taps are host arrays.  Limits (SB200_E_INVALID, nothing launched):
 * 1 <= nchannels <= 16, 1 <= ntaps <= 64, 2^28 <= step <= 2^34, tau0 + (n_out - 1) step < 2^63, for every row p sum_j |H[p][j]| <= 65535
 * (the accumulator cannot wrap), gain <= 65535, row_stride >= n_in, a multiple of 4 and <= 2^40, n_in <= 2^40, n_out <= 2^40, accumulate
 * 0 or 1.  n_out = 0 launches nothing and n_in = 0 means all-zero rows.  One kernel launch; sb200_last_kernel_ms times it. */
int sb200_combine_arbitrary(sb200_handle* h, const int16_t* rows, uint64_t row_stride_samples, uint64_t n_in_samples,
                            const sb200_duc_channel* channels, uint32_t nchannels, uint64_t tau0, uint64_t step,
                            const int16_t* taps, uint32_t ntaps, int16_t* out, uint64_t n_out_samples,
                            uint32_t accumulate, void* cuda_stream);

/* Radio channel simulator: nlinks independent links, each from T = ntx input rows x_t[0 .. n_in) to R = nrx output rows y_r[0 .. n_out) of
 * COMPLEX16 through a sampling-clock offset, multipath, a carrier offset and seeded noise, in the manner of GNU Radio's channel_model; an
 * extension without a reference counterpart.  Row t of link l is at x + l * in_link_stride + t * in_row_stride samples, row r of y at
 * y + l * out_link_stride + r * out_row_stride.  For link l with record {tau0, step, phase_inc, phase0, noise_q8}, L = ntaps complex Q14
 * taps g[r][t][j] (taps + ((l R + r) T + t) L * 2: re, im) and every output row r and sample m:
 *  1. sample clock   tau = tau0 + m * step (uint64, Q32.32 input samples), t' = tau + 2^23, i = t' >> 32, p = (t' >> 24) & 255,
 *                    s_t(m) = sat16((sum_{k=0..7} H[p][k] * x_t(i - 3 + k) + 2^13) >> 14)      int32, re and im independently,
 *                    x_t = 0 outside [0, n_in), s_t(m) = 0 for m < 0;
 *                    H[p][k] = rint(16384 sinc(d) I0(5 sqrt(1 - (d / 4)^2)) / I0(5)), d = k - 3 - p / 256: row 0 is the unit impulse at
 *                    k = 3, so step = 2^32 with a whole-sample tau0 is a pure delay, bit for bit (Q14, not Q15, for that reason)
 *  2. multipath      u_r(m) = sat16((sum_t sum_{j<L} g[r][t][j] (x) s_t(m - j) + 2^13) >> 14)     complex product, int32
 *                    (re = g.re s.re - g.im s.im, im = g.re s.im + g.im s.re)
 *  3. carrier offset theta = phase0 + m * phase_inc (mod 2^32), (C, S) = NCO[theta >> 20] (the Q14 table of sb200_channelize),
 *                    v.re = sat16((u.re C - u.im S + 2^13) >> 14), v.im = sat16((u.im C + u.re S + 2^13) >> 14)
 *  4. noise          (w0, w1, w2, w3) = Philox4x32-10(counter (u32(m >> 1), u32(m >> 33), r, l), key (u32(seed), u32(seed >> 32))),
 *                    (wa, wb) = (w0, w1) for even m, (w2, w3) for odd m; a = wa | 1, e = clz32(a), mant = u32(a << e) >> 20 in [2048, 4095],
 *                    Lq = 11629080 e + LNT[mant - 2048], LNT[j] = rint(-ln((2048 + j + 0.5) / 4096) 2^24), Rn = floor(sqrt(2 Lq)) exactly,
 *                    (Cn, Sn) = NCO[wb >> 20], n.re = (sigma Rn Cn + 2^33) >> 34, n.im = (sigma Rn Sn + 2^33) >> 34 (int64, arithmetic
 *                    shifts, sigma = noise_q8), y_r(m) = (sat16(v.re + n.re), sat16(v.im + n.im))
 * Stage 4 is a fixed-point Box-Muller on the NCO table: the noise has a standard deviation of noise_q8 / 256 LSB per real component, and
 * Rn is at most about 6.7 sigma; noise_q8 = 0 adds none.  Every output is a closed form of (link, r, m): any window of outputs equals the
 * same slice of the whole.  Limits (SB200_E_INVALID, nothing launched): 1 <= ntx, nrx <= 4, 1 <= ntaps <= 64, step in
 * [2^32 - 2^24, 2^32 + 2^24], tau0 < 2^62, n_in and n_out <= 2^30, noise_q8 < 2^24, for every link and r the sum over t and j of
 * |g.re| + |g.im| <= 65535 (the accumulator cannot wrap), the four strides multiples of 4 and below 2^40, and no two output rows overlapping.  Every pointer
 * may be host or device memory (device x and y 16-byte aligned, device taps 4-byte aligned, device links 8-byte aligned); when links or
 * taps are on the device their limits are checked there (one small kernel and one read-back).  One simulation launch; sb200_last_kernel_ms
 * times it.  The two outputs of sb200_tx11n_batch go in as the rows of a link (in_row_stride = the distance between them). */
typedef struct sb200_link { uint64_t tau0, step; uint32_t phase_inc, phase0, noise_q8, reserved; } sb200_link;
int sb200_channel_sim(sb200_handle* h, const int16_t* x, uint64_t in_link_stride, uint64_t in_row_stride, uint32_t ntx, uint64_t n_in,
                      const sb200_link* links, const int16_t* taps, uint32_t ntaps, uint32_t nlinks,
                      uint64_t seed, int16_t* y, uint64_t out_link_stride, uint64_t out_row_stride, uint32_t nrx, uint64_t n_out, void* cuda_stream);

/* Spectrum meter: TSpecMeter<N> of the reference spectrum analyser (kernel/sdl/inc/sdlmeasure.hpp:66-121; kernel/sdl/exe/speanalyzer/
 * specanalyzer.cpp feeds it through THanningWin<16>), with overlap, a window and averaging.  nrows rows of COMPLEX16, row r at
 * iq + r * row_stride samples: a capture (nrows = 1) or the rows a channelizer wrote.  With N = fft_len, frame f of a row covers samples
 * [f hop, f hop + N), nframes = n_in >= N ? (n_in - N) / hop + 1 : 0 (no partial frame is formed, as the pin queue would form none).  Per frame:
 *     x'[n] = window ? (x[n] * w[n] + 2^14) >> 15 : x[n]            re and im independently, w Q15 in [0, 32767]
 *     X     = FFT<N>(x')                                             exactly FFTSSEEx<N> and the bit-reversed read-out of FFT<N>
 *             (core/inc/fft_r4dif.h:11-141): radix-4 stages FFTSSE<N'> with the input >> 2, saturating adds and subtracts, mul_j, mul_shift
 *             by the twiddle (pmaddwd, >> 15, the wrapping pack; twiddles (trunc(32767 cos(2 pi j M / N')), trunc(-32767 sin(2 pi j M / N'))),
 *             M = 1, 2, 3), down to FFTSSEEx<4> (input >> 2) or FFTSSEEx<8> (input >> 3) with their XOR (one's-complement) negations
 *     P[k]  = re^2 + im^2                                            wrapping int32 (SquaredNorm = pmaddwd(x, x): -32768 twice is INT32_MIN)
 *     P[0]  = 0
 *     out[(r * ngroups + g) * N + k] = sum of P_f[k] over f in [g avg, (g + 1) avg)    int64, ngroups = nframes / avg
 * Bins are in natural FFT order, as TSpecMeter emits them: bin k is at +k fs / N (k < N / 2) or (k - N) fs / N.  Trailing frames that do
 * not fill a group are not used.  With window = NULL, hop = N and avg = 1 every output row is TSpecMeter<N>'s output row bit for bit.
 * hop gives overlapped (Welch) frames, the window keeps a strong channel's leakage off a weak neighbour, and avg keeps the output small (at
 * avg = 1 it is twice the size of the capture).  iq and out may be host, page-locked or device pointers (device: 16-byte aligned, and the
 * call is then asynchronous on the stream); window is a host array.  Limits (SB200_E_INVALID, nothing launched): fft_len a power of two,
 * 4 .. 32768; 1 <= hop <= 2^32; 1 <= avg <= 2^31; 1 <= nrows <= 64; row_stride >= n_in, a multiple of 4 and <= 2^40; n_in <= 2^40; window
 * entries in [0, 32767].  ngroups = 0 launches nothing.  One kernel launch; sb200_last_kernel_ms times it. */
int sb200_spectrum(sb200_handle* h, const int16_t* iq, uint64_t row_stride_samples, uint32_t nrows, uint64_t n_in_samples,
                   uint32_t fft_len, uint64_t hop_samples, uint32_t avg, const int16_t* window, int64_t* out, void* cuda_stream);

/* Power meter: TPowerMeter<N> of the reference spectrum analyser (sdlmeasure.hpp:9-63) over consecutive blocks of N = block_len samples of
 * each row (rows as in sb200_spectrum): out[r * (n_in / N) + b] for block b = samples [b N, b N + N); a partial last block is not used.  As
 * the reference computes it:
 *     per 4-sample vector i < N / 4:   s = hadd(SquaredNorm(x[4i .. 4i + 3]))     wrapping int32, both steps
 *                                      avg += (uint)((size_t)s / N)              s converted to 64 bits: a wrapped negative s divides as 2^64 + s
 *     per tail sample (N % 4 != 0):    avg += (uint)((size_t)(re^2 + im^2) / N)   the same, one sample at a time
 * with avg a uint (it wraps).  The speanalyzer graph puts TDCRemoveEx<4> (brick/inc/dc.hpp:45-85) before the meter; it subtracts
 * CF_VecDC::direct_current, which no TDCEstimator in that graph ever updates, so it stays at its reset value and the brick changes nothing:
 * this call leaves it out.  Pointers as in sb200_spectrum.  Limits (SB200_E_INVALID, nothing launched): 1 <= block_len <= 65536 and the row
 * limits of sb200_spectrum.  n_in < block_len launches nothing.  One kernel launch; sb200_last_kernel_ms times it. */
int sb200_power_meter(sb200_handle* h, const int16_t* iq, uint64_t row_stride_samples, uint32_t nrows, uint64_t n_in_samples,
                      uint32_t block_len, uint32_t* out, void* cuda_stream);

/* Same as sb200_rx11a_batch for captures at `sample_rate_mhz` = 20, 40 or 44.  20: the capture is already at the channel rate (slots counted in
 * 20 Msps samples; sample j stands where TDownSample2 would have put sample 2j of a 40 Msps capture).  44 Msps slots first pass the reference's 11:10 linear
 * resampler (TDownSample44_40 / Down44to40, Brick11/src/sampling.hpp:37-65, 44MTo40M.hpp:63-123; graph
 * CreateDemodGraph11a_44M, fb11ademod_config.hpp:244-317), each slot starting the interpolator afresh; detect_index then
 * refers to the resampled 20 Msps stream. */
int sb200_rx11a_batch_ex(sb200_handle* h, const int16_t* iq, uint64_t iq_total_samples,
                         const uint64_t* frame_off, const uint32_t* frame_len, uint32_t nframes, uint32_t sample_rate_mhz,
                         uint8_t* out_bytes, uint32_t out_stride, sb200_frame_result* res, void* cuda_stream);

/* 802.11b (DSSS 1/2 Mbps, CCK 5.5/11 Mbps, long preamble).  Same slot convention as sb200_rx11a_batch but 44 Msps samples.
 * out_bytes row i receives frame_length-1 PSDU bytes: like TBB11bFrameSink (PHY_11b.hpp:721-739) the verdict is taken on the
 * first three FCS bytes and the fourth is never delivered; crc32 holds those three bytes (little endian, top byte 0). */
typedef struct sb200_frame_result_11b {
    uint32_t status;        /* SB200_FRAME_* */
    uint32_t rate_kbps;     /* CF_11bRxVector::data_rate_kbps: 1000 / 2000 / 5500 / 11000 */
    uint32_t length;        /* CF_11bRxVector::frame_length (PSDU bytes incl. FCS) */
    uint32_t crc32;         /* first three FCS bytes as received */
    uint32_t sample_index;  /* CF_MemSamples::mem_sample_index at the event (44 Msps samples into the slot) */
    uint32_t detect_vec;    /* index of the first 4-sample vector routed to the demod branch */
} sb200_frame_result_11b;
int sb200_rx11b_batch(sb200_handle* h, const int16_t* iq, uint64_t iq_total_samples,
                      const uint64_t* frame_off, const uint32_t* frame_len, uint32_t nframes,
                      uint8_t* out_bytes, uint32_t out_stride, sb200_frame_result_11b* res, void* cuda_stream);

/* 802.11b continuous captures (SURVEY.md §8(f) rank 1 for the DSSS/CCK chain): capture s = samples [stream_off[s], +stream_len[s]) at 44 Msps;
 * events are reported in the order MAC11b_Receive meets them (kernel/bb/demod11/fb11b_demod.cpp:26-75): after FRAME_OK / CRC32_FAIL the
 * source seeks past the last FCS byte (352 / 176 / 64 / 32 samples), every event ends with Flush, ctx.reset and Reset, and the DC
 * estimate, descrambler register and differential reference carry over.  res and out_bytes hold nstreams x max_frames entries (row
 * s * max_frames + k = event k of capture s; entries past nframes_out[s] are zero); sample_index = CF_MemSamples::mem_sample_index
 * when the event was seen, detect_vec counts vectors since the start of the capture.  All pointers host or device. */
int sb200_rx11b_streams(sb200_handle* h, const int16_t* iq, uint64_t iq_total_samples, const uint64_t* stream_off, const uint32_t* stream_len,
                        uint32_t nstreams, uint32_t max_frames, uint8_t* out_bytes, uint32_t out_stride, sb200_frame_result_11b* res,
                        uint32_t* nframes_out, void* cuda_stream);

/* 802.11n 2x2 receive path (HT mixed format, 20 MHz, two spatial streams; the reference accepts MCS 8, 9 and 10 only,
 * PHY_11n.hpp:496-501).  Replaces the graph of kernel/bb/demod11/fb11ndemod_config.hpp:167-262 (CreateDemodGraph11n) driven like
 * kernel/bb/demod11/fb11n_demod.cpp:29-81: TMemSamples2 -> TDownSample2 -> TCCA11n | TFreqEstimator_11n ... TSisoChannelEst |
 * TFreqComp_11n -> T11nDataSymbol -> 2 x TFFT64 -> {SIG: TSisoChannelComp, TMrcCombine, T11nSigDemap, T11nViterbiSig, T11nSigParser |
 * HT-LTF: TMimoChannelEst | data: TMimoChannelComp, TPilotTrack_11n, T11nDemap*, T11nDeinterleave*_S0/_S1, TStreamJoin/Concat,
 * T11aViterbi<40000,312,192,36>, T11aDesc, TBB11aFrameSink}.  iq0 / iq1 are the two antenna captures (40 Msps, interleaved int16
 * I,Q), both host or both device; slot i covers samples [frame_off[i], frame_off[i]+frame_len[i]) of BOTH captures. */
typedef struct sb200_frame_result_11n {
    uint32_t status;        /* SB200_FRAME_* */
    uint32_t mcs;           /* CF_HTRxVector::ht_frame_mcs.  It has no reset: when the L-SIG is refused before HT-SIG is parsed, a
                             * capture of sb200_rx11n_streams reports its previous event's value (0 for the first), a batch slot 0 */
    uint32_t length;        /* CF_11aRxVector::frame_length: HT LENGTH once HT-SIG parsed, else 2 x L-SIG LENGTH, else 0 */
    uint32_t crc32;         /* received FCS */
    uint32_t nsym;          /* CF_11aRxVector::total_symbols: data symbols + 4 (PHY_11n.hpp:508) */
    uint32_t detect_index;  /* 20 Msps sample index, relative to the slot, of the first sample routed to the L-LTF branch */
    int16_t  cfo_est;       /* CF_CFOffset::CFO_est: 2^16/2pi radians per 20 Msps sample */
    uint16_t lsig_length;   /* 2 x L-SIG LENGTH (PHY_11n.hpp:476) */
} sb200_frame_result_11n;
int sb200_rx11n_batch(sb200_handle* h, const int16_t* iq0, const int16_t* iq1, uint64_t iq_total_samples,
                      const uint64_t* frame_off, const uint32_t* frame_len, uint32_t nframes,
                      uint8_t* out_bytes, uint32_t out_stride, sb200_frame_result_11n* res, void* cuda_stream);
/* 802.11n continuous captures (SURVEY.md §8(f) rank 1 for the HT chain): capture s = the same range [stream_off[s], +stream_len[s]) of
 * both antenna buffers; events in the order RxThread meets them (kernel/bb/demod11/fb11n_demod.cpp:29-81).  After each event the graph is
 * flushed and reset and the source continues with the next 28-sample block, while TCCA11n and MimoAutoCorr keep their history
 * (cca_11n.hpp:146-163, autocorr.hpp:9-42) — carried per capture on the device.  res / out_bytes / sample_index are HOST arrays of
 * nstreams x max_frames entries (row s * max_frames + k); sample_index = CF_MemSamples::mem_sample_index when event k was seen; the
 * sample_index and detect_index fields inside res are relative to the restart. */
int sb200_rx11n_streams(sb200_handle* h, const int16_t* iq0, const int16_t* iq1, uint64_t iq_total_samples, const uint64_t* stream_off,
                        const uint32_t* stream_len, uint32_t nstreams, uint32_t max_frames, uint8_t* out_bytes, uint32_t out_stride,
                        sb200_frame_result_11n* res, uint32_t* sample_index, uint32_t* nframes_out, void* cuda_stream);

/* Stage taps for parity tests (host outputs, any may be NULL): siso [n][2][64][2] legacy channel per antenna, hinv [n][4][64][2]
 * inverse 2x2 channel (11,12,21,22), eq [n][2][max_sym][64][2] per-stream equalised data symbols, theta [n][max_sym] NCO phase
 * after each data symbol, sig [n][16] the nine L-SIG/HT-SIG bytes, soft [n][soft_stride] stream-parsed soft values. */
int sb200_rx11n_taps(sb200_handle* h, const int16_t* iq0, const int16_t* iq1, uint64_t iq_total_samples, const uint64_t* frame_off,
                     const uint32_t* frame_len, uint32_t nframes, uint32_t max_sym, sb200_frame_result_11n* res,
                     int16_t* siso, int16_t* hinv, int16_t* eq, int16_t* theta, uint8_t* sig, uint8_t* soft, uint64_t soft_stride);

/* RX_BLOCK ingest: `blocks` = nblocks x 128 bytes (16-byte descriptor + 28 COMPLEX16, kernel/core/inc/_rx_manager.h:79-113) as stored
 * in *.dmp files and the RX DMA ring; iq_out receives 28*nblocks samples (host or device, 16-byte aligned).  Replaces
 * LoadSoraDumpFile (kernel/brick/inc/brickutil.h:21-59) with a device-side gather; left_shift = 2 applies the legacy 14-bit fix
 * (RX_COMPLEX16_INVALID_BITS, kernel/core/inc/const.h:73; dot11a/dot11/arx_fd.c:530), 0 leaves samples untouched. */
int sb200_rxblocks_unpack(sb200_handle* h, const void* blocks, uint64_t nblocks, uint32_t left_shift, int16_t* iq_out, void* cuda_stream);
/* The descriptor words the unpack drops: per RX_BLOCK the VStreamBits word (which virtual streams the block is valid for) and the radio's
 * TimeStamp (___RX_DESC, kernel/core/inc/_rx_manager.h:97-107); either output may be NULL, host or device. */
int sb200_rxblocks_desc(sb200_handle* h, const void* blocks, uint64_t nblocks, uint32_t* vstream_bits, uint32_t* timestamps, void* cuda_stream);

/* 802.11a transmit: the brick modulator graphs CreateModGraph11a_40M + CreatePreamble11a_40M (kernel/bb/demod11/fb11amod_config.hpp:75-118,
 * 150-158) driven like Test11A_FB_Mod (kernel/bb/demod11/fb11a_mod.cpp:27-107), one warp per OFDM symbol.  Frame i = payload[pay_off[i] ..
 * +pay_len[i]) is the MPDU WITHOUT FCS (the modulator appends CRC-32, as CF_11aTxVector::crc32 does); seeds[i] = CF_ScramblerSeed::sc_seed
 * (NULL: 0xFF as fb11amod_config.hpp:50).  Slot i of `out` (out_stride_samples complex samples) receives lead_samples zeros, the 640-sample
 * preamble, 160 samples per symbol (SIGNAL + the reference's symbol count, TBB11aSrc::GetPadingByte) and zeros to the end of the slot;
 * nsamples[i] = lead + 640 + 160 * symbols.  sample_bits 8: COMPLEX8 as `demod11 -m` writes; 16: COMPLEX16 = COMPLEX8 << 8 as
 * ConvertModFile2DumpFile_8b (demod11/modulate11a.cpp:178-179) feeds the receiver — such a slot goes straight into sb200_rx11a_batch.
 * All pointers host or device. */
int sb200_tx11a_batch(sb200_handle* h, const uint8_t* payload, uint64_t payload_total, const uint64_t* pay_off, const uint32_t* pay_len,
                      const uint8_t* seeds, uint32_t nframes, uint32_t rate_kbps, uint32_t lead_samples, uint32_t sample_bits,
                      void* out, uint64_t out_stride_samples, uint32_t* nsamples, void* cuda_stream);

/* 802.11b transmit: the brick modulator graph CreateModGraph (kernel/bb/demod11/fb11bmod_config.hpp:19-45: TBB11bSrc, TSc741, TBB11bMRSelect,
 * Barker/CCK spreaders, TQuickPulseShaper, TPackSample16to8, TModSink) driven like Test11B_FB_Mod (kernel/bb/demod11/fb11b_mod.cpp:28-32).
 * Long preamble only (PHY_11b.hpp:96-100 rejects the short one).  Frame i = payload[pay_off[i] .. +pay_len[i]) is the MPDU WITHOUT FCS
 * (CF_11bTxVector::crc32 is appended); rate_kbps 1000 / 2000 / 5500 / 11000; init_phase = CF_DifferentialMap::last_phase in front of the
 * first byte (0 on a fresh context).  Slot i of `out` (out_stride_samples complex samples at 44 Msps, a multiple of 8; out 16-byte
 * aligned) receives lead_samples zeros, 4 samples per chip, the shaper's 5 flush vectors, and zeros to the end of the slot;
 * nsamples[i] = lead + what CF_TxSampleBuffer::tx_sample_cnt ends at.  sample_bits 8: COMPLEX8 as `demod11 -m` writes; 16: COMPLEX16 =
 * COMPLEX8 << 8, which goes straight into sb200_rx11b_batch.  final_phase[i] (may be NULL) = last_phase as frame i leaves it, i.e. the
 * init_phase of the next frame modulated on the same context (the reference never resets it).  All pointers host or device. */
int sb200_tx11b_batch(sb200_handle* h, const uint8_t* payload, uint64_t payload_total, const uint64_t* pay_off, const uint32_t* pay_len,
                      uint32_t nframes, uint32_t rate_kbps, uint32_t init_phase, uint32_t lead_samples, uint32_t sample_bits,
                      void* out, uint64_t out_stride_samples, uint32_t* nsamples, uint32_t* final_phase, void* cuda_stream);

/* Page-locked (DMA-able) host memory for capture buffers, as the reference's user-mode extension maps for a radio
 * (SoraURadioMapRxSampleBuf, kernel/core/inc/_user_mode_ext.h:100).  Host captures handed to any entry point from such a buffer cross
 * PCIe without an intermediate staging copy.  NULL on failure (or without a device). */
void* sb200_host_alloc(size_t bytes);
void  sb200_host_free(void* p);

/* Legacy 802.11b transmit filter: BB11BPMDSpreadFIR4SSE (variant 0) and BB11BPMDSpreadFIR4ASM (variant 1) of kernel/inc/bb/bbb.h:188-200
 * (bodies: kernel/bb/dot11b/bbb_fir.c:92-110 + :413-566, and :113-135 + :137-386) — the 37-tap pulse shaper BB11BPMDPacketGenSignal
 * (bbb_tx.c:116-150) runs over the 4x zero-stuffed chip stream of a frame — for a batch of frames.  Frame i = chips[frame_off[i] ..
 * +frame_len[i]) COMPLEX8 samples (int8 re, im), frame_off and frame_len multiples of 8 (the reference returns E_FAIL on uiInputSize & 7
 * and wants 16-byte aligned buffers); out receives frame_len[i] filtered COMPLEX8 samples at the same offsets.  As in the reference the
 * filter starts at the frame's SECOND 16-byte block (output n answers input n + 8; the first eight inputs never enter) and samples past the
 * end of the frame read as zero (the reference's caller zeroes 64 bytes of tail).  variant 0 reproduces the compiled x64 body bit for bit,
 * including what its outer +-1 taps really do (DESIGN.md; the tests check it against the reference's own compiled filter body).
 * All pointers host or device; device buffers 16-byte aligned. */
int sb200_tx11b_fir37(sb200_handle* h, const int8_t* chips, uint64_t chips_total_samples, const uint64_t* frame_off, const uint32_t* frame_len,
                      uint32_t nframes, uint32_t variant, int8_t* out, void* cuda_stream);

/* Legacy 802.11b transmitter, long or short preamble: BB11BPMDBufferTx4XWithLongHeader / ...WithShortHeader (kernel/bb/dot11b/bbb_tx.c:508-758,
 * declared in kernel/inc/bb/bbb.h:204-240) — PLCP frame with CRC-16, the table scrambler (seed 0x6C long, 0x1B short) over PLCP + PSDU + FCS,
 * Barker DBPSK preamble (long: and header), DQPSK header (short), DBPSK / DQPSK / CCK 5.5 / CCK 11 data, each chip followed by three zero
 * samples, then TX_FIR_DEPTH zeros rounded up to a multiple of 128 samples — optionally run through the 37-tap filter as
 * BB11BPMDPacketGenSignal (bbb_tx.c:119-150) does.  Frame i = payload[pay_off[i] .. +pay_len[i]) is the MPDU WITHOUT FCS; CRC-32 is
 * appended, or, with flags SB200_TX11B_LEGACY_FCS_IN_PAYLOAD, the payload's last 4 bytes are sent verbatim as the FCS (PSDU 4 .. 4095 bytes).
 * SB200_TX11B_LEGACY_PBCC is refused (SB200_E_INVALID): ModSelect PBCC only changes the LENGTH field in the reference (bbb_tx.c:51-57), the
 * data would still be CCK.  Short preamble at 1 Mbps writes preamble and header only, as the reference does (its short-preamble switch has
 * no 1 Mbps case, bbb_tx.c:563-605).  filter 0 = the encoder output (what BB11BPMDBufferTx4X* writes), 1 = BB11BPMDSpreadFIR4SSE over it,
 * 2 = BB11BPMDSpreadFIR4ASM (see sb200_tx11b_fir37); the filtered stream is computed from the chips directly, never stored zero-stuffed.
 * Slot i of `out` (out_stride_samples COMPLEX8 samples at 44 Msps, a multiple of 8; out 16-byte aligned) receives nsamples[i] samples and
 * zeros to the end of the slot.  All pointers host or device.  The caller's payload is not modified (the reference scrambles its buffer in
 * place; the legacy entry points of sora_b200_legacy.h reproduce that). */
#define SB200_TX11B_LEGACY_FCS_IN_PAYLOAD 1u
#define SB200_TX11B_LEGACY_PBCC           2u
int sb200_tx11b_legacy_batch(sb200_handle* h, const uint8_t* payload, uint64_t payload_total, const uint64_t* pay_off, const uint32_t* pay_len,
                             uint32_t nframes, uint32_t rate_kbps, uint32_t short_preamble, uint32_t flags, uint32_t filter, int8_t* out,
                             uint64_t out_stride_samples, uint32_t* nsamples, void* cuda_stream);

/* Legacy 802.11a transmitter: BB11ATxFrameMod / BB11ATxBufferMod6M (kernel/bb/dot11a/dot11/atx_fe.c, atx_tpl_imp.h:5-58, declared in
 * kernel/inc/bb/bba.h:239-247) at SampleRate 40 or 44 — the caller's 640-sample preamble, SIGNAL, the data symbols (scrambler from 0xFF,
 * the lutst/mapa_* constellation, pilots +-10720, IFFT64x with a wrapping << 2, a window that carries three samples into the next symbol),
 * each 160-sample chunk upsampled afresh to 176 at 44 Msps (Upsample40MTo44M_160, with its one-sample over-read), Copy_NT (>> 6, int8
 * saturation), the 8-sample tail, then zeros to a multiple of 128 bytes (ALIGN_WITH_RCB_BUFFER_PADDING_ZERO).  Frame i =
 * payload[pay_off[i] .. +pay_len[i]) is the MPDU WITHOUT FCS; CRC-32 is appended, or, with flags SB200_TX11A_LEGACY_FCS_IN_PAYLOAD, the
 * payload's last 4 bytes are sent verbatim as the FCS (BB11ATxFrameMod sends PACKET_BASE::Reserved1).  MPDU + FCS may be 4096 bytes, as
 * atx_fe.c:23 admits; GetSignal then shifts LENGTH 4096 into the parity bit, and so does this.  preamble: the 640 COMPLEX16 samples of the
 * reference's PREAMBLE40_11A_LUT (not part of this library; host or device; exactly 640 are read).  Slot i of `out` (out_stride_samples
 * COMPLEX8 samples, a multiple of 8; out 16-byte aligned) receives nsamples[i] samples — the RCB-padded signal length, what
 * SoraPacketSetSignalLength stores, divided by 2 — and zeros to the end of the slot.  SB200_E_INVALID for a rate that is not an 802.11a
 * rate, a sample rate other than 40 / 44, MPDU + FCS over 4096 bytes, or a slot too small.  All pointers host or device. */
#define SB200_TX11A_LEGACY_FCS_IN_PAYLOAD 1u
int sb200_tx11a_legacy_batch(sb200_handle* h, const uint8_t* payload, uint64_t payload_total, const uint64_t* pay_off, const uint32_t* pay_len,
                             uint32_t nframes, uint32_t rate_kbps, uint32_t sample_rate_mhz, uint32_t flags, const int16_t* preamble, int8_t* out,
                             uint64_t out_stride_samples, uint32_t* nsamples, void* cuda_stream);

/* 802.11n transmit, two spatial streams, HT-mixed format: the modulator graphs CreatePreambleGraph11n + CreateSigGraph11n + CreateModGraph11n
 * (kernel/bb/demod11/fb11nmod_config.hpp:74-171) driven like Test11N_FB_Mod (kernel/bb/demod11/fb11n_mod.cpp:44-70).  Frame i =
 * payload[pay_off[i] .. +pay_len[i]) is the MPDU WITHOUT FCS (CF_11nTxVector::crc32 is appended); mcs 8 .. 14 (the modulator graph's own
 * range, fb11nmod_config.hpp:146-155; the reference's receiver admits 8 .. 10 only, PHY_11n.hpp:496-501 — see option "ht_mcs_limit"); seeds[i] = CF_ScramblerSeed::sc_seed (NULL: 0xAB as fb11nmod_config.hpp:52).  Slot i of out0 / out1
 * (out_stride_samples COMPLEX16 samples at 40 Msps each, the two transmit chains) receives lead_samples zeros, L-STF + L-LTF (640), L-SIG
 * + HT-SIG (480), HT-STF + 2 HT-LTF (480), 160 samples per DATA symbol — one more symbol than HT-SIG announces when the graph's Flush
 * padding spills over a symbol boundary — and zeros to the end of the slot; nsamples[i] = lead + samples written.  The two slots go
 * straight into sb200_rx11n_batch as the two antenna captures.  All pointers host or device (out0 and out1 on the same side). */
int sb200_tx11n_batch(sb200_handle* h, const uint8_t* payload, uint64_t payload_total, const uint64_t* pay_off, const uint32_t* pay_len,
                      const uint8_t* seeds, uint32_t nframes, uint32_t mcs, uint32_t lead_samples, int16_t* out0, int16_t* out1,
                      uint64_t out_stride_samples, uint32_t* nsamples, void* cuda_stream);

/* Standalone K=7 Viterbi over `nblocks` independent blocks of `nsoft` soft values (uint8 0..7, one per coded bit after
 * puncturing; block b starts at soft + b*soft_stride).  frame_len_bytes L sets the flush point 8L+16+6 exactly like
 * CF_11aRxVector::frame_length; each block yields L+2 bytes (SERVICE + PSDU, not descrambled) at out + b*out_stride.
 * depth/lookahead = TRELLIS_DEPTH/TRELLIS_LOOKAHEAD (256/24 for 11a, 192/36 for 11n).  A trailing partial puncture group (nsoft not a
 * multiple of 2 / 3 / 4 soft values at rate 1/2 / 2/3 / 3/4) is ignored, as the reference brick keeps it buffered.  A block whose soft values
 * end before its flush point is defined only up to its last traceback window: the bytes of the windows that fired, the rest of its row
 * unspecified. */
int sb200_viterbi_k7(sb200_handle* h, const uint8_t* soft, uint64_t soft_stride, uint32_t nsoft, uint32_t nblocks,
                     int code_rate, uint32_t frame_len_bytes, uint32_t depth, uint32_t lookahead,
                     uint8_t* out, uint64_t out_stride, void* cuda_stream);

/* Stage taps for parity tests: decodes the slots like sb200_rx11a_batch and additionally returns, per slot,
 * FreqCoeffs / ChannelCoeffs (64 COMPLEX16 each) and per symbol (0 = SIGNAL) the FFT output, the equalised and the
 * pilot-tracked symbol (64 COMPLEX16 each, FFT bin order) and the de-interleaved soft bits of the data symbols.
 * All tap buffers are host memory; any may be NULL.  soft rows are soft_stride bytes, data symbols back to back. */
int sb200_rx11a_taps(sb200_handle* h, const int16_t* iq, uint64_t iq_total_samples,
                     const uint64_t* frame_off, const uint32_t* frame_len, uint32_t nframes, uint32_t max_sym,
                     sb200_frame_result* res, int16_t* freq_coeffs, int16_t* chan_coeffs,
                     int16_t* fft_out, int16_t* equalized, int16_t* tracked, uint8_t* soft, uint64_t soft_stride);

#ifdef __cplusplus
}
#endif
#endif
