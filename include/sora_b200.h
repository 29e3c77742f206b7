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
