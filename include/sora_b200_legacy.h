/* sora_b200_legacy.h — the reference's legacy C baseband interfaces for 802.11a and 802.11b receive, served by the GPU engine.
 *
 * SURVEY.md §8(f) rank 4.  Same entry-point names, argument order, HRESULT values and result fields as
 *   kernel/inc/bb/bba.h:15-24 (BB11A_* codes), :61-70 (ri_* result fields), :191-262 (BB11ARx* prototypes) and
 *   kernel/core/inc/_rx_stream.h:22-50 (SORA_RADIO_RX_STREAM, SoraGenRadioRxStreamOffline),
 * so that a caller written against them (kernel/bb/demod11/demod11a.cpp:53-200 CsFrameDemod, UMXDot11/dot11arx.c) links against
 * libsora_b200.so after swapping the include.  The context is this library's own struct: only the documented public fields keep
 * their names; the reference's private working state (`__` fields, FIFOs, Viterbi thread state) has no counterpart because the
 * decode runs on the device.  The demodulator behind it is the brick receive chain of include/sora_b200.h (the reference's newer
 * implementation of the same PHY), not a restatement of dot11a/dot11/arx_*.c: verdicts and payloads agree wherever both decode.
 * BB11ARxViterbiWorker is a no-op that returns FALSE (there is no separate Viterbi thread to pump).
 */
#ifndef SORA_B200_LEGACY_H
#define SORA_B200_LEGACY_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef int32_t HRESULT;
typedef uint32_t ULONG;
typedef unsigned char BOOLEAN, UCHAR, *PUCHAR;
typedef volatile uint32_t FLAG, *PFLAG;
#ifndef FAILED
#define FAILED(hr) (((HRESULT)(hr)) < 0)
#define SUCCEEDED(hr) (((HRESULT)(hr)) >= 0)
#endif

#define BB11A_CHANNEL_CLEAN      ((HRESULT)0x00000200L)
#define BB11A_OK_POWER_DETECTED  ((HRESULT)0x00000201L)
#define BB11A_OK_FRAME           ((HRESULT)0x00000202L)
#define BB11A_E_PD_LAG           ((HRESULT)0x80006000L)
#define BB11A_E_SYNC_FAIL        ((HRESULT)0x80006001L)
#define BB11A_E_INVALID_SIG      ((HRESULT)0x80006002L)
#define BB11A_E_FRAME_SIZE       ((HRESULT)0x80006003L)
#define BB11A_E_CRC32            ((HRESULT)0x80006004L)
#define BB11A_E_FORCE_STOP       ((HRESULT)0x80006005L)

#define SORA_RX_BLOCK_SIZE 128u                 /* 16-byte descriptor + 7 x 16 bytes of samples (_rx_manager.h:79-113) */

typedef struct __SORA_RADIO_RX_STREAM {         /* _rx_stream.h:22-30 */
    PUCHAR __pStartPt; ULONG __nRxBufSize; PUCHAR __pEndPt; PUCHAR __pScanPt; ULONG __VStreamMask;
} SORA_RADIO_RX_STREAM, *PSORA_RADIO_RX_STREAM;
void SoraGenRadioRxStreamOffline(PSORA_RADIO_RX_STREAM pRxStream, PUCHAR pInput, ULONG Size);

typedef struct _BB11A_RX_CONTEXT {
    /* carrier sense configuration (bba.h:43-47) */
    unsigned int SampleRate; ULONG uiCSCorrThreshold; unsigned int uiCSMaxFetchRxBlock, uiCSMinFetchRxBlock;
    /* results (bba.h:61-70) */
    volatile FLAG* ri_pbWorkIndicator;
    char* ri_pbFrame; unsigned int ri_uiFrameMaxSize;
    unsigned int ri_uiFrameSize;                /* LENGTH of the PSDU incl. FCS (arx_fd.c:265) */
    unsigned int ri_uiDataRate;                 /* kbps */
    unsigned int ri_uiFrameType;
    /* engine state */
    void* b200_engine; void* b200_events; unsigned int b200_shift;
} BB11A_RX_CONTEXT, *PBB11A_RX_CONTEXT;

void    BB11ARxContextInit(PBB11A_RX_CONTEXT pRxContextA, unsigned int SampleRate, ULONG rxThreshold, ULONG rxMaxBlockCount, ULONG rxMinBlockCount, volatile FLAG* WorkIndicator);
void    BB11APrepareRx(PBB11A_RX_CONTEXT pRxContextA, char* pcFrame, unsigned int unFrameMaxSize);
BOOLEAN BB11ARxViterbiWorker(void* pContext);
void    BB11ARxReset(PBB11A_RX_CONTEXT pRxContextA);
void    BB11ARxContextCleanup(PBB11A_RX_CONTEXT pRxContextA);
HRESULT BB11ARxCarrierSense(PBB11A_RX_CONTEXT pRxContextA, PSORA_RADIO_RX_STREAM pRxStream);
HRESULT BB11ARxFrameDemod(PBB11A_RX_CONTEXT pRxContextA, PSORA_RADIO_RX_STREAM pRxStream);
/* not in the reference: selects the legacy 14-bit sample fix (left shift by 2) for old captures such as kernel/test-data/fsample-6.dmp */
void    BB11ARxSetSampleShift(PBB11A_RX_CONTEXT pRxContextA, unsigned int left_shift);

/* ---- 802.11b: kernel/inc/bb/bbb.h:8-36 (BB11B_* codes), :134-197 (contexts), :199-262 (prototypes); driver loop kernel/bb/demod11/demod11b.cpp:73-174.
 * Only the fields a caller reads or writes keep their names: thresholds, block counts, reset flags, DC offset, work indicator, and the
 * BB11bCommon results (b_length = PSDU length incl. FCS, b_dataRate = PLCP SIGNAL code, counters).  Power detection and demodulation are
 * the brick receive graph of fb11bdemod_config.hpp on the device (energy detector instead of the legacy LH/HL gain logic): BB11BSpd stops
 * at the block in which that graph's carrier sense fires, BB11BRx returns the frame that follows. */
#define BB11B_E_ENERGY           ((HRESULT)0x80050100L)
#define BB11B_E_DOWNSAMPLE       ((HRESULT)0x80050101L)
#define BB11B_E_BARKER           ((HRESULT)0x80050102L)
#define BB11B_E_SFD              ((HRESULT)0x80050103L)
#define BB11B_E_DATA             ((HRESULT)0x80050105L)
#define BB11B_E_PD_LAG           ((HRESULT)0x80050106L)
#define BB11B_E_FORCE_STOP       ((HRESULT)0x80050107L)
#define BB11B_E_PLCP_HEADER_CRC  ((HRESULT)0x80050210L)
#define BB11B_E_PLCP_HEADER_SIG  ((HRESULT)0x80050211L)
#define BB11B_OK_FRAME           ((HRESULT)0x0000007FL)
#define BB11B_OK_POWER_DETECTED  ((HRESULT)0x00000101L)
#define BB11B_CHANNEL_CLEAN      ((HRESULT)0x00000102L)

typedef struct _SORA_COMPLEX16 { int16_t re, im; } SORA_COMPLEX16;
typedef struct _BB11B_COMMON {                  /* bbb.h:84-127, result part */
    unsigned int b_length;                      /* PSDU length incl. CRC-32 */
    unsigned char b_dataRate;                   /* PLCP SIGNAL: 0x0A, 0x14, 0x37, 0x6E */
    char b_isLongPreamble;
    unsigned long b_crc32;
    unsigned int b_errEnergyLoss, b_errFrame, b_errPLCPHeader, b_goodFrameCounter;
    PUCHAR b_outputPt; ULONG b_maxOutputSize;
} BB11B_COMMON, *PBB11B_COMMON;
typedef struct __BB11B_RX_CONTEXT {             /* bbb.h:134-158 */
    unsigned int b_maxDescCount; int b_resetFlag; short b_energyLeast; volatile FLAG* b_workIndicator; int b_shiftRight;
    SORA_COMPLEX16 b_dcOffset;
    BB11B_COMMON BB11bCommon;
    void* b200_engine; void* b200_events;
} BB11B_RX_CONTEXT, *PBB11B_RX_CONTEXT;
typedef struct _BB11B_SPD_CONTEXT {             /* bbb.h:161-186 */
    unsigned int b_minDescCount, b_maxDescCount, b_threshold, b_thresholdLH, b_thresholdHL, b_gainLevel, b_gainLevelNext;
    int b_resetFlag; volatile FLAG* b_workIndicator; SORA_COMPLEX16 b_dcOffset; char b_reestimateOffset; ULONG b_evalEnergy;
    void* b200_rx;                              /* the receive context initialised together with this one */
} BB11B_SPD_CONTEXT, *PBB11B_SPD_CONTEXT;

void    BB11BRxSpdContextInit(PBB11B_RX_CONTEXT pRxContext, PBB11B_SPD_CONTEXT pSpdContext, PFLAG pfCanWork, ULONG nRxMaxBlockCount, ULONG nSPDMaxBlockCount,
                              ULONG nSPDMinBlockCount, ULONG nSPDThreashold, ULONG nSPDThreasholdLow, ULONG nSPDThreasholdHigh, ULONG nShiftRight);
void    BB11BRxSpdContextCleanUp(PBB11B_RX_CONTEXT pRxContext);
void    BB11BPrepareRx(PBB11B_RX_CONTEXT pRxContext, void* pOutputBuf, ULONG OutputBufSize);
HRESULT BB11BSpd(PBB11B_SPD_CONTEXT pSpdContext, PSORA_RADIO_RX_STREAM pRxStream);
HRESULT BB11BRx(PBB11B_RX_CONTEXT pRxContext, PSORA_RADIO_RX_STREAM pRxStream);

/* ---- 802.11b transmit filter: kernel/inc/bb/bbb.h:188-200.  The 37-tap pulse shaper over the 4x zero-stuffed chip stream (COMPLEX8), the
 * last stage of BB11BPMDPacketGenSignal (kernel/bb/dot11b/bbb_tx.c:116-150).  uiInputSize in samples, a multiple of 8 (else E_FAIL, as in
 * the reference); *puiOutputSize = uiInputSize.  Runs on a process-wide engine created on first use (device SB200_DEVICE, default 0); E_FAIL
 * without a GPU.  The SSE entry reproduces the reference's compiled intrinsic body bit for bit, the ASM entry its 32-bit assembly body
 * (they differ in the outermost +-1 taps, see sb200_tx11b_fir37 in sora_b200.h). */
#define SORA_S_OK    ((HRESULT)0)
#define SORA_E_FAIL  ((HRESULT)0x80004005L)
typedef struct _SORA_COMPLEX8 { int8_t re, im; } SORA_COMPLEX8, *PCOMPLEX8;
HRESULT BB11BPMDSpreadFIR4SSE(const SORA_COMPLEX8* pcSrc, uint32_t uiInputSize, SORA_COMPLEX8* pcDest, ULONG* puiOutputSize);
HRESULT BB11BPMDSpreadFIR4ASM(const SORA_COMPLEX8* pcSrc, uint32_t uiInputSize, SORA_COMPLEX8* pcDest, ULONG* puiOutputSize);

/* ---- 802.11b transmitter: kernel/inc/bb/bbb.h:204-240, kernel/bb/dot11b/bbb_tx.c (encoder) + the filter above, long and short preamble.
 * Served by sb200_tx11b_legacy_batch on the same process-wide engine.  Side effects callers see are reproduced: the encoder scrambles the
 * caller's PSDU + FCS in place (Buffer variants: pbData[0 .. dataLength + 4); Packet variants: every MDL of the chain and Reserved1), and
 * BB11BPMDPacketGenSignal stores the signal length in bytes into the packet's TX descriptor.  E_FAIL (SORA_E_FAIL) as in the reference
 * (PreambleType other than 0 / 1; GenSignal buffers shorter than BB11B_MAX_SYMBOL_LENGTH) and also without a GPU, for a rate code other
 * than 0x0A / 0x14 / 0x37 / 0x6E, for ModSelect PBCC (sb200_tx11b_legacy_batch), for a PSDU over 4095 bytes, and when an MDL chain does not
 * add up to PacketSize.  PACKET_BASE, TX_DESC and MDL carry only the fields bbb_tx.c and the SoraPacket* helpers use. */
#define DOT11B_PLCP_DATA_RATE_1M        0x0A
#define DOT11B_PLCP_DATA_RATE_2M        0x14
#define DOT11B_PLCP_DATA_RATE_5P5M      0x37
#define DOT11B_PLCP_DATA_RATE_11M       0x6E
#define DOT11B_PLCP_IS_LONG_PREAMBLE    0
#define DOT11B_PLCP_IS_SHORT_PREAMBLE   1
#define DOT11B_PLCP_IS_CCK              0
#define DOT11B_PLCP_IS_PBCC             1
typedef struct _DOT11B_PLCP_TXVECTOR {          /* kernel/inc/dot11_plcp.h:55-59 */
    UCHAR DateRate;                             /* PLCP SIGNAL code */
    UCHAR PreambleType;                         /* 0 = long, 1 = short */
    UCHAR ModSelect;                            /* 0 = CCK, 1 = PBCC (refused) */
} DOT11B_PLCP_TXVECTOR, *PDOT11B_PLCP_TXVECTOR;
typedef SORA_COMPLEX8 TXSAMPLE, *PTXSAMPLE;
typedef struct _MDL {                           /* the fields of the WDK MDL the encoder walks */
    struct _MDL* Next; void* StartVa; ULONG ByteOffset; ULONG ByteCount;
} MDL, *PMDL;
typedef struct _TX_DESC {                       /* where the modulated samples go */
    PTXSAMPLE pSampleBuffer; ULONG SampleBufferSize; ULONG SignalLength;   /* sizes in bytes */
} TX_DESC, *PTX_DESC;
typedef struct __PACKET_BASE {                  /* kernel/core/inc/_packet_base.h:44-56 */
    PMDL pMdl; PTX_DESC pTxDesc; int32_t fStatus; ULONG PacketSize;
    ULONG Reserved1;                            /* the FCS (CRC-32) the Packet variants send */
    ULONG Reserved2, Reserved3, Reserved4; void* pReserved;
} PACKET_BASE, *PPACKET_BASE;
/* (MTU 1500 + long PLCP frame 24 + CRC-32 4) x 8 bits x 4 x 11 x sizeof(COMPLEX8), kernel/inc/bb/bbb.h:75-80 */
#define BB11B_MAX_SYMBOL_LENGTH ((1500u + 24u + 4u) * 8u * 4u * 11u * 2u)

void    BB11BTxVectorInit(PDOT11B_PLCP_TXVECTOR pTxVector, UCHAR cDataRate, UCHAR cModSelect, UCHAR cPreambleType);
/* pbData = MPDU + FCS (dataLength + 4 bytes); pOutput receives *pOutputLength COMPLEX8 samples: the 4x zero-stuffed chips and zero padding */
HRESULT BB11BPMDBufferTx4XWithShortHeader(PDOT11B_PLCP_TXVECTOR pTxVector, PUCHAR pbData, unsigned int dataLength, PUCHAR pOutput, unsigned int* pOutputLength);
HRESULT BB11BPMDBufferTx4XWithLongHeader(PDOT11B_PLCP_TXVECTOR pTxVector, PUCHAR pbData, unsigned int dataLength, PUCHAR pOutput, unsigned int* pOutputLength);
HRESULT BB11BPMDPacketTx4X(PDOT11B_PLCP_TXVECTOR pTxVector, PPACKET_BASE pSendSlot, PUCHAR pOutput, ULONG BufferLength, ULONG* puiOutputLength);
/* encoder into pTempBuffer, then BB11BPMDSpreadFIR4SSE into the packet's sample buffer (bbb_tx.c:119-150) */
HRESULT BB11BPMDPacketGenSignal(PPACKET_BASE pPacket, PDOT11B_PLCP_TXVECTOR pTxVector, PUCHAR pTempBuffer, ULONG TempBufferLength);
void    SoraPacketGetTxSampleBuffer(PPACKET_BASE pPacket, PTXSAMPLE* ppBuffer, ULONG* pBufferSize);
void    SoraPacketSetSignalLength(PPACKET_BASE pPacket, ULONG uLen);

/* ---- 802.11a transmitter: kernel/inc/bb/bba.h:146-186 (BB11A_TX_VECTOR, DOT11A_RATE_*), :201-206, :239-247; kernel/bb/dot11a/dot11/atx_fe.c.
 * Served by sb200_tx11a_legacy_batch on the same process-wide engine, at SampleRate 40 or 44.  Only the public fields of BB11A_TX_VECTOR keep
 * their names; the reference's working buffers have no counterpart.  The 640-sample preamble table PREAMBLE40_11A_LUT is not part of this
 * library: a caller hands it in once per process with BB11ATxSetPreamble (in the Sora tree: BB11ATxSetPreamble(PREAMBLE40_11A())).
 * BB11ATxFrameMod sends the MDL chain and Reserved1 as the FCS, writes the signal and its zero padding to a multiple of 128 bytes into the
 * packet's sample buffer and stores that length in bytes (SoraPacketSetSignalLength).  BB11AModulateACK writes the 14-byte ACK to RA at
 * 6 Mbps into PhyACKBuffer (sized by the caller, as in the reference) and returns the padded length in bytes.  E_FAIL (SORA_E_FAIL) as in
 * the reference (a rate code not in DOT11A_RATE_*, PacketSize + 4 > 4096), and, without writing anything, where the reference would assert
 * or overrun (SampleRate other than 40 / 44, a sample buffer too small), when the MDL chain does not add up to PacketSize, without a GPU, and
 * until BB11ATxSetPreamble was called; BB11AModulateACK returns 0 in those cases. */
#define DOT11A_RATE_6M  0xB
#define DOT11A_RATE_9M  0xF
#define DOT11A_RATE_12M 0xA
#define DOT11A_RATE_18M 0xE
#define DOT11A_RATE_24M 0x9
#define DOT11A_RATE_36M 0xD
#define DOT11A_RATE_48M 0x8
#define DOT11A_RATE_54M 0xC
typedef struct _MAC_ADDRESS { UCHAR Address[6]; } MAC_ADDRESS, *PMAC_ADDRESS;   /* kernel/inc/dot11_pkt.h:35-39 */
typedef struct _BB11A_TX_VECTOR {
    unsigned int SampleRate;                    /* 40 or 44 (Msps) */
    unsigned int ti_uiDataRate;                 /* DOT11A_RATE_* */
    unsigned int ti_uiBufferLength;
} BB11A_TX_VECTOR, *PBB11A_TX_VECTOR;

void    BB11ATxContextInit(PBB11A_TX_VECTOR info, unsigned int SampleRate);
HRESULT BB11ATxFrameMod(PBB11A_TX_VECTOR info, PPACKET_BASE pPacket);
ULONG   BB11AModulateACK(unsigned int SampleRate, const PMAC_ADDRESS RecvMacAddress, void* PhyACKBuffer);
/* not in the reference: the 640 COMPLEX16 samples of PREAMBLE40_11A_LUT, copied; process-wide; NULL forgets them */
void    BB11ATxSetPreamble(const void* preamble640);

#ifdef __cplusplus
}
#endif
#endif
