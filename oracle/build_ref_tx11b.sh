#!/bin/sh
# oracle/_ref/libtx11b_legacy_ref.so: the reference's legacy 802.11b encoder, compiled from its own source — the six plain-C files behind
# BB11BPMDBufferTx4XWith{Long,Short}Header (kernel/bb/dot11b/bbb_tx.c, bbb_scramble.c, bbb_dbpsk.c, bbb_dqpsk.c, bbb_cck5.c, bbb_cck11.c:
# PLCP frame, table scrambler, Barker DBPSK / DQPSK and CCK 5.5 / 11 look-up tables, 4x zero stuffing).  The Windows headers they include
# are replaced by a shim written here (integer typedefs, MDL / PACKET_BASE with the fields the code reads, COMPLEX8); the PLCP constants and
# structs (kernel/inc/dot11_plcp.h), the rate codes (kernel/inc/bb/bbb.h:47-50) and CalcCRC16 with its table (kernel/core/inc/CRC16.h) are
# cut out of the reference with sed at build time.  Two fixes, both in build-time copies under oracle/_ref/: bbb_tx.h:187 declares
# PLCPGetLength with two parameters where bbb_tx.c:39 defines three (the line is dropped), and SORA_EXTERN_C is plain `extern` so that
# SSEFilterTaps (bbb_tx.h:189) stays a declaration.  The sources are read where they lie, on stdin, so that their quoted includes resolve
# to the shim directory.  Nothing of the reference is copied into the repository.  TEST INFRASTRUCTURE ONLY.
#   usage: oracle/build_ref_tx11b.sh [reference root, default /root/reference]
set -e
REF="${1:-/root/reference}"
SRC="$REF/kernel/bb/dot11b"
HERE="$(cd "$(dirname "$0")" && pwd)"
[ -f "$SRC/bbb_tx.c" ] || { echo "build_ref_tx11b: $SRC/bbb_tx.c not found (fine outside the build container: the prebuilt oracle/_ref is used)"; exit 0; }
INC="$HERE/_ref/tx11b_inc"
rm -rf "$INC"; mkdir -p "$INC/bb"
{
  cat <<'HDR'
#pragma once
#include <stdint.h>
#include <string.h>
typedef int32_t HRESULT; typedef unsigned char UCHAR, *PUCHAR, BOOLEAN; typedef unsigned short USHORT, *PUSHORT; typedef unsigned int UINT, *PUINT;
typedef uint32_t ULONG, *PULONG; typedef short SHORT; typedef void* PVOID;
#define IN
#define OUT
#define S_OK 0
#define E_FAIL ((HRESULT)0x80004005L)
#define FALSE 0
#define SORA_EXTERN_C extern
#define SELECTANY
#define FINL static inline
#define A16 __attribute__((aligned(16)))
#define UNREFERENCED_PARAMETER(x) (void)(x)
typedef struct { signed char re, im; } COMPLEX8, *PCOMPLEX8, TXSAMPLE, *PTXSAMPLE;
typedef struct _MDL { struct _MDL* Next; void* StartVa; UINT ByteOffset; UINT ByteCount; } MDL, *PMDL;
typedef struct { PMDL pMdl; UINT PacketSize; ULONG Reserved1; } PACKET_BASE, *PPACKET_BASE;
void SoraPacketGetTxSampleBuffer(PPACKET_BASE, PTXSAMPLE*, ULONG*); void SoraPacketSetSignalLength(PPACKET_BASE, ULONG);
HRESULT BB11BPMDSpreadFIR4SSE(PCOMPLEX8, ULONG, PCOMPLEX8, ULONG*);
HDR
  tr -d '\r' < "$REF/kernel/inc/dot11_plcp.h" | sed -n '/^#define DOT11B_PLCP_LONG_PREAMBLE_SYNC_VALUE/,/^#pragma pack(pop)/p'
  tr -d '\r' < "$REF/kernel/inc/bb/bbb.h" | sed -n '/^#define DOT11B_PLCP_DATA_RATE_/p'
  tr -d '\r' < "$REF/kernel/inc/bb/bbb.h" | sed -n '/^#define BB11B_MAX_TRANSMIT_UNIT/p;/^#define BB11B_MAX_SYMBOL_LENGTH/,/sizeof(COMPLEX8))/p'
} > "$INC/bb/bbb.h"
{
  echo '#pragma once'
  echo '#include "bb/bbb.h"'
  tr -d '\r' < "$REF/kernel/core/inc/CRC16.h" | sed -n '/LUT_CRC16\[256\] =/,/^FINL void CalcCRC16Incremental/p' | sed '$d' \
    | sed 's/^SORA_EXTERN_C SELECTANY extern const/static const/; /^SORA_EXTERN_C$/d'
} > "$INC/CRC16.h"
: > "$INC/complex.h"
tr -d '\r' < "$SRC/bbb_tx.h" | sed '/^USHORT PLCPGetLength(IN PDOT11B_PLCP_TXVECTOR pTxVector, IN OUT PUINT ext);/d' > "$INC/bbb_tx.h"
tr -d '\r' < "$SRC/bbb_lut.h" > "$INC/bbb_lut.h"
cat > "$INC/entry.c" <<'ENTRY'
/* plain-C entry points around the compiled encoder */
#include "bb/bbb.h"
#include "bbb_tx.h"
#include <stdlib.h>
HRESULT BB11BPMDBufferTx4XWithShortHeader(PDOT11B_PLCP_TXVECTOR, PUCHAR, UINT, PUCHAR, PUINT);
HRESULT BB11BPMDBufferTx4XWithLongHeader(PDOT11B_PLCP_TXVECTOR, PUCHAR, UINT, PUCHAR, PUINT);
void FIRInit(void) {}
/* BB11BPMDPacketGenSignal is linked but not driven from here: the filter body is oracle/_ref/libfir37_ref.so (build_ref.sh) */
void SoraPacketGetTxSampleBuffer(PPACKET_BASE p, PTXSAMPLE* b, ULONG* n) { (void)p; *b = 0; *n = 0; }
void SoraPacketSetSignalLength(PPACKET_BASE p, ULONG n) { (void)p; (void)n; }
HRESULT BB11BPMDSpreadFIR4SSE(PCOMPLEX8 s, ULONG n, PCOMPLEX8 d, ULONG* o) { (void)s; (void)d; *o = n; return E_FAIL; }
/* what BB11BPMDBufferTx4XWith{Short,Long}Header (bbb_tx.c:508-758) writes for psdu_with_fcs[0 .. len) (len >= 4: MPDU + FCS); the
   caller's bytes are left as they were (the reference scrambles its buffer in place; scrambled[] receives that, when not NULL) */
int ref_tx11b_legacy(const unsigned char* psdu_with_fcs, unsigned len, unsigned rate_code, unsigned short_preamble, signed char* out_c8,
                     unsigned* n, unsigned char* scrambled) {
    DOT11B_PLCP_TXVECTOR v; memset(&v, 0, sizeof v);
    v.DateRate = (UCHAR)rate_code; v.PreambleType = (UCHAR)(short_preamble ? DOT11B_PLCP_IS_SHORT_PREAMBLE : DOT11B_PLCP_IS_LONG_PREAMBLE); v.ModSelect = DOT11B_PLCP_IS_CCK;
    unsigned char* b = (unsigned char*)malloc(len + 1); memcpy(b, psdu_with_fcs, len);
    UINT m = 0; HRESULT r = short_preamble ? BB11BPMDBufferTx4XWithShortHeader(&v, b, len - 4, (PUCHAR)out_c8, &m)
                                           : BB11BPMDBufferTx4XWithLongHeader(&v, b, len - 4, (PUCHAR)out_c8, &m);
    if (scrambled) memcpy(scrambled, b, len);
    free(b); *n = m; return (int)r;
}
/* the look-up tables the encoder runs on, as raw bytes (tests compare the regenerated tables with them entry for entry) */
const void* ref_tx11b_table(int which, unsigned* bytes) {
    extern const unsigned char gc_ScramblerLUT[256][128];
    switch (which) {
        case 0: *bytes = sizeof(gc_ScramblerLUT); return gc_ScramblerLUT;
        case 1: *bytes = sizeof(gc_DBPSKUCHARSpreadedComplexLUT); return gc_DBPSKUCHARSpreadedComplexLUT;
        case 2: *bytes = sizeof(gc_DQPSKUCHARSpreadedComplexLUT); return gc_DQPSKUCHARSpreadedComplexLUT;
        case 3: *bytes = sizeof(gc_CCK5UCHARSpreadedComplexLUT); return gc_CCK5UCHARSpreadedComplexLUT;
        case 4: *bytes = sizeof(gc_CCK11UCHARSpreadedComplexLUT); return gc_CCK11UCHARSpreadedComplexLUT;
        case 5: *bytes = sizeof(LUT_CRC16); return LUT_CRC16;
        default: *bytes = 0; return 0;
    }
}
ENTRY
printf '#include "CRC16.h"\n#include "bbb_lut.h"\n' > "$INC/entry_pre.h"
OBJS=""
cd "$INC"
for f in bbb_tx bbb_scramble bbb_dbpsk bbb_dqpsk bbb_cck5 bbb_cck11; do
  tr -d '\r' < "$SRC/$f.c" | ${CC:-gcc} -x c -O2 -fPIC -w -I. -c - -o "$f.o"
  OBJS="$OBJS $f.o"
done
${CC:-gcc} -O2 -fPIC -w -I. -include entry_pre.h -c entry.c -o entry.o
${CC:-gcc} -shared -o "$HERE/_ref/libtx11b_legacy_ref.so.tmp.$$" $OBJS entry.o && mv -f "$HERE/_ref/libtx11b_legacy_ref.so.tmp.$$" "$HERE/_ref/libtx11b_legacy_ref.so"
echo "build_ref_tx11b: oracle/_ref/libtx11b_legacy_ref.so"
