// ORACLE — TEST INFRASTRUCTURE ONLY (see ops.h).
// Lookup tables of the reference, regenerated from closed forms that were diffed against the
// reference headers (tools/refcheck.py; tests/test_tables_vs_reference.py):
//   usin/ucos/uatan2      kernel/core/inc/intalglut.h:4,3648,7332   (P = 3.141593, as the generator used)
//   FFT twiddles          kernel/core/inc/fft_lut_twiddle.h:61434-61583
//   Viterbi branch LUTs   kernel/bb/Brick11/src/viterbilut.h:51-185
//   de-interleaver maps   kernel/bb/Brick11/src/deinterleaver.hpp:9-860
//   soft-demap tables     kernel/bb/Brick11/src/demapper.h:56-130 (data, carried run-length coded)
#pragma once
#include "ops.h"
#include <vector>

namespace sbo {

struct Tables {
    int16_t sin_lut[65536];
    int16_t cos_lut[65536];
    int16_t atan2_lut[256 * 256];
    alignas(16) c16 tw64[3][16];        // [M-1][j]
    alignas(16) c16 tw16[3][4];
    alignas(16) c16 tw128[3][32], tw32[3][8], tw8[4];   // transmit side: IFFT<128> (fft_lut_twiddle.h wFFTLUT128_*, wFFTLUT32_*, wFFTLUT8)
    alignas(16) uint8_t vit_ma[64][16]; // [soft*8 + g][lane]
    alignas(16) uint8_t vit_mb[64][16];
    uint16_t deint48[48], deint96[96], deint192[192], deint288[288];
    uint8_t demap_bpsk[256], demap_q16_2[256], demap_q64_2[256], demap_q64_3[256];
    alignas(16) c16 sts_pattern[16][16]; // TCCA11a::sts_corr_pattern (cca.hpp:266-276)
    uint8_t scramble_lut[128];           // scramble.hpp:279-296
    uint32_t crc32_lut[256];
    Tables();
};
const Tables& tables();

static inline int16_t usin(int16_t r) { return tables().sin_lut[(uint16_t)r]; }
static inline int16_t ucos(int16_t r) { return tables().cos_lut[(uint16_t)r]; }
int16_t uatan2(int y, int x);           // kernel/core/inc/intalg.h:96-108

void fft64(v128* inout /*16 vectors, destroyed*/, v128* out);   // fft_r4dif.h:134-141 FFT<64>
void ifft64(v128* inout, v128* out);                             // ifft_r4dif.h IFFT<64>
void ifft128(v128* inout /*32 vectors, destroyed*/, v128* out);  // ifft_r4dif.h:12-160 IFFT<128> = IFFTSSE<128>, 4 x (IFFTSSE<32>, 4 x IFFTSSEEx<8>), 7-bit reversal
// When set, ifft128 on this thread appends every input it is handed (128 c16 each): tests read back the symbols a transmitter transformed.
extern thread_local std::vector<c16>* ifft128_log;

} // namespace sbo
