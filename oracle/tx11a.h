// ORACLE — TEST INFRASTRUCTURE ONLY (see ops.h).
// CPU restatement of the reference's 802.11a brick transmit graphs
//   kernel/bb/demod11/fb11amod_config.hpp:75-118 (CreateModGraph11a_40M) and :150-158 (CreatePreamble11a_40M),
//   driven like kernel/bb/demod11/fb11a_mod.cpp:27-107 (Test11A_FB_Mod: preamble, then SIGNAL + DATA, 32 trailing zero samples).
// PINNED BY THE COMPILED GRAPH: the reference holds no output vector of this brick graph (usr/HwVeri/data/ofdm.bin, tests/golden/ofdm.bin,
// comes from the legacy transmitter, another window and IFFT rounding, and matches this restatement to +-1 away from symbol edges), but
// oracle/build_ref_mod.sh compiles the graph's own bricks where they lie, and every stage below and whole frames at all 8 rates equal them
// bit for bit (tests/test_cpu_tx_reference.py).  Only the 40 Msps graph is compiled; CreateModGraph11a_44M is not.
#pragma once
#include "tables.h"
#include <stddef.h>
#include <vector>

namespace sbo {
// preamble as TTS11aSrc builds it (Brick11/src/preamble11a.hpp:22-104), 640 x COMPLEX16 before the 16->8 bit pack
void tx11a_preamble16(c16* out640);
// whole PPDU as COMPLEX8 pairs (re, im): 640 + 160 * (1 + nsym) samples followed by `tail_zeros` zero samples.
// payload = MPDU without FCS (the modulator appends CRC-32).  Returns the number of complex samples written (0 on bad arguments).
size_t tx11a_modulate(const uint8_t* payload, uint32_t len, uint32_t rate_kbps, uint8_t sc_seed, int8_t* out, size_t cap_samples, uint32_t tail_zeros);
// symbol count the reference transmits (TBB11aSrc::GetPadingByte, PHY_11a.hpp:107-123): the tail is counted as a whole byte and
// 9 Mbps pads to a pair of symbols, so this can exceed the standard's N_SYM by one
uint32_t tx11a_nsym(uint32_t len, uint32_t rate_kbps);
// the stages tx11a_modulate chains, each as the brick it restates (bits one per byte, LSB of each input byte first):
//   T11aSc: n bytes under the per-byte scramble_ctrl (0 none, 1 scramble, 2 tail), register carried in reg
void tx11a_scramble(const uint8_t* in, const uint8_t* ctrl, size_t n, uint8_t& reg, uint8_t* out);
//   TConvEncode_12 / _23 / _34 (cr CR_12 / CR_23 / CR_34) from state 0: coded bits in air order before interleaving
void tx11a_encode_bits(const std::vector<uint8_t>& bytes, int cr, std::vector<uint8_t>& coded);
//   T11Interleave: 48 * nbpsc coded bits -> the same bits in on-air order
void tx11a_interleave(const uint8_t* coded, int nbpsc, uint8_t* air);
//   TMap11a*<>: 48 * nbpsc on-air bits -> 48 data points
void tx11a_map(const uint8_t* air, int nbpsc, c16* d48);
//   T11aAddPilot<>: 48 data points -> 64 carriers with the pilots of pilot_index, which then advances
void tx11a_add_pilot(const c16* d48, unsigned& pilot_index, c16* f64);
//   TIFFTx: 64 carriers -> 160 samples;  TPackSample16to8: n COMPLEX16 -> n COMPLEX8 (saturating)
void tx11a_ifftx(const c16* f64, c16* out160);
void tx11a_pack8(const c16* in, size_t n, int8_t* out);
// the LEGACY transmitter (tx11a_legacy.cpp): BB11ATxFrameMod / BB11ATxBufferMod6M; pinned by usr/HwVeri/data/ofdm.bin
size_t tx11a_legacy_modulate(const uint8_t* mpdu, uint32_t len, int append_crc, uint32_t rate_kbps, const c16* preamble640, int8_t* out, size_t cap_samples);
uint32_t tx11a_legacy_nsym(uint32_t psdu_len, uint32_t rate_kbps);
}
