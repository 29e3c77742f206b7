// ORACLE — TEST INFRASTRUCTURE ONLY (see ops.h).
// CPU restatement of the reference's 802.11b brick transmit graph
//   kernel/bb/demod11/fb11bmod_config.hpp:19-45 (CreateModGraph: TBB11bSrc -> TSc741 -> TBB11bMRSelect ->
//   {TBB11bDBPSKSpread, TBB11bDQPSKSpread, TCCK5Encode, TCCK11Encode} -> TQuickPulseShaper -> TPackSample16to8 -> TModSink),
//   driven like kernel/bb/demod11/fb11b_mod.cpp:28-32 (Process then Flush).
// PARITY UNPINNED: the reference holds no output vector of this graph (the *.mf.bin captures under kernel/HWTest come from another
// shaping filter: 18 leading zeros and a 1,0,-2,0,4 ramp that neither this graph's 20-tap shaper nor the legacy 37-tap FIR produces).
// What is checked: the stage tables rebuilt from the reference's formulas, and a round trip through the receive oracle, which IS
// pinned by those captures.  Not yet compared with the graph's own compiled bricks (oracle/build_ref_mod.sh compiles the 802.11a
// modulator only).
#pragma once
#include <stdint.h>
#include <stddef.h>

namespace sbo {
// chips the frame occupies (long preamble + PLCP header at 1 Mbps, PSDU = payload + CRC-32 at rate_kbps); 0 for an unknown rate
uint32_t tx11b_nchips(uint32_t len, uint32_t rate_kbps);
// samples TModSink ends up holding: 4 per chip plus the shaper's 5 flush vectors, padded to TPackSample16to8's burst of 8
uint32_t tx11b_nsamples(uint32_t len, uint32_t rate_kbps);
// Whole PPDU at 44 Msps as COMPLEX8 pairs.  payload = MPDU without FCS; init_phase = CF_DifferentialMap::last_phase before the
// first byte (0 on a fresh context; the reference never resets it between frames).  Returns samples written (0: bad arguments).
// final_phase (may be NULL) receives last_phase as the graph leaves it, i.e. the next frame's init_phase on the same context.
size_t tx11b_modulate(const uint8_t* payload, uint32_t len, uint32_t rate_kbps, uint32_t init_phase, int8_t* out, size_t cap_samples, uint32_t* final_phase = nullptr);
// the twenty shaper taps h(8) .. h(-11) (pulse.hpp:279-305)
void tx11b_taps(int16_t* out20);
}
