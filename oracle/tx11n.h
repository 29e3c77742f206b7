// ORACLE — TEST INFRASTRUCTURE ONLY (see ops.h).
// CPU restatement of the reference's 802.11n two-stream HT-mixed-format transmit graphs
//   kernel/bb/demod11/fb11nmod_config.hpp:74-171 (CreateSigGraph11n, CreateModGraph11n, CreatePreambleGraph11n), driven like
//   kernel/bb/demod11/fb11n_mod.cpp:44-70 (L-STF + L-LTF, L-SIG + HT-SIG x 2, HT-STF + HT-LTF x 2, DATA; Process then Flush).
// Purpose: the reference ships no 802.11n vector at all (SURVEY.md §8c), so the receive oracle (rx11n.cpp) cannot be pinned; this
// restates the OTHER half of the reference's 11n code, so that the two independently restated halves can be played against each other
// (tests/test_cpu_oracle_tx11n.py).  PARITY UNPINNED like the receive side; the four preamble tables are regenerated from their
// defining formula and compared with the reference's literal tables when the reference tree is present.  Not yet compared with the
// graphs' own compiled bricks (oracle/build_ref_mod.sh compiles the 802.11a modulator only).
#pragma once
#include "tables.h"
#include <stddef.h>

namespace sbo {
// The four 40 Msps preamble tables (Brick11/src/_b_lstf.h:105-125, _b_lltf.h:108-130, _b_htstf.h:105-117, _b_htltf.h): 128-point inverse
// DFTs of the L-STF / L-LTF / HT-LTF tone sets, each scaled to the same total power (x sqrt(24 / tones)) times one common amplitude,
// rounded to nearest.  lstf[320] starts at n = 0, lltf[320] at n = -64 (double guard interval), htstf[160] and htltf[160] at n = -32.
void tx11n_preamble_tables(c16* lstf320, c16* lltf320, c16* htstf160, c16* htltf160);
// data symbols the graph emits: ht_symbol_count (ieee80211n_cmn.h:35-41) plus the extra symbol the Flush padding produces when the
// padded byte stream does not end on a symbol boundary
uint32_t tx11n_nsym(uint32_t len, uint32_t mcs, uint32_t* nsym_signalled);
// Whole PPDU, two streams of COMPLEX16 at 40 Msps: 640 + 480 + 480 + 160 * symbols samples each.  payload = MPDU without FCS, mcs 8..10
// (the receiver's range), seed = CF_ScramblerSeed::sc_seed (0xAB in fb11nmod_config.hpp:52).  Returns samples per stream (0: bad arguments).
size_t tx11n_modulate(const uint8_t* payload, uint32_t len, uint32_t mcs, uint8_t sc_seed, c16* out0, c16* out1, size_t cap_samples);
}
