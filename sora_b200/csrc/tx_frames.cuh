// sora_b200 — the transmitters' rates and frame lengths, stated once: the rate tables of 802.11a, 802.11b and 802.11n (MCS 8 .. 14), the
// code rates, and the sizing arithmetic the kernels, the batch calls (tx.cu) and the legacy entry points (legacy_shim.cpp) share.  Plain
// structs and arithmetic only, so that host C++ without CUDA can include it too.
#pragma once
#include <stddef.h>
#include <stdint.h>

#ifdef __CUDACC__
#define SB_HD __host__ __device__
#else
#define SB_HD
#endif

namespace sb {

enum { CR_12 = 0, CR_23 = 1, CR_34 = 2 };              // convolutional code rates (the Viterbi kernels take them as a template parameter)

// 802.11a rates: SIGNAL rate code, coded bits per subcarrier, code rate, data bits per symbol (ieee80211a_cmn.h:66-157; bba.h:179-186,
// atx.h:20-57), and the N_DBPS the brick modulator's padding rule uses (doubled at 9 Mbps, PHY_11a.hpp:113-116)
struct Rate11a { uint32_t kbps, code, nbpsc, cr, ndbps, ndbps_pad; };
constexpr Rate11a kRates11a[8] = {{6000, 0xB, 1, CR_12, 24, 24}, {9000, 0xF, 1, CR_34, 36, 72}, {12000, 0xA, 2, CR_12, 48, 48},
    {18000, 0xE, 2, CR_34, 72, 72}, {24000, 0x9, 4, CR_12, 96, 96}, {36000, 0xD, 4, CR_34, 144, 144}, {48000, 0x8, 6, CR_23, 192, 192},
    {54000, 0xC, 6, CR_34, 216, 216}};
// 802.11b rates: SIGNAL rate code, chips per PSDU byte (bb/bbb.h:47-50, DataRate.h:40-43)
struct Rate11b { uint32_t kbps, code, chips_per_byte; };
constexpr Rate11b kRates11b[4] = {{1000, 0x0A, 88}, {2000, 0x14, 44}, {5500, 0x37, 16}, {11000, 0x6E, 8}};
// 802.11n MCS 8 .. 14, two spatial streams (ieee80211const.h:35-55; the range the receiver accepts, PHY_11n.hpp:496-501): N_BPSCS, code rate,
// N_DBPS over both streams, input bursts of the encoder and of the stream parser in bytes.  MCS 11 .. 14 are the 16-QAM / 64-QAM branches
// of the modulator graph (fb11nmod_config.hpp:133-155: enc11 .. enc14).
struct Mcs11n { uint32_t mcs, nbpsc, cr, ndbps, enc_in, parse_in; };
constexpr Mcs11n kMcs11n[7] = {{8, 1, CR_12, 52, 1, 13}, {9, 2, CR_12, 104, 1, 26}, {10, 2, CR_34, 156, 3, 26}, {11, 4, CR_12, 208, 1, 52},
    {12, 4, CR_34, 312, 3, 52}, {13, 6, CR_23, 416, 2, 78}, {14, 6, CR_34, 468, 3, 78}};

// The entry of `rates` whose `key` (the rate in kbps unless told otherwise) is v, or null
template <class R, size_t N> const R* find_rate(const R (&rates)[N], uint32_t v, uint32_t R::*key = &R::kbps) {
    for (const R& r : rates) if (r.*key == v) return &r;
    return nullptr;
}

// ---- 802.11a (tx11a_kernels.cuh) ----
SB_HD inline uint32_t tx11a_nsym(uint32_t len, uint32_t ndbps, uint32_t ndbps_pad) {   // TBB11aSrc::GetPadingByte
    const uint32_t bits = (2u + len + 4u + 1u) * 8u, padded = (bits + ndbps_pad - 1u) / ndbps_pad * ndbps_pad;
    return (bits + ((padded - bits + 7u) / 8u) * 8u) / ndbps;
}
// samples of a frame behind its lead: the preamble, SIGNAL and nsym data symbols
inline uint64_t tx11a_samples(uint32_t nsym) { return 640u + 160ull * (1u + nsym); }

// ---- 802.11b (tx11b_kernels.cuh) ----
SB_HD inline uint32_t tx11b_nchips(uint32_t len, uint32_t chips_per_byte) { return 24u * 88u + (len + 4u) * chips_per_byte; }
SB_HD inline uint32_t tx11b_nsamples(uint32_t nchips) { return ((nchips + 5u) * 4u + 7u) / 8u * 8u; }   // + 5 flush vectors, bursts of 8

// ---- legacy 802.11b (tx11b_legacy_kernels.cuh) ----
SB_HD inline uint32_t tx11b_legacy_plcp_bytes(uint32_t short_preamble) { return short_preamble ? 15u : 24u; }
SB_HD inline uint32_t tx11b_legacy_header_chips(uint32_t short_preamble) { return short_preamble ? 9u * 88u + 6u * 44u : 24u * 88u; }
// chips per PSDU byte: the short preamble's 1 Mbps case sends no data chips (the reference's switch has no such case)
inline uint32_t tx11b_legacy_data_chips(const Rate11b& r, uint32_t short_preamble) { return short_preamble && r.kbps == 1000 ? 0u : r.chips_per_byte; }
SB_HD inline uint32_t tx11b_legacy_nsamples(uint32_t psdu_len, uint32_t short_preamble, uint32_t data_chips_per_byte) {
    const uint32_t n = 4u * (tx11b_legacy_header_chips(short_preamble) + psdu_len * data_chips_per_byte);
    return (n + 37u + 127u) & ~127u;                                                   // TX_FIR_DEPTH zeros, rounded up to a multiple of 128
}

// ---- legacy 802.11a (tx11a_legacy_kernels.cuh) ----
SB_HD inline uint32_t tx11a_legacy_nsym(uint32_t psdu_len, uint32_t ndbps) { return (22u + 8u * psdu_len + ndbps - 1u) / ndbps; }
// GetSignalBytes / 2 (atx_tpl.h:69-83) and its RCB padding to 128 bytes (_tx_manager2.h:29-38)
SB_HD inline uint32_t tx11a_legacy_signal(uint32_t nsym, uint32_t sr44) { return (sr44 ? 176u : 160u) * (5u + nsym) + 8u; }
SB_HD inline uint32_t tx11a_legacy_padded(uint32_t nsym, uint32_t sr44) { return (tx11a_legacy_signal(nsym, sr44) + 63u) & ~63u; }

// ---- 802.11n (tx11n_kernels.cuh) ----
struct Tx11nJob {
    uint32_t mcs, nbpsc, code_rate, ndbps;   // 8..14; N_BPSCS; CR_12 / CR_23 / CR_34; N_DBPS over both streams
    uint32_t enc_in, parse_in;               // input bursts of the encoder and of the stream parser, bytes (conv_enc.hpp, streamparser.hpp)
    uint32_t lead, max_sym;                  // zero samples in front; symbols per frame the grid covers (3 SIG + data)
};
inline Tx11nJob tx11n_job(const Mcs11n& m, uint32_t lead) { return Tx11nJob{m.mcs, m.nbpsc, m.cr, m.ndbps, m.enc_in, m.parse_in, lead, 0}; }
SB_HD inline uint32_t tx11n_nsym_signalled(uint32_t len, uint32_t ndbps) { return ((len + 4u) * 8u + 16u + 6u + ndbps - 1u) / ndbps; }   // ht_symbol_count
// data symbols the graph emits: the Flush padding (FlushPort: encoder burst, then stream-parser burst) can add one
SB_HD inline uint32_t tx11n_nsym_emitted(uint32_t len, const Tx11nJob& j, uint32_t* enc_bits, uint32_t* coded_bits) {
    const uint32_t ns = tx11n_nsym_signalled(len, j.ndbps);
    uint32_t bytes = (ns * j.ndbps + 7u) / 8u; bytes = (bytes + j.enc_in - 1u) / j.enc_in * j.enc_in;
    const uint32_t cbytes = j.code_rate == CR_12 ? 2u * bytes : j.code_rate == CR_34 ? bytes / 3u * 4u : bytes / 2u * 3u;
    if (enc_bits) *enc_bits = bytes * 8u; if (coded_bits) *coded_bits = cbytes * 8u;
    return (cbytes + j.parse_in - 1u) / j.parse_in;
}
// samples of a frame behind its lead: L-STF, L-LTF, L-SIG, HT-SIG, HT-STF, two HT-LTFs and nsym data symbols
inline uint64_t tx11n_samples(uint32_t nsym) { return 1600u + 160ull * nsym; }

} // namespace sb
