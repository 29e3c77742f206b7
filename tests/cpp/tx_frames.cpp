// Host build of sora_b200/csrc/tx_frames.cuh, for tests/test_cpu_tx_frames.py: the rate tables and the smallest out_stride_samples each batch
// transmitter accepts for a frame, composed from the header's sizing functions the way the per-slot checks of tx.cu compose them.  Every
// strides_* function fills out[len] for len = 0 .. n - 1 (MPDU bytes without FCS, or PSDU bytes with it for the legacy transmitters) and
// returns 0, or -1 for a rate the table does not have.
//
//   g++ -O2 -std=c++17 -shared -fPIC -I sora_b200/csrc -o tx_frames.so tests/cpp/tx_frames.cpp
#include "tx_frames.cuh"

using namespace sb;

extern "C" {

uint32_t ndbps_11a(uint32_t kbps) { const Rate11a* r = find_rate(kRates11a, kbps); return r ? r->ndbps : 0; }
uint32_t chips_11b(uint32_t kbps) { const Rate11b* r = find_rate(kRates11b, kbps); return r ? r->chips_per_byte : 0; }
uint32_t ndbps_11n(uint32_t mcs) { const Mcs11n* m = find_rate(kMcs11n, mcs, &Mcs11n::mcs); return m ? m->ndbps : 0; }

int strides_11a(uint32_t kbps, uint32_t lead, uint32_t n, uint64_t* out) {
    const Rate11a* r = find_rate(kRates11a, kbps);
    if (!r) return -1;
    for (uint32_t len = 0; len < n; len++) out[len] = lead + tx11a_samples(tx11a_nsym(len, r->ndbps, r->ndbps_pad));
    return 0;
}
int strides_11b(uint32_t kbps, uint32_t lead, uint32_t n, uint64_t* out) {
    const Rate11b* r = find_rate(kRates11b, kbps);
    if (!r) return -1;
    for (uint32_t len = 0; len < n; len++) out[len] = (uint64_t)lead + tx11b_nsamples(tx11b_nchips(len, r->chips_per_byte));
    return 0;
}
int strides_11n(uint32_t mcs, uint32_t lead, uint32_t n, uint64_t* out) {
    const Mcs11n* m = find_rate(kMcs11n, mcs, &Mcs11n::mcs);
    if (!m) return -1;
    const Tx11nJob job = tx11n_job(*m, lead);
    for (uint32_t len = 0; len < n; len++) out[len] = lead + tx11n_samples(tx11n_nsym_emitted(len, job, nullptr, nullptr));
    return 0;
}
int strides_11b_legacy(uint32_t kbps, uint32_t short_preamble, uint32_t n, uint64_t* out) {
    const Rate11b* r = find_rate(kRates11b, kbps);
    if (!r) return -1;
    for (uint32_t size = 0; size < n; size++) out[size] = tx11b_legacy_nsamples(size, short_preamble, tx11b_legacy_data_chips(*r, short_preamble));
    return 0;
}
int strides_11a_legacy(uint32_t kbps, uint32_t sample_rate_mhz, uint32_t n, uint64_t* out) {
    const Rate11a* r = find_rate(kRates11a, kbps);
    if (!r) return -1;
    for (uint32_t size = 0; size < n; size++) out[size] = tx11a_legacy_padded(tx11a_legacy_nsym(size, r->ndbps), sample_rate_mhz == 44);
    return 0;
}

}
