// sora_b200 — OFDM subcarrier bookkeeping shared by the 802.11a and 802.11n receive kernels: where bin i of warp_fft64's output sits,
// and the 802.11a data-subcarrier order.  Device code only (__brev): the host emulators that compile fixed.cuh and tables.cuh do not need it.
#pragma once

namespace sb {

__device__ __forceinline__ int bitrev6(int i) { return (int)(__brev((unsigned)i) >> 26); }

__device__ __forceinline__ int data_index(int bin) {   // demapper11a.hpp:22-36 subcarrier order; -1 for non-data bins
    if (bin >= 38) { if (bin == 43 || bin == 57) return -1; return bin - 38 - (bin > 43) - (bin > 57); }
    if (bin >= 1 && bin <= 26) { if (bin == 7 || bin == 21) return -1; return 24 + bin - 1 - (bin > 7) - (bin > 21); }
    return -1;
}
__device__ __forceinline__ int data_bin(int d) {       // inverse of data_index, d = 0..47
    return d < 24 ? 38 + d + (d >= 5) + (d >= 18) : d - 23 + (d >= 30) + (d >= 43);
}

} // namespace sb
