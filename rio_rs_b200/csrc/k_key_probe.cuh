// k_key_probe.cuh -- the first probe of the open-addressing key tables that the set kernels build per call: the erase-key hash set
// of set_erase (DESIGN.md 3.18) and the key -> position table of set_write_weights_by_key (3.21).  Device code only.
#pragma once
#include "k_set_churn.cuh"

namespace rio {

// a key's first slot in a table of 1 << lg slots: the top lg bits of key * kChurnHashMul
__device__ __forceinline__ uint64_t churn_slot(unsigned long long key, uint32_t lg) { return (key * kChurnHashMul) >> (64 - lg); }

}  // namespace rio
