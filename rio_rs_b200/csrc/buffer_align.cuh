// buffer_align.cuh -- the alignment the kernels of librio_cuda assume of a caller's device buffers (the _dev entry points of
// include/rio_cuda.h).  Read by csrc/engine.cu, which stages a buffer these rules do not let a launcher take in place, and by the
// host-side launcher restatements of the test suite, which report a buffer that breaks them as a launch error.
#pragma once
#include <cstdint>

namespace rio {

// ---- alignment the kernels assume of a caller's buffers (the _dev entry points of include/rio_cuda.h) -------------------------
// Bytes at which a buffer must start for the launcher to take it in place.  Every buffer the engine allocates is 256-byte aligned.
// A buffer not listed here is read and written one element at a time and needs only its element's natural alignment: 8 bytes for
// keys, 4 for node indices and features.  That covers the flat and ranked hash kernels, the failure-domain walks, the CUDA-core
// affinity kernel for K != 16, the no-live-node fill and the directory lookup and upsert.
constexpr uint32_t kAlignTrieKeys = 16;   // launch_assign_trie, dense form: k_assign_trie loads two keys per ulonglong2
constexpr uint32_t kAlignTrieOut = 8;     // launch_assign_trie, dense form: k_assign_trie stores two indices per uint2
// The feature rows of launch_assign_affinity(_ranked, _spread) and of the tensor-core launchers: at K == 16 every one of them loads
// rows as float4 (the wgmma passes as float2).
inline uint32_t affinity_feats_align(uint32_t K) { return K == 16 ? 16u : 4u; }

}  // namespace rio
