// k_set_commit.cuh -- launchers of the delta commit of a resident set (DESIGN.md 3.20): one pass that compares every row's idx with what
// the directory answers for its key, a one-block scan of the per-block selected counts, and the ordered manifest of the selected rows.
// The kernels live in k_directory.cu beside k_dir_lookup and share its key normalisation, home slot and probe loop.  The write itself
// is the existing directory upsert over the manifest's keys and targets.
#pragma once
#include "kernels.cuh"

namespace rio {

// rows per block of the diff and list passes (256 threads x 4 rows): d_block_cnt and d_block_off have one entry per kCommitRows rows
constexpr uint32_t kCommitRows = 1024;

// Declared weak, as in k_changes.cuh: the engine's host code can be linked without these launchers (rio_cuda_set_commit_changes then
// answers with an error); librio_cuda.so always links them.
//
// n > 0 rows.  d_flag[i] = 1 iff d_idx[i] differs from the directory's answer for d_keys[i] (RIO_NONE for an absent or removed key; the
// key normalised as the directory normalises it), else 0; for a selected row d_from[i] = that answer (other entries are not written).
// d_block_cnt[b] = the selected rows of [b * kCommitRows, (b + 1) * kCommitRows), d_block_off[b] = the selected rows before that range,
// *d_total = all of them.
__attribute__((weak)) void launch_commit_diff(const Launch &L, const DirDev &dir, const uint64_t *d_keys, const uint32_t *d_idx, uint64_t n,
                                              uint8_t *d_flag, uint32_t *d_from, uint32_t *d_block_cnt, uint32_t *d_block_off,
                                              unsigned long long *d_total);
// From the outputs of launch_commit_diff: the j-th selected row i, in increasing row order, gives d_rows[j] = i, d_mkeys[j] = d_keys[i]
// (as stored), d_mfrom[j] = d_from[i] and d_mto[j] = d_idx[i].
__attribute__((weak)) void launch_commit_list(const Launch &L, const uint64_t *d_keys, const uint32_t *d_idx, uint64_t n, const uint8_t *d_flag,
                                              const uint32_t *d_from, const uint32_t *d_block_cnt, const uint32_t *d_block_off, uint64_t *d_rows,
                                              uint64_t *d_mkeys, uint32_t *d_mfrom, uint32_t *d_mto);

}  // namespace rio
