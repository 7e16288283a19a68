// set_commit_launchers.cpp -- TEST INFRASTRUCTURE: host restatements of the launchers declared in csrc/k_set_commit.cuh, linked beside
// launchers.cpp and the other doubles by tests/test_gpu_set_commit.py so that rio_cuda_set_commit_changes runs without a GPU.
//
// Like launchers.cpp: each function does, sequentially and in the plainest way, what the launcher is SPECIFIED to do (DESIGN.md 3.20).
// Nothing here says anything about the kernels.
#include "../../../rio_rs_b200/csrc/k_set_commit.cuh"
#include "../../../rio_rs_b200/csrc/spec.cuh"

namespace rio {

static uint32_t answer(const DirDev &dir, uint64_t raw) {
    const unsigned long long key = raw == kEmptyKey ? kEmptyKey - 1 : raw;
    uint64_t s = (key * kGolden64) >> dir.shift;
    for (uint64_t probes = 0; probes <= dir.mask; probes++, s = (s + 1) & dir.mask) {
        if (dir.slots[s].key == key) return (uint32_t)dir.slots[s].val;
        if (dir.slots[s].key == kEmptyKey) break;
    }
    return kNone;
}

void launch_commit_diff(const Launch &L, const DirDev &dir, const uint64_t *keys, const uint32_t *idx, uint64_t n, uint8_t *flag, uint32_t *from,
                        uint32_t *block_cnt, uint32_t *block_off, unsigned long long *total) {
    if (!n) return;
    const uint64_t nb = (n + kCommitRows - 1) / kCommitRows;
    for (uint64_t b = 0; b < nb; b++) block_cnt[b] = 0;
    for (uint64_t i = 0; i < n; i++) {
        const uint32_t a = answer(dir, keys[i]);
        flag[i] = a != idx[i] ? 1 : 0;
        if (flag[i]) { from[i] = a; block_cnt[i / kCommitRows]++; }
    }
    uint32_t run = 0;
    for (uint64_t b = 0; b < nb; b++) { block_off[b] = run; run += block_cnt[b]; }
    *total = run;
    if (L.launch_counter) *L.launch_counter += 2;
}

void launch_commit_list(const Launch &L, const uint64_t *keys, const uint32_t *idx, uint64_t n, const uint8_t *flag, const uint32_t *from, const uint32_t *,
                        const uint32_t *, uint64_t *rows, uint64_t *mkeys, uint32_t *mfrom, uint32_t *mto) {
    if (!n) return;
    uint64_t j = 0;
    for (uint64_t i = 0; i < n; i++) {
        if (!flag[i]) continue;
        rows[j] = i; mkeys[j] = keys[i]; mfrom[j] = from[i]; mto[j] = idx[i];
        j++;
    }
    if (L.launch_counter) ++*L.launch_counter;
}

}  // namespace rio
