"""Builds librio_cuda.so in-tree with nvcc for sm_90a (H100), ahead of time: no JIT cache, nothing compiled at run time."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "librio_cuda.so")
SOURCES = ["k_assign.cu", "k_trie.cu", "k_ranked.cu", "k_spread.cu", "k_affinity_umma.cu", "k_affinity_set.cu", "k_affinity_bounded.cu", "k_set_bounded_affinity.cu", "k_directory.cu", "engine.cu", "resolver.cu", "durable.cu"]
HEADERS = ["kernels.cuh", "buffer_align.cuh", "k_ranked.cuh", "k_rank_common.cuh", "k_spread.cuh", "k_affinity_ranked.cuh", "k_affinity_spread.cuh", "k_affinity_set.cuh", "k_affinity_bounded.cuh", "k_set_bounded_affinity.cuh", "k_affinity_common.cuh", "k_changes.cuh", "k_ranked_changes.cuh", "k_spread_changes.cuh", "spec.cuh", "bounded_tail.cuh", "trie_table.hpp", os.path.join("..", "..", "include", "rio_cuda.h"), os.path.join("..", "..", "include", "rio_cuda_dev.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def is_fresh():
    if not os.path.exists(SO):
        return False
    t = os.path.getmtime(SO)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS]
    return all(os.path.getmtime(d) <= t for d in deps)


def build(force=False, verbose=False):
    """Compile every CUDA source of the product into rio_rs_b200/librio_cuda.so.  RIO_BUILD_TUNING=1 also compiles the A/B
    tuning points of the flat rendezvous kernel (tools/tune_assign.py); the shipped library carries the default only."""
    if not force and is_fresh():
        return SO
    cmd = [_nvcc()] + NVCC_FLAGS + (["-DRIO_ASSIGN_TUNING"] if os.environ.get("RIO_BUILD_TUNING") else []) + (["-Xptxas", "-v"] if verbose else []) + ["-o", SO] + [os.path.join(CSRC, s) for s in SOURCES] + ["-ldl"]
    env = dict(os.environ)
    env.pop("CC", None)   # nvcc picks its host compiler itself; a CC meant for other builds must not override it
    env.pop("CXX", None)
    subprocess.check_call(cmd, env=env)
    return SO


if __name__ == "__main__":
    import sys
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
