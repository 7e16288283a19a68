"""ctypes wrapper of tests/ranked_oracle.c, the CPU oracle of the ranked placement lists (DESIGN.md 3.9; test infrastructure).

The library is compiled once per process into a temporary directory, so neither the tests nor tools/bench_ranked.py write into the
source tree."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="rio_ranked_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libranked_oracle.so")
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else (shutil.which("gcc") or "cc")
        subprocess.check_call([cc, "-O3", "-pthread", "-shared", "-fPIC", "-o", so, os.path.join(_HERE, "ranked_oracle.c"), "-lm"])
        L = C.CDLL(so)
        u64p, u32p = C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)
        L.orc_assign_ranked_hrw.restype = None
        L.orc_assign_ranked_hrw.argtypes = [u64p, C.c_size_t, u64p, u32p, C.c_uint32, C.c_uint32, u32p, C.c_int]
        L.orc_assign_ranked_hrw2.restype = None
        L.orc_assign_ranked_hrw2.argtypes = [u64p, C.c_size_t, u64p, u32p, C.c_uint32, C.c_uint32, C.c_uint32, u32p, C.c_int]
        _lib = L
    return _lib


def _args(keys, seeds, weights):
    keys = np.ascontiguousarray(keys, dtype=np.uint64)
    seeds = np.ascontiguousarray(seeds, dtype=np.uint64)
    weights = np.ascontiguousarray(weights, dtype=np.uint32)
    return keys, seeds, weights, lambda a, t: a.ctypes.data_as(C.POINTER(t))


def assign_ranked_hrw(keys, seeds, weights, ranks, threads=8):
    """(n, ranks) uint32: flat weighted rendezvous (DESIGN.md 3.4) over the live set minus the earlier ranks, rank by rank."""
    keys, seeds, weights, p = _args(keys, seeds, weights)
    out = np.empty((len(keys), ranks), dtype=np.uint32)
    lib().orc_assign_ranked_hrw(p(keys, C.c_uint64), len(keys), p(seeds, C.c_uint64), p(weights, C.c_uint32), len(seeds), ranks,
                                p(out, C.c_uint32), threads)
    return out


def assign_ranked_hrw2(keys, seeds, weights, ranks, bits=12, threads=8):
    """(n, ranks) uint32: HRW2 (DESIGN.md 3.8) over the live set minus the earlier ranks, rank by rank."""
    keys, seeds, weights, p = _args(keys, seeds, weights)
    out = np.empty((len(keys), ranks), dtype=np.uint32)
    lib().orc_assign_ranked_hrw2(p(keys, C.c_uint64), len(keys), p(seeds, C.c_uint64), p(weights, C.c_uint32), len(seeds), bits, ranks,
                                 p(out, C.c_uint32), threads)
    return out


def assign_ranked(policy, keys, seeds, weights, ranks, bits=12, threads=8):
    if policy == "hrw2":
        return assign_ranked_hrw2(keys, seeds, weights, ranks, bits=bits, threads=threads)
    return assign_ranked_hrw(keys, seeds, weights, ranks, threads=threads)
