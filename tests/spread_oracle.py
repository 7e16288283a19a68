"""ctypes wrapper of tests/spread_oracle.c, the CPU oracle of the failure-domain ranked lists (DESIGN.md 3.12; test infrastructure).

The library is compiled once per process into a temporary directory, so neither the tests nor tools/bench_ranked_spread.py write into
the source tree."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None
NONE = 0xFFFFFFFF


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="rio_spread_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libspread_oracle.so")
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else (shutil.which("gcc") or "cc")
        subprocess.check_call([cc, "-O3", "-pthread", "-shared", "-fPIC", "-o", so, os.path.join(_HERE, "spread_oracle.c"), "-lm"])
        L = C.CDLL(so)
        u64p, u32p = C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)
        L.orc_assign_spread_hrw.restype = None
        L.orc_assign_spread_hrw.argtypes = [u64p, C.c_size_t, u64p, u32p, u32p, C.c_uint32, C.c_uint32, u32p, C.c_int]
        L.orc_assign_spread_hrw2.restype = None
        L.orc_assign_spread_hrw2.argtypes = [u64p, C.c_size_t, u64p, u32p, u32p, C.c_uint32, C.c_uint32, C.c_uint32, u32p, C.c_int]
        _lib = L
    return _lib


def assign_spread(policy, keys, seeds, weights, domains, ranks, bits=12, threads=8):
    """(n, ranks) uint32: the policy's placement over the live set minus the domains of the earlier ranks, rank by rank.
    weights[j] == 0: node j is not live; domains[j] == NONE: node j is a domain of its own."""
    keys = np.ascontiguousarray(keys, dtype=np.uint64)
    seeds = np.ascontiguousarray(seeds, dtype=np.uint64)
    weights = np.ascontiguousarray(weights, dtype=np.uint32)
    domains = np.ascontiguousarray(domains, dtype=np.uint32)
    assert len(seeds) == len(weights) == len(domains)
    out = np.empty((len(keys), ranks), dtype=np.uint32)
    p = lambda a, t: a.ctypes.data_as(C.POINTER(t))
    if policy == "hrw2":
        lib().orc_assign_spread_hrw2(p(keys, C.c_uint64), len(keys), p(seeds, C.c_uint64), p(weights, C.c_uint32), p(domains, C.c_uint32),
                                     len(seeds), bits, ranks, p(out, C.c_uint32), threads)
    else:
        lib().orc_assign_spread_hrw(p(keys, C.c_uint64), len(keys), p(seeds, C.c_uint64), p(weights, C.c_uint32), p(domains, C.c_uint32),
                                    len(seeds), ranks, p(out, C.c_uint32), threads)
    return out
