"""ctypes wrapper of tests/affinity_c32_ref.c, the exact fp32 reference of the affinity cost c32 (DESIGN.md 3.6; test
infrastructure) and of the ranked (3.9) and failure-domain (3.14) lists it defines.

The library is compiled once per process into a temporary directory, so nothing is written into the source tree.  MUTANTS name the
cost functions a subtly wrong kernel could compute; they exist only to show that the fixtures of tests/test_gpu_affinity_c32.py tell
them apart from c32."""
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
C32 = 0
MUTANTS = {"separate multiply and add": 1, "reversed k order": 2, "fp64 dot rounded to fp32": 3, "pairwise summation": 4,
           "integer-image order": 5, "bf16 product only": 6, "split without hl": 7}
SPLIT6 = 8
THREADS = max(1, min(32, os.cpu_count() or 1))


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="rio_c32_ref_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libaffinity_c32_ref.so")
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else (shutil.which("gcc") or "cc")
        subprocess.check_call([cc, "-O2", "-ffp-contract=off", "-fno-fast-math", "-pthread", "-shared", "-fPIC", "-o", so,
                               os.path.join(_HERE, "affinity_c32_ref.c"), "-lm"])
        L = C.CDLL(so)
        fp, dp, u8p, u32p = C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_uint8), C.POINTER(C.c_uint32)
        L.c32_costs.restype = None
        L.c32_costs.argtypes = [fp, C.c_uint64, fp, C.c_uint32, C.c_uint32, C.c_int, fp, dp, C.c_int]
        L.c32_lists.restype = None
        L.c32_lists.argtypes = [fp, C.c_uint64, fp, C.c_uint32, C.c_uint32, u8p, u32p, C.c_uint32, C.c_int, u32p, C.c_int]
        _lib = L
    return _lib


def _p(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def _feats(fo, fn):
    fo = np.ascontiguousarray(fo, dtype=np.float32)
    fn = np.ascontiguousarray(fn, dtype=np.float32)
    assert fo.ndim == fn.ndim == 2 and fo.shape[1] == fn.shape[1] and 1 <= fo.shape[1] <= 256
    return fo, fn


def c32(fo, fn, mode=C32):
    """(n, M) float32: -acc with acc = fmaf(f[k], F[j][k], acc) for k = 0..K-1 from 0.f (mode C32), or a mutant's cost."""
    fo, fn = _feats(fo, fn)
    out = np.empty((len(fo), len(fn)), dtype=np.float32)
    lib().c32_costs(_p(fo, C.c_float), len(fo), _p(fn, C.c_float), len(fn), fo.shape[1], mode, _p(out, C.c_float), None, THREADS)
    return out


def S(fo, fn):
    """(n, M) float64: sum_k |f_k F_jk|, the scale of the error bounds."""
    fo, fn = _feats(fo, fn)
    out = np.empty((len(fo), len(fn)), dtype=np.float64)
    lib().c32_costs(_p(fo, C.c_float), len(fo), _p(fn, C.c_float), len(fn), fo.shape[1], C32, None, _p(out, C.c_double), THREADS)
    return out


def _lists(fo, fn, live, dom, R, mode):
    fo, fn = _feats(fo, fn)
    live = np.ascontiguousarray(live, dtype=np.uint8)
    assert len(live) == len(fn)
    if dom is not None:
        dom = np.ascontiguousarray(dom, dtype=np.uint32)
        assert len(dom) == len(fn)
    out = np.empty((len(fo), R), dtype=np.uint32)
    lib().c32_lists(_p(fo, C.c_float), len(fo), _p(fn, C.c_float), len(fn), fo.shape[1], _p(live, C.c_uint8), _p(dom, C.c_uint32), R, mode,
                    _p(out, C.c_uint32), THREADS)
    return out


def ranked(fo, fn, live, R, mode=C32):
    """(n, R) uint32: the first R live nodes in (c32, j) order, NONE past the live set.  Unranked is ranked(..., 1)."""
    return _lists(fo, fn, live, None, R, mode)


def spread(fo, fn, live, dom, R, mode=C32):
    """(n, R) uint32: the best R domain representatives in (c32, j) order (DESIGN.md 3.14); a label of NONE is a domain of its own."""
    return _lists(fo, fn, live, dom, R, mode)
