"""Builds the C++ conformance harness against the C++ mirror of the trait and runs it (GPU), and checks on CPU that it
compiles and links against librio_cuda.so.  The harnesses are compiled into a temporary directory, once per process, so the
suite also runs from a read-only source tree."""
import atexit
import os
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_EXES = {}


def _build(name="backend_conformance"):
    from rio_rs_b200 import build

    build.build()
    if name not in _EXES:
        d = tempfile.mkdtemp(prefix="rio_cpp_harness_")
        atexit.register(shutil.rmtree, d, True)
        exe = os.path.join(d, name)
        src = os.path.join(ROOT, "tests", "cpp", name + ".cpp")
        libdir = os.path.join(ROOT, "rio_rs_b200")
        subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-o", exe, src, "-L" + libdir, "-lrio_cuda", "-Wl,-rpath," + libdir])
        _EXES[name] = exe
    return _EXES[name]


def test_cpp_mirror_compiles_and_links():
    assert os.path.exists(_build())


@pytest.mark.gpu
def test_cpp_backend_conformance_on_gpu():
    r = subprocess.run([_build()], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "all passed" in r.stdout


def test_cpp_durable_harness_compiles_and_links():
    assert os.path.exists(_build("durable_conformance"))


@pytest.mark.gpu
def test_cpp_durable_conformance_on_gpu(tmp_path):
    """The reference's SqliteObjectPlacement tests + restart recovery + the written-through place_batch, through the C ABI
    (rio_cuda_durable_*, libsqlite3.so.0 dlopen'ed): SURVEY 8(f) row 3 below the language bindings."""
    r = subprocess.run([_build("durable_conformance"), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "durable: all passed" in r.stdout
