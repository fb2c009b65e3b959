"""In-tree build of libdra_alloc.so for sm_90a (nvcc cross-compiles without a GPU)."""
from __future__ import annotations

import atexit
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libdra_alloc.so")
SRC = [os.path.join(HERE, "csrc", "dra_api.cu"), os.path.join(HERE, "csrc", "dra_host.cpp")]
DEPS = SRC + [os.path.join(HERE, "csrc", "dra_device.cuh"), os.path.join(ROOT, "include", "dra_alloc.h"),
              os.path.join(ROOT, "include", "dra_driver.hpp")]
CPP_TEST_SRC = os.path.join(ROOT, "tests", "cpp", "driver_test.cpp")
CPP_TEST_EXE = os.path.join(ROOT, "tests", "cpp", "driver_test")


def nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def stale() -> bool:
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in DEPS)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not stale():
        return SO
    srcs = [s for s in SRC if os.path.exists(s)]
    cmd = [nvcc(), "-shared", "-Xcompiler", "-fPIC", "-std=c++17", "-O3", "-lineinfo",
           "-gencode", "arch=compute_90a,code=sm_90a",
           "-I", os.path.join(ROOT, "include"), "-o", SO] + srcs + ["-ldl"]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd))
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stdout + r.stderr)
    return SO


def build_cpp_tests(force: bool = False) -> str:
    """tests/cpp/driver_test: the C++ host layer's own test program, linked against libdra_alloc.so.  Linked in the tree
    when the tree is writable; a read-only tree whose program is missing or older than its source gets it linked into a
    temporary directory instead (removed at exit), and that path is returned."""
    build()
    if (not force and os.path.exists(CPP_TEST_EXE)
            and os.path.getmtime(CPP_TEST_EXE) >= max(os.path.getmtime(CPP_TEST_SRC), os.path.getmtime(SO))):
        return CPP_TEST_EXE
    exe = CPP_TEST_EXE
    if not os.access(os.path.dirname(CPP_TEST_EXE), os.W_OK):
        tmp = tempfile.mkdtemp(prefix="dra_driver_test_")
        atexit.register(shutil.rmtree, tmp, True)
        exe = os.path.join(tmp, "driver_test")
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), CPP_TEST_SRC, "-o", exe,
           "-L", HERE, "-ldra_alloc", "-Wl,-rpath," + HERE]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("g++ failed:\n" + r.stdout + r.stderr)
    return exe


def build_cpp_place_test(force: bool = False) -> str:
    """tests/cpp/place_test: the C++ host layer's test of Driver::PlaceBatch, linked like driver_test (in the tree when
    it is writable, else into a temporary directory removed at exit)."""
    build()
    src, exe = os.path.join(ROOT, "tests", "cpp", "place_test.cpp"), os.path.join(ROOT, "tests", "cpp", "place_test")
    if not force and os.path.exists(exe) and os.path.getmtime(exe) >= max(os.path.getmtime(src), os.path.getmtime(SO)):
        return exe
    if not os.access(os.path.dirname(exe), os.W_OK):
        tmp = tempfile.mkdtemp(prefix="dra_place_test_")
        atexit.register(shutil.rmtree, tmp, True)
        exe = os.path.join(tmp, "place_test")
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
           "-L", HERE, "-ldra_alloc", "-Wl,-rpath," + HERE]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("g++ failed:\n" + r.stdout + r.stderr)
    return exe


def build_cpp_capacity_test(force: bool = False) -> str:
    """tests/cpp/capacity_test: the C++ host layer's test of Driver::PodCapacityBatch, linked like driver_test (in the
    tree when it is writable, else into a temporary directory removed at exit)."""
    build()
    src, exe = os.path.join(ROOT, "tests", "cpp", "capacity_test.cpp"), os.path.join(ROOT, "tests", "cpp", "capacity_test")
    if not force and os.path.exists(exe) and os.path.getmtime(exe) >= max(os.path.getmtime(src), os.path.getmtime(SO)):
        return exe
    if not os.access(os.path.dirname(exe), os.W_OK):
        tmp = tempfile.mkdtemp(prefix="dra_capacity_test_")
        atexit.register(shutil.rmtree, tmp, True)
        exe = os.path.join(tmp, "capacity_test")
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
           "-L", HERE, "-ldra_alloc", "-Wl,-rpath," + HERE]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("g++ failed:\n" + r.stdout + r.stderr)
    return exe



def build_cpp_why_test(force: bool = False) -> str:
    """tests/cpp/why_test: the C++ host layer's test of Driver::UnsuitableReasonsBatch, linked like driver_test (in the
    tree when it is writable, else into a temporary directory removed at exit)."""
    build()
    src, exe = os.path.join(ROOT, "tests", "cpp", "why_test.cpp"), os.path.join(ROOT, "tests", "cpp", "why_test")
    if not force and os.path.exists(exe) and os.path.getmtime(exe) >= max(os.path.getmtime(src), os.path.getmtime(SO)):
        return exe
    if not os.access(os.path.dirname(exe), os.W_OK):
        tmp = tempfile.mkdtemp(prefix="dra_why_test_")
        atexit.register(shutil.rmtree, tmp, True)
        exe = os.path.join(tmp, "why_test")
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
           "-L", HERE, "-ldra_alloc", "-Wl,-rpath," + HERE]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("g++ failed:\n" + r.stdout + r.stderr)
    return exe


def build_cpp_place_why_test(force: bool = False) -> str:
    """tests/cpp/place_why_test: the C++ host layer's test of Driver::PlaceBatchWithReasons, linked like driver_test (in
    the tree when it is writable, else into a temporary directory removed at exit)."""
    build()
    src, exe = os.path.join(ROOT, "tests", "cpp", "place_why_test.cpp"), os.path.join(ROOT, "tests", "cpp", "place_why_test")
    if not force and os.path.exists(exe) and os.path.getmtime(exe) >= max(os.path.getmtime(src), os.path.getmtime(SO)):
        return exe
    if not os.access(os.path.dirname(exe), os.W_OK):
        tmp = tempfile.mkdtemp(prefix="dra_place_why_test_")
        atexit.register(shutil.rmtree, tmp, True)
        exe = os.path.join(tmp, "place_why_test")
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
           "-L", HERE, "-ldra_alloc", "-Wl,-rpath," + HERE]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("g++ failed:\n" + r.stdout + r.stderr)
    return exe


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
