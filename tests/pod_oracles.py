"""ctypes loader of the CPU oracles of the pod-level calls — TEST INFRASTRUCTURE ONLY.

tests/pod_oracles.c holds place pods (spec §13), preemption with optional disruption budgets (§14), preempt and place
(§15) and pod capacity (§16), all on the §12 evaluation of oracle/dra_oracle.c (which it includes once), with one
selector state for the four.  It is compiled on first use into a cache file in the temporary directory, named by a hash
of its sources, so a read-only tree works too.  place_oracle.py, preempt_oracle.py, preempt_place_oracle.py and
capacity_oracle.py each wrap one of its calls."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRCS = [os.path.join(_HERE, "pod_oracles.c"), os.path.join(_ROOT, "oracle", "dra_oracle.c"),
         os.path.join(_ROOT, "oracle", "dra_oracle.h"), os.path.join(_ROOT, "include", "dra_alloc.h")]

_vp, _u32 = C.c_void_p, C.c_uint32
_ARGTYPES = {
    "pod_oracle_set_selectors": [_vp, _u32, _vp, _u32],
    "pod_oracle_place_pods": [_vp, _u32, _vp, _u32, _vp, _vp, _u32, _vp, _u32, _vp, _vp, _vp, _vp, _u32, _vp, _u32],
    "pod_oracle_capacity": [_vp, _u32, _vp, _u32, _vp, _vp, _u32, _vp, _u32, _vp, _vp, _u32, _vp, _vp, _vp, _vp, _u32],
    "pod_oracle_preempt": [_vp, _u32, _vp, _u32, _vp, _vp, _u32, _vp, _vp, _u32, _vp, _vp,
                           _vp, _u32, _vp, _vp, _u32, _vp, _vp, _u32, _vp, _vp, _u32,
                           _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _u32, _u32],
    "pod_oracle_preempt_place": [_vp, _u32, _vp, _u32, _vp, _vp, _u32, _vp, _vp, _u32, _vp, _vp,
                                 _vp, _u32, _vp, _vp, _u32, _vp, _vp, _u32,
                                 _vp, _vp, _u32, _vp, _vp, _vp, _u32],
}

_lib = None


def build() -> str:
    h = hashlib.sha256()
    for s in _SRCS:
        with open(s, "rb") as f:
            h.update(f.read())
    so = os.path.join(tempfile.gettempdir(), f"dra_pod_oracles_{os.getuid()}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.run([os.environ.get("CC", "gcc"), "-O2", "-std=c11", "-Wall", "-fPIC", "-pthread", "-shared",
                        "-fvisibility=hidden", "-o", tmp, _SRCS[0]], check=True)
        os.replace(tmp, so)
    return so


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        for name, argtypes in _ARGTYPES.items():
            f = getattr(_lib, name)
            f.argtypes = argtypes
            f.restype = None if name == "pod_oracle_set_selectors" else C.c_int
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _nz(a, dtype):
    """an array that is never NULL (NULL means something else to the callee)"""
    a = np.ascontiguousarray(a if a is not None else [], dtype=dtype)
    return a if len(a) else np.zeros(1, dtype)


_sel_keep = []


def set_selectors(attrs=None, sels=None):
    """Selector context for the following calls of all four oracles (spec §10); call with no arguments to clear."""
    _sel_keep.clear()
    if sels is None or len(sels) == 0:
        lib().pod_oracle_set_selectors(None, 0, None, 0)
        return
    a = np.ascontiguousarray(attrs) if attrs is not None else np.zeros(0, dtype=np.uint8)
    s_ = np.ascontiguousarray(sels).reshape(-1, 8)
    _sel_keep.extend([a, s_])                          # the C side keeps the pointers
    lib().pod_oracle_set_selectors(_p(a) if len(a) else None, len(a), _p(s_), len(s_))
