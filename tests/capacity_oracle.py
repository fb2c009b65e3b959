"""ctypes wrapper of the CPU oracle of spec §16 (pod capacity) — TEST INFRASTRUCTURE ONLY.

tests/capacity_oracle.c counts the copies of each pod a candidate node takes with the §12 evaluation of
oracle/dra_oracle.c (which it includes); it is compiled on first use into a cache file in the temporary directory, named
by a hash of its sources, so a read-only tree works too.  `capacity_naive` below is the independent restatement on top of
oracle/naive.py's `eval_pod`: the two share no code, and the CPU suite checks one against the other."""
from __future__ import annotations

import copy
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRCS = [os.path.join(_HERE, "capacity_oracle.c"), os.path.join(_ROOT, "oracle", "dra_oracle.c"),
         os.path.join(_ROOT, "oracle", "dra_oracle.h"), os.path.join(_ROOT, "include", "dra_alloc.h")]
F_EXHAUSTIVE = O.F_EXHAUSTIVE
ST_OK, ST_INVALID, ST_POD, ST_SEARCH_LIMIT = 0, 5, 6, 7

_lib = None


def build() -> str:
    h = hashlib.sha256()
    for s in _SRCS:
        with open(s, "rb") as f:
            h.update(f.read())
    so = os.path.join(tempfile.gettempdir(), f"dra_capacity_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
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
        vp, u32 = C.c_void_p, C.c_uint32
        _lib.capacity_oracle_capacity.argtypes = [vp, u32, vp, u32, vp, vp, u32, vp, u32, vp, vp, u32, vp, vp, vp, vp, u32]
        _lib.capacity_oracle_capacity.restype = C.c_int
        _lib.capacity_oracle_set_selectors.argtypes = [vp, u32, vp, u32]
        _lib.capacity_oracle_set_selectors.restype = None
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _nz(a, dtype):
    """an array that is never NULL (NULL means something else to the callee)"""
    a = np.ascontiguousarray(a if a is not None else [], dtype=dtype)
    return a if len(a) else np.zeros(1, dtype)


def capacity(gpus, node_off, table, claims, pod_off, cand_nodes=None, cand_off=None, max_copies: int = 64, flags: int = 0):
    """spec §16.  cand_nodes/cand_off None = every pod against every node (pair = pod * n_node + node).  Returns
    (pair_copies u16, pair_stop u8, pod_total u64, pod_nodes u32).  Raises ValueError on the arguments §16 rejects.
    Inputs are not modified."""
    g = np.ascontiguousarray(gpus, dtype=O.GPU_DTYPE)
    off = np.ascontiguousarray(node_off, dtype=np.uint32)
    t = np.ascontiguousarray(table)
    c = _nz(claims, O.CLAIM_DTYPE)
    n_claim = len(claims) if claims is not None else 0
    po = np.ascontiguousarray(pod_off, dtype=np.uint32)
    n_pod, n_node = len(po) - 1, len(off) - 1
    cn = co = None
    if cand_nodes is not None or cand_off is not None:
        co = np.ascontiguousarray(cand_off, dtype=np.uint32)
        cn = _nz(cand_nodes, np.uint32)
    n_pair = n_pod * n_node if co is None else int(co[-1])
    copies = np.zeros(max(n_pair, 1), np.uint16)
    stop = np.zeros(max(n_pair, 1), np.uint8)
    total = np.zeros(max(n_pod, 1), np.uint64)
    nodes = np.zeros(max(n_pod, 1), np.uint32)
    rc = lib().capacity_oracle_capacity(_p(g), len(g), _p(off), n_node, _p(t), _p(c), n_claim, _p(po), n_pod, _p(cn), _p(co),
                                        max_copies, _p(copies), _p(stop), _p(total), _p(nodes), flags)
    if rc != 0:
        raise ValueError(f"capacity_oracle_capacity: rc={rc}")
    return copies[:n_pair], stop[:n_pair], total[:n_pod], nodes[:n_pod]


_sel_keep = []


def set_selectors(attrs=None, sels=None):
    """Selector context for the following calls (spec §10); call with no arguments to clear."""
    _sel_keep.clear()
    if sels is None or len(sels) == 0:
        lib().capacity_oracle_set_selectors(None, 0, None, 0)
        return
    a = np.ascontiguousarray(attrs) if attrs is not None else np.zeros(0, dtype=np.uint8)
    s_ = np.ascontiguousarray(sels).reshape(-1, 8)
    _sel_keep.extend([a, s_])                          # the C side keeps the pointers
    lib().capacity_oracle_set_selectors(_p(a) if len(a) else None, len(a), _p(s_), len(s_))


def capacity_naive(gpus, node_off, table, claims, pod_off, cands, exhaustive, max_copies: int = 64):
    """spec §16 restated on oracle/naive.py's pod evaluation (small cases, no selectors).  gpus / claims: lists of dicts
    as naive.py takes them; cands: one list of node indices per pod, or None for every node ascending.  Returns the four
    outputs as lists."""
    from oracle import naive as N
    n_node = len(node_off) - 1
    G0 = N._state(gpus)
    pair_copies, pair_stop, pod_total, pod_nodes = [], [], [], []
    for p in range(len(pod_off) - 1):
        mine = []
        for n in (range(n_node) if cands is None else cands[p]):
            pod = [dict(c, node=n) for c in claims[pod_off[p]:pod_off[p + 1]]]
            if n >= n_node:
                mine.append((0, ST_POD))
            elif not pod:
                mine.append((max_copies, ST_OK))
            elif len(pod) > 32 or any(N._invalid(c, n_node, True) for c in pod):
                mine.append((0, ST_INVALID))
            else:
                g0, g1 = node_off[n], node_off[n + 1]
                G = [None] * g0 + copy.deepcopy(G0[g0:g1])
                copies, stop = 0, ST_OK
                while copies < max_copies:
                    placed, recs = N.eval_pod(G, g0, g1, table, pod, n_node, exhaustive, True)
                    if not placed:
                        stop = ST_SEARCH_LIMIT if recs[0][0][4] == ST_SEARCH_LIMIT else ST_POD
                        break
                    copies += 1
                mine.append((copies, stop))
        pair_copies += [c for c, _ in mine]
        pair_stop += [s for _, s in mine]
        pod_total.append(sum(c for c, _ in mine))
        pod_nodes.append(sum(1 for c, _ in mine if c))
    return pair_copies, pair_stop, pod_total, pod_nodes
