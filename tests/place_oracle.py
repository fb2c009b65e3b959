"""ctypes wrapper of the CPU oracle of spec §13 (place pods) — TEST INFRASTRUCTURE ONLY.

tests/place_oracle.c walks the candidates of each pod and evaluates the pod with the §12 evaluation of
oracle/dra_oracle.c (which it includes); it is compiled on first use into a cache file in the temporary directory,
named by a hash of its sources, so a read-only tree works too.  `place_pods_naive` below is the independent restatement
on top of oracle/naive.py's `eval_pod`: the two share no code, and the CPU suite checks one against the other."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRCS = [os.path.join(_HERE, "place_oracle.c"), os.path.join(_ROOT, "oracle", "dra_oracle.c"),
         os.path.join(_ROOT, "oracle", "dra_oracle.h"), os.path.join(_ROOT, "include", "dra_alloc.h")]
NONE = 0xFFFFFFFF
F_EXHAUSTIVE = O.F_EXHAUSTIVE

_lib = None


def build() -> str:
    h = hashlib.sha256()
    for s in _SRCS:
        with open(s, "rb") as f:
            h.update(f.read())
    so = os.path.join(tempfile.gettempdir(), f"dra_place_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
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
        _lib.place_oracle_place_pods.argtypes = [vp, u32, vp, u32, vp, vp, u32, vp, u32, vp, vp, vp, vp, u32, vp, u32]
        _lib.place_oracle_place_pods.restype = C.c_int
        _lib.place_oracle_set_selectors.argtypes = [vp, u32, vp, u32]
        _lib.place_oracle_set_selectors.restype = None
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def place_pods(gpus, node_off, table, claims, pod_off, cand_nodes=None, cand_off=None, out_off=None, n_out=None,
               flags: int = 0):
    """spec §13 (choose the node, then allocate).  cand_nodes/cand_off None = every pod against every node, ascending.
    Returns (out, pod_node, gpus_after).  Inputs are not modified."""
    g = np.ascontiguousarray(gpus, dtype=O.GPU_DTYPE).copy()
    off = np.ascontiguousarray(node_off, dtype=np.uint32)
    t = np.ascontiguousarray(table)
    c = np.ascontiguousarray(claims, dtype=O.CLAIM_DTYPE)
    po = np.ascontiguousarray(pod_off, dtype=np.uint32)
    cn = None if cand_nodes is None else np.ascontiguousarray(cand_nodes, dtype=np.uint32)
    co = None if cand_off is None else np.ascontiguousarray(cand_off, dtype=np.uint32)
    if co is not None and (cn is None or len(cn) == 0):
        cn = np.zeros(1, np.uint32)                   # an empty list still needs an address (NULL means the dense form)
    oo = None if out_off is None else np.ascontiguousarray(out_off, dtype=np.uint32)
    if n_out is None:
        n_out = len(c) if oo is None else 0
    out = np.zeros(max(n_out, 1), dtype=O.OUT_DTYPE)
    pod_node = np.zeros(max(len(po) - 1, 1), dtype=np.uint32)
    rc = lib().place_oracle_place_pods(_p(g), len(g), _p(off), len(off) - 1, _p(t), _p(c), len(c), _p(po), len(po) - 1,
                                       _p(cn), _p(co), _p(oo), _p(out), n_out, _p(pod_node), flags)
    if rc != 0:
        raise ValueError(f"place_oracle_place_pods: rc={rc}")
    return out[:n_out], pod_node[:len(po) - 1], g


_sel_keep = []


def set_selectors(attrs=None, sels=None):
    """Selector context for the following calls (spec §10); call with no arguments to clear."""
    _sel_keep.clear()
    if sels is None or len(sels) == 0:
        lib().place_oracle_set_selectors(None, 0, None, 0)
        return
    a = np.ascontiguousarray(attrs) if attrs is not None else np.zeros(0, dtype=np.uint8)
    s_ = np.ascontiguousarray(sels).reshape(-1, 8)
    _sel_keep.extend([a, s_])                          # the C side keeps the pointers
    lib().place_oracle_set_selectors(_p(a) if len(a) else None, len(a), _p(s_), len(s_))


def place_pods_naive(gpus, node_off, table, claims, pod_off, cands, exhaustive, out_off=None):
    """spec §13 restated on oracle/naive.py's pod evaluation (small cases only).  gpus / claims: lists of dicts as
    naive.py takes them; cands: one list of node indices per pod, or None for every node ascending.
    Returns (out list, pod_node list, gpus_after)."""
    from oracle import naive as N
    n_node = len(node_off) - 1
    have_off = out_off is not None
    G = N._state(gpus)

    def as_placed(c):                                 # slots and validity as if the claim named a node of the inventory
        return dict(c, node=0)

    sl = [N._slots(as_placed(c), 1, have_off) for c in claims]
    base = list(out_off) if have_off else list(range(len(claims)))
    n_out = max([b + s for b, s in zip(base, sl)], default=0)
    out = [None] * n_out
    pod_node = []
    for p in range(len(pod_off) - 1):
        c0, c1 = pod_off[p], pod_off[p + 1]
        pod = claims[c0:c1]
        pod_node.append(NONE)
        if not pod:
            continue
        if len(pod) > N.MAX_POD:
            for i in range(c0, c1):
                out[base[i]: base[i] + sl[i]] = [(NONE, 0, 0, N._oprof(claims[i]), 5)] * sl[i]
            continue
        hit_limit = False
        for node in (range(n_node) if cands is None else cands[p]):
            if node >= n_node:
                continue
            placed, recs = N.eval_pod(G, node_off[node], node_off[node + 1], table, [dict(c, node=node) for c in pod],
                                      n_node, exhaustive, have_off)
            if placed:
                for i, r in zip(range(c0, c1), recs):
                    out[base[i]: base[i] + len(r)] = r
                pod_node[p] = node
                break
            hit_limit = hit_limit or any(r[0][4] == 7 for r in recs)
        if pod_node[p] == NONE:
            for i in range(c0, c1):
                st_ = 5 if N._invalid(as_placed(claims[i]), 1, have_off) else 7 if hit_limit else 6
                out[base[i]: base[i] + sl[i]] = [(NONE, 0, 0, N._oprof(claims[i]), st_)] * sl[i]
    return out, pod_node, N._dump(gpus, G)
