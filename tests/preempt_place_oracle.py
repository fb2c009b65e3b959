"""ctypes wrapper of the CPU oracle of spec §15 (preempt and place) — TEST INFRASTRUCTURE ONLY.

tests/preempt_place_oracle.c runs the sequential schedule on tests/preempt_oracle.c's pair judgement and oracle/dra_oracle.c's
pod evaluation (which it includes); it is compiled on first use into a cache file in the temporary directory, named by
a hash of its sources, so a read-only tree works too.  `preempt_place_naive` below is the independent restatement: the
host loop itself, per pod preempt_oracle.preempt_naive with that one pod against the running pods not evicted yet, §9 for
its victims and oracle/naive.py's `eval_pod` on the chosen node.  The two share no code, and the CPU suite checks one
against the other."""
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
_SRCS = [os.path.join(_HERE, "preempt_place_oracle.c"), os.path.join(_HERE, "preempt_oracle.c"),
         os.path.join(_ROOT, "oracle", "dra_oracle.c"), os.path.join(_ROOT, "oracle", "dra_oracle.h"),
         os.path.join(_ROOT, "include", "dra_alloc.h")]
NONE = 0xFFFFFFFF
F_EXHAUSTIVE = O.F_EXHAUSTIVE
FITS, EVICT, NO, SEARCH_LIMIT, INVALID = 0, 1, 2, 3, 4

_lib = None


def build() -> str:
    h = hashlib.sha256()
    for s in _SRCS:
        with open(s, "rb") as f:
            h.update(f.read())
    so = os.path.join(tempfile.gettempdir(), f"dra_preempt_place_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
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
        _lib.pp_oracle_preempt_place.argtypes = [vp, u32, vp, u32, vp, vp, u32, vp, vp, u32, vp, vp,
                                                 vp, u32, vp, vp, u32, vp, vp, u32,
                                                 vp, vp, u32, vp, vp, vp, u32]
        _lib.pp_oracle_preempt_place.restype = C.c_int
        _lib.pp_oracle_set_selectors.argtypes = [vp, u32, vp, u32]
        _lib.pp_oracle_set_selectors.restype = None
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _nz(a, dtype):
    """an array that is never NULL (NULL means something else to the callee)"""
    a = np.ascontiguousarray(a if a is not None else [], dtype=dtype)
    return a if len(a) else np.zeros(1, dtype)


def pending_slots(claims, out_off=None):
    """n_out of the pending claims: slots as if each claim named a node of the inventory"""
    if out_off is None:
        return len(claims)
    placed = np.array(claims, dtype=O.CLAIM_DTYPE, copy=True)
    placed["node"] = 0
    ok = (placed["kind"] == 0) & (placed["count"] >= 1) & (placed["count"] <= 32)
    sl = np.where(ok, placed["count"], 1).astype(np.int64)
    return int(max((int(b) + int(s) for b, s in zip(out_off, sl)), default=0))


def preempt_place(gpus, node_off, table, claims, pod_off, prio, run_claims, run_pod_off, run_prio, run_out,
                  run_out_off=None, cand_nodes=None, cand_off=None, out_off=None, n_out=None, flags: int = 0):
    """spec §15.  cand_nodes/cand_off None = every pod against every node, ascending.  Returns (out, pod_node,
    pod_status, evicted_by, gpus_after).  Raises ValueError on the arguments §15 rejects.  Inputs are not modified."""
    g = np.ascontiguousarray(gpus, dtype=O.GPU_DTYPE).copy()
    off = np.ascontiguousarray(node_off, dtype=np.uint32)
    t = np.ascontiguousarray(table)
    c = _nz(claims, O.CLAIM_DTYPE)
    n_claim = len(claims) if claims is not None else 0
    po = np.ascontiguousarray(pod_off, dtype=np.uint32)
    pr = _nz(prio, np.int32)
    n_pod = len(po) - 1
    cn = co = None
    if cand_nodes is not None or cand_off is not None:
        co = np.ascontiguousarray(cand_off, dtype=np.uint32)
        cn = _nz(cand_nodes, np.uint32)
    oo = None if out_off is None else _nz(out_off, np.uint32)
    if n_out is None:
        n_out = pending_slots(claims, out_off) if n_claim else 0
    rc_ = _nz(run_claims, O.CLAIM_DTYPE)
    rpo = np.ascontiguousarray(run_pod_off, dtype=np.uint32)
    rpr = _nz(run_prio, np.int32)
    ro = _nz(run_out, O.OUT_DTYPE)
    n_rout = len(run_out) if run_out is not None else 0
    roo = None if run_out_off is None else _nz(run_out_off, np.uint32)
    n_run = len(rpo) - 1
    out = np.zeros(max(n_out, 1), O.OUT_DTYPE)
    pnode = np.zeros(max(n_pod, 1), np.uint32)
    pstat = np.zeros(max(n_pod, 1), np.uint8)
    ev = np.full(max(n_run, 1), NONE, np.uint32)
    rc = lib().pp_oracle_preempt_place(_p(g), len(g), _p(off), len(off) - 1, _p(t), _p(c), n_claim, _p(po), _p(pr), n_pod,
                                       _p(cn), _p(co), _p(rc_), len(run_claims) if run_claims is not None else 0, _p(rpo),
                                       _p(rpr), n_run, _p(roo), _p(ro), n_rout, _p(oo), _p(out), n_out, _p(pnode),
                                       _p(pstat), _p(ev), flags)
    if rc != 0:
        raise ValueError(f"pp_oracle_preempt_place: rc={rc}")
    return out[:n_out], pnode[:n_pod], pstat[:n_pod], ev[:n_run], g


_sel_keep = []


def set_selectors(attrs=None, sels=None):
    """Selector context for the following calls (spec §10); call with no arguments to clear."""
    _sel_keep.clear()
    if sels is None or len(sels) == 0:
        lib().pp_oracle_set_selectors(None, 0, None, 0)
        return
    a = np.ascontiguousarray(attrs) if attrs is not None else np.zeros(0, dtype=np.uint8)
    s_ = np.ascontiguousarray(sels).reshape(-1, 8)
    _sel_keep.extend([a, s_])                          # the C side keeps the pointers
    lib().pp_oracle_set_selectors(_p(a) if len(a) else None, len(a), _p(s_), len(s_))


def preempt_place_naive(gpus, node_off, table, claims, pod_off, prio, cands, exhaustive, run_claims, run_pod_off,
                        run_prio, run_out, out_off=None):
    """spec §15 as the host loop, on the naive restatements (small cases, no selectors, running pods without out_off).
    gpus / claims / run_claims: lists of dicts as naive.py takes them; run_out: list of (gpu, start, size, profile,
    status); cands: one list of node indices per pod, or None for every node ascending.  Returns (out list, pod_node,
    pod_status, evicted_by, gpus_after)."""
    from oracle import naive as N
    from preempt_oracle import preempt_naive
    n_node = len(node_off) - 1
    have_off = out_off is not None
    G = N._state(gpus)
    base = list(out_off) if have_off else list(range(len(claims)))
    sl = [N._slots(dict(c, node=0), 1, have_off) for c in claims]
    n_out = max([b + s for b, s in zip(base, sl)], default=0)
    out = [None] * n_out
    n_run = len(run_pod_off) - 1
    evicted_by = [NONE] * n_run
    pod_node, pod_status = [], []

    def release(r):                                   # §9 on the state dicts
        for i in range(run_pod_off[r], run_pod_off[r + 1]):
            c, (gpu, start, size, _, st) = run_claims[i], run_out[i]
            if st != 0:
                continue
            g = G[gpu]
            if c["kind"] == 0:
                g["full"] = False
            elif c["kind"] == 1:
                g["used"] -= set(range(start, min(start + size, 16))) if start < 16 else set()
            elif c["kind"] == 2:
                g["mem"] = (g["mem"] + c["mem_limit_mib"]) % (1 << 32)
                g["share"] = (g["share"] - 1) % (1 << 16)

    for p in range(len(pod_off) - 1):
        c0, c1 = pod_off[p], pod_off[p + 1]
        pod = claims[c0:c1]
        alive = [r for r in range(n_run) if evicted_by[r] == NONE]
        idx = [i for r in alive for i in range(run_pod_off[r], run_pod_off[r + 1])]
        rpo = [0]
        for r in alive:
            rpo.append(rpo[-1] + run_pod_off[r + 1] - run_pod_off[r])
        _, _, node, st, nv, rows = preempt_naive(
            N._dump(gpus, G), node_off, table, pod, [0, len(pod)], [prio[p]], None if cands is None else [cands[p]],
            exhaustive, [run_claims[i] for i in idx], rpo, [run_prio[r] for r in alive], [run_out[i] for i in idx],
            None, max(len(alive), 1))
        node, st = node[0], st[0]
        pod_node.append(node)
        pod_status.append(st)
        for v in rows[0][: nv[0]]:
            evicted_by[alive[v]] = p
            release(alive[v])
        if node != NONE:
            if pod:
                _, recs = N.eval_pod(G, node_off[node], node_off[node + 1], table, [dict(c, node=node) for c in pod],
                                     n_node, exhaustive, have_off)
                for i, r in zip(range(c0, c1), recs):
                    out[base[i]: base[i] + len(r)] = r
            continue
        for i in range(c0, c1):
            bad = len(pod) > N.MAX_POD or N._invalid(dict(claims[i], node=0), 1, have_off)
            out[base[i]: base[i] + sl[i]] = [(NONE, 0, 0, N._oprof(claims[i]),
                                              5 if bad else 7 if st == SEARCH_LIMIT else 6)] * sl[i]
    return out, pod_node, pod_status, evicted_by, N._dump(gpus, G)
