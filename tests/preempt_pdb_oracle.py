"""ctypes wrapper of the CPU oracle of spec §14 with disruption budgets — TEST INFRASTRUCTURE ONLY.

tests/preempt_pdb_oracle.c (on tests/preempt_oracle.c, which it includes) counts each member's budget in the "members
of V up to and including v" form; it is compiled on first use into a cache file in the temporary directory, named by a
hash of its sources, so a read-only tree works too.  `preempt_naive_pdb` below is the independent restatement on top of
oracle/naive.py's `eval_pod`, written as kube-scheduler's decrement-then-below-zero loop: the two share no code, and the
CPU suite checks one against the other."""
from __future__ import annotations

import bisect
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
_SRCS = [os.path.join(_HERE, "preempt_pdb_oracle.c"), os.path.join(_HERE, "preempt_oracle.c"),
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
    so = os.path.join(tempfile.gettempdir(), f"dra_preempt_pdb_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
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
        _lib.preempt_oracle_preempt_pdb.argtypes = [vp, u32, vp, u32, vp, vp, u32, vp, vp, u32, vp, vp,
                                                    vp, u32, vp, vp, u32, vp, vp, u32, vp, vp, u32,
                                                    vp, vp, vp, vp, vp, vp, vp, vp, u32, u32]
        _lib.preempt_oracle_preempt_pdb.restype = C.c_int
        _lib.preempt_oracle_set_selectors.argtypes = [vp, u32, vp, u32]
        _lib.preempt_oracle_set_selectors.restype = None
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _nz(a, dtype):
    """an array that is never NULL (NULL means something else to the callee)"""
    a = np.ascontiguousarray(a if a is not None else [], dtype=dtype)
    return a if len(a) else np.zeros(1, dtype)


def preempt_pdb(gpus, node_off, table, claims, pod_off, prio, run_claims, run_pod_off, run_prio, run_out, run_pdb,
                pdb_allowed, run_out_off=None, cand_nodes=None, cand_off=None, max_victims: int = 8, flags: int = 0,
                n_pdb=None):
    """spec §14 with disruption budgets: run_pdb[r] (NONE: none; None: no array), pdb_allowed[b] (None: no array);
    n_pdb defaults to len(pdb_allowed).  Returns preempt()'s six outputs, then pair_violations and pod_violations."""
    g = np.ascontiguousarray(gpus, dtype=O.GPU_DTYPE)
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
    n_node = len(off) - 1
    n_pair = n_pod * n_node if co is None else int(co[-1])
    rc_ = _nz(run_claims, O.CLAIM_DTYPE)
    rpo = np.ascontiguousarray(run_pod_off, dtype=np.uint32)
    rpr = _nz(run_prio, np.int32)
    ro = _nz(run_out, O.OUT_DTYPE)
    n_rout = len(run_out) if run_out is not None else 0
    roo = None if run_out_off is None else _nz(run_out_off, np.uint32)
    pst = np.zeros(max(n_pair, 1), np.uint8)
    pvi = np.zeros(max(n_pair, 1), np.uint32)
    pnode = np.zeros(max(n_pod, 1), np.uint32)
    pstat = np.zeros(max(n_pod, 1), np.uint8)
    nvic = np.zeros(max(n_pod, 1), np.uint32)
    vic = np.zeros(max(n_pod * max_victims, 1), np.uint32)
    pvv = np.zeros(max(n_pair, 1), np.uint32)
    podv = np.zeros(max(n_pod, 1), np.uint32)
    rp = None if run_pdb is None else _nz(run_pdb, np.uint32)
    al = None if pdb_allowed is None else _nz(pdb_allowed, np.int32)
    n_pdb = (0 if pdb_allowed is None else len(pdb_allowed)) if n_pdb is None else n_pdb
    rc = lib().preempt_oracle_preempt_pdb(_p(g), len(g), _p(off), n_node, _p(t), _p(c), n_claim, _p(po), _p(pr), n_pod,
                                          _p(cn), _p(co), _p(rc_), len(run_claims) if run_claims is not None else 0,
                                          _p(rpo), _p(rpr), len(rpo) - 1, _p(roo), _p(ro), n_rout, _p(rp), _p(al), n_pdb,
                                          _p(pst), _p(pvi), _p(pvv), _p(pnode), _p(pstat), _p(nvic), _p(podv),
                                          _p(vic) if max_victims else None, max_victims, flags)
    if rc != 0:
        raise ValueError(f"preempt_oracle_preempt_pdb: rc={rc}")
    return (pst[:n_pair], pvi[:n_pair], pnode[:n_pod], pstat[:n_pod], nvic[:n_pod],
            vic[:n_pod * max_victims].reshape(n_pod, max_victims), pvv[:n_pair], podv[:n_pod])


_sel_keep = []


_sel_keep = []


def set_selectors(attrs=None, sels=None):
    """Selector context for the following calls of this oracle (spec §10); call with no arguments to clear."""
    _sel_keep.clear()
    if sels is None or len(sels) == 0:
        lib().preempt_oracle_set_selectors(None, 0, None, 0)
        return
    a = np.ascontiguousarray(attrs) if attrs is not None else np.zeros(0, dtype=np.uint8)
    s_ = np.ascontiguousarray(sels).reshape(-1, 8)
    _sel_keep.extend([a, s_])                          # the C side keeps the pointers
    lib().preempt_oracle_set_selectors(_p(a) if len(a) else None, len(a), _p(s_), len(s_))


def preempt_naive_pdb(gpus, node_off, table, claims, pod_off, prio, cands, exhaustive, run_claims, run_pod_off, run_prio,
                      run_out, run_pdb, pdb_allowed, run_out_off=None, max_victims: int = 8):
    """preempt_naive with disruption budgets, as kube-scheduler's filterPodsWithPDBViolation and SelectVictimsOnNode
    write them: run_pdb[r] the running pod's budget (NONE: none; None: no budgets), pdb_allowed[b] its
    disruptionsAllowed.  Returns the six outputs, then pair_violations and pod_violations, as lists."""
    from oracle import naive as N
    if len(pod_off) == 1:                                # no pending pods: the running pods are not examined
        return [], [], [], [], [], [], [], []
    n_node = len(node_off) - 1
    G0 = N._state(gpus)
    prio, run_prio = [int(x) for x in prio], [int(x) for x in run_prio]

    def node_of(g):
        return bisect.bisect_right(list(node_off), g) - 1

    # where each running pod is, and its OK slots as (gpu, kind, start, size, mem_limit)
    have_off = run_out_off is not None
    effects, where = [], []
    for r in range(len(run_pod_off) - 1):
        eff = []
        for i in range(run_pod_off[r], run_pod_off[r + 1]):
            c = run_claims[i]
            n = c["count"] if (c["kind"] == 0 and c["node"] < n_node and 1 <= c["count"] <= 32
                               and (have_off or c["count"] == 1)) else 1
            base = run_out_off[i] if have_off else i
            for rec in run_out[base: base + n]:
                if rec[4] == 0:
                    eff.append((rec[0], c["kind"], rec[1], rec[2], c["mem_limit_mib"]))
        nodes = {node_of(e[0]) for e in eff}
        assert len(nodes) <= 1
        effects.append(eff)
        where.append(nodes.pop() if nodes else None)

    def apply(W, g0, r, add):
        for gpu, kind, start, size, lim in effects[r]:
            if not g0 <= gpu < g0 + len(W):
                continue
            g = W[gpu - g0]
            if kind == 0:
                g["full"] = add
            elif kind == 1:
                cells = set(range(start, min(start + size, 16))) if start < 16 else set()
                g["used"] = (g["used"] | cells) if add else (g["used"] - cells)
            elif kind == 2:
                g["mem"] = (g["mem"] - lim if add else g["mem"] + lim) % (1 << 32)
                g["share"] = (g["share"] + (1 if add else -1)) % (1 << 16)

    def evaluate(W, g0, pod):
        """(placed, hit the search limit) on a private copy"""
        G = [None] * g0 + copy.deepcopy(W)
        placed, recs = N.eval_pod(G, g0, g0 + len(W), table, pod, n_node, exhaustive, True)
        return placed, any(r and r[0][4] == 7 for r in recs)

    def judge(p, n):
        """(status, victims in eviction order, violating victims)"""
        c0, c1 = pod_off[p], pod_off[p + 1]
        if n >= n_node:
            return NO, [], 0
        if c1 - c0 > 32:
            return INVALID, [], 0
        pod = [dict(c, node=n) for c in claims[c0:c1]]
        g0, g1 = node_off[n], node_off[n + 1]
        S = copy.deepcopy(G0[g0:g1])
        placed, lim = evaluate(S, g0, pod)
        if placed:
            return FITS, [], 0
        if any(N._invalid(c, n_node, True) for c in pod):
            return INVALID, [], 0
        V = sorted((r for r in range(len(where)) if where[r] == n and run_prio[r] < prio[p]),
                   key=lambda r: (-run_prio[r], r))
        for r in V:
            apply(S, g0, r, False)
        placed, lim = evaluate(S, g0, pod)
        if not placed:
            return (SEARCH_LIMIT if lim else NO), [], 0
        violating = set()                                # filterPodsWithPDBViolation, on a fresh copy of the budgets
        if run_pdb is not None:
            left = [int(x) for x in pdb_allowed]
            for r in V:
                b = int(run_pdb[r])
                if b != NONE:
                    left[b] -= 1
                    if left[b] < 0:
                        violating.add(r)
        gone = set()
        for phase in (True, False):                      # reprievePod over the violating pods, then the others
            for r in V:
                if (r in violating) != phase:
                    continue
                S2 = copy.deepcopy(S)
                apply(S2, g0, r, True)
                if evaluate(S2, g0, pod)[0]:
                    S = S2
                else:
                    gone.add(r)
        return EVICT, [r for r in V if r in gone], len(gone & violating)   # victims re-sorted by importance: V order

    pair_status, pair_victims, pod_node, pod_status, n_victims, rows = [], [], [], [], [], []
    pair_viol, pod_viol = [], []
    for p in range(len(pod_off) - 1):
        cl = list(range(n_node)) if cands is None else list(cands[p])
        judged = [judge(p, n) for n in cl]
        pair_status += [s for s, _, _ in judged]
        pair_victims += [len(v) if s == EVICT else 0 for s, v, _ in judged]
        viol = [x if s == EVICT else 0 for s, _, x in judged]
        pair_viol += viol
        fits = [k for k, (s, _, _) in enumerate(judged) if s == FITS]
        evict = [k for k, (s, _, _) in enumerate(judged) if s == EVICT]

        def key(k):
            v = judged[k][1]
            hi = max((run_prio[r] for r in v), default=-(1 << 31))
            last = min((r for r in v if run_prio[r] == hi), default=NONE)
            return (viol[k], hi, sum(run_prio[r] + (1 << 31) for r in v), len(v), -last, k)

        row = [NONE] * max_victims
        if fits:
            pod_node.append(cl[fits[0]]); pod_status.append(FITS); n_victims.append(0); pod_viol.append(0)
        elif evict:
            k = min(evict, key=key)
            v = judged[k][1]
            pod_node.append(cl[k]); pod_status.append(EVICT); n_victims.append(len(v)); pod_viol.append(viol[k])
            row[:min(len(v), max_victims)] = v[:max_victims]
        else:
            pod_viol.append(0)
            pod = claims[pod_off[p]:pod_off[p + 1]]
            inv = len(pod) > 32 or any(N._invalid(dict(c, node=0), 1, True) for c in pod)
            pod_node.append(NONE); n_victims.append(0)
            pod_status.append(INVALID if inv else SEARCH_LIMIT if any(s == SEARCH_LIMIT for s, _, _ in judged) else NO)
        rows.append(row)
    return pair_status, pair_victims, pod_node, pod_status, n_victims, rows, pair_viol, pod_viol
