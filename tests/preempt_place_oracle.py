"""ctypes wrapper of the CPU oracle of spec §15 (preempt and place) — TEST INFRASTRUCTURE ONLY.

pod_oracle_preempt_place (tests/pod_oracles.c, loaded by tests/pod_oracles.py) runs the sequential schedule on the §14
pair judgement without budgets and oracle/dra_oracle.c's pod evaluation.  `preempt_place_naive` below is the
independent restatement: the host loop itself, per pod preempt_oracle.preempt_naive with that one pod against the
running pods not evicted yet, §9 for its victims and oracle/naive.py's `eval_pod` on the chosen node.  The two share no
code, and the CPU suite checks one against the other."""
from __future__ import annotations

import numpy as np

from oracle import oracle as O
from pod_oracles import _nz, _p, lib, set_selectors  # noqa: F401  (set_selectors: the selectors of every pod oracle)

NONE = 0xFFFFFFFF
F_EXHAUSTIVE = O.F_EXHAUSTIVE
FITS, EVICT, NO, SEARCH_LIMIT, INVALID = 0, 1, 2, 3, 4


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
                  run_out_off=None, cand_nodes=None, cand_off=None, out_off=None, n_out=None, flags: int = 0,
                  fill: int | None = None):
    """spec §15.  cand_nodes/cand_off None = every pod against every node, ascending.  Returns (out, pod_node,
    pod_status, evicted_by, gpus_after).  Raises ValueError on the arguments §15 rejects.  Inputs are not modified.
    fill: every byte of the four outputs starts as `fill`, so what the call does not write (slots no claim owns, and
    evicted_by when there are no pending pods) keeps it; None: zeros, and evicted_by 0xFFFFFFFF."""
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
    def filled(n, dtype):
        return np.full(max(n, 1) * np.dtype(dtype).itemsize, fill, np.uint8).view(dtype)
    if fill is None:
        out = np.zeros(max(n_out, 1), O.OUT_DTYPE)
        pnode = np.zeros(max(n_pod, 1), np.uint32)
        pstat = np.zeros(max(n_pod, 1), np.uint8)
        ev = np.full(max(n_run, 1), NONE, np.uint32)
    else:
        out, pnode, pstat, ev = (filled(n_out, O.OUT_DTYPE), filled(n_pod, np.uint32), filled(n_pod, np.uint8),
                                 filled(n_run, np.uint32))
    rc = lib().pod_oracle_preempt_place(_p(g), len(g), _p(off), len(off) - 1, _p(t), _p(c), n_claim, _p(po), _p(pr),
                                        n_pod, _p(cn), _p(co), _p(rc_),
                                        len(run_claims) if run_claims is not None else 0, _p(rpo), _p(rpr), n_run,
                                        _p(roo), _p(ro), n_rout, _p(oo), _p(out), n_out, _p(pnode), _p(pstat), _p(ev),
                                        flags)
    if rc != 0:
        raise ValueError(f"pod_oracle_preempt_place: rc={rc}")
    return out[:n_out], pnode[:n_pod], pstat[:n_pod], ev[:n_run], g


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
        if len(pod) > N.MAX_POD or any(N._invalid(dict(c, node=0), 1, have_off) for c in pod):
            # invalid in the call's slot mode: not handed to §14, which judges as if out_off were given
            node, st = NONE, INVALID
        else:
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
            for v in rows[0][: nv[0]]:
                evicted_by[alive[v]] = p
                release(alive[v])
        pod_node.append(node)
        pod_status.append(st)
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
