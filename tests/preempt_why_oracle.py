"""Spec §19 (why preemption judged each node as it did) restated in Python — TEST INFRASTRUCTURE ONLY.

`preempt_why` takes each pair's status from the C oracle of §14 (preempt_oracle.preempt), builds S' with §9's arithmetic on
the node's records, and answers with place_why_oracle.pair_reason on S or S'.  `preempt_place_why` reaches §15's W_p by
running the C oracle of §15 (preempt_place_oracle.preempt_place) on the pods before p, then answers pod p as
`preempt_why` does, against W_p and the running pods not evicted yet.  `preempt_why_naive` and `preempt_place_why_naive`
state the same thing a second time on preempt_naive / preempt_place_naive and naive_pod_reason (oracle/naive.py, no
selectors), sharing no code with the first; the CPU suite checks that the two agree."""
from __future__ import annotations

import bisect
import copy

import numpy as np

import place_why_oracle as PW
import preempt_oracle as P
import preempt_place_oracle as PP
import why_oracle as Y
from oracle import oracle as O

NONE = 0xFFFFFFFF
FITS, EVICT, NO, SEARCH_LIMIT, INVALID = P.FITS, P.EVICT, P.NO, P.SEARCH_LIMIT, P.INVALID


def _cand_lists(n_pod, n_node, cand_nodes, cand_off):
    if cand_off is None:
        return [list(range(n_node)) for _ in range(n_pod)]
    return [[int(x) for x in cand_nodes[cand_off[p]:cand_off[p + 1]]] for p in range(n_pod)]


def _run_effects(gpus, node_off, run_claims, run_pod_off, run_out, run_out_off):
    """per running pod: (node or None, its OK slots as (gpu, kind, start, size, mem_limit)), slots counted as §9 counts
    them (the call-level faults are the C oracle's to find)"""
    n_node = len(node_off) - 1
    have_off = run_out_off is not None
    res = []
    for r in range(len(run_pod_off) - 1):
        eff, nodes = [], set()
        for i in range(int(run_pod_off[r]), int(run_pod_off[r + 1])):
            c = run_claims[i]
            n = int(c["count"]) if (c["kind"] == Y.KIND_GPU and c["node"] < n_node and 1 <= c["count"] <= Y.MAX_COUNT
                                    and (have_off or c["count"] == 1)) else 1
            base = int(run_out_off[i]) if have_off else i
            for o in run_out[base:base + n]:
                if o["status"] == Y.ST_OK:
                    eff.append((int(o["gpu"]), int(c["kind"]), int(o["start"]), int(o["size"]), int(c["mem_limit_mib"])))
                    nodes.add(int(gpus[int(o["gpu"])]["node"]))
        res.append((nodes.pop() if nodes else None, eff))
    return res


def _release(g, eff):
    """§9 for one running pod's OK slots on the records g, in their u16 / u32 arithmetic"""
    for gpu, kind, start, size, lim in eff:
        x = g[gpu]
        if kind == Y.KIND_GPU:
            x["flags"] = int(x["flags"]) & ~Y._FULL & 0xFF
        elif kind == Y.KIND_MIG:
            m = (((1 << size) - 1) << start) & 0xFFFF if start < 16 else 0
            x["busy"] = int(x["busy"]) & ~m & 0xFFFF
        elif kind == Y.KIND_SHARED:
            x["mem_free_mib"] = (int(x["mem_free_mib"]) + lim) & 0xFFFFFFFF
            x["share_cnt"] = (int(x["share_cnt"]) - 1) & 0xFFFF


def _pod_pairs(g, node_off, table, claims, c0, c1, prio_p, nodes, statuses, effects, run_prio, alive, backtrack,
               attrs, sels):
    """pod (claims c0..c1, priority prio_p) at its candidates `nodes` with their §14 statuses on the records g: (reason,
    blocking claim) per pair"""
    n_node = len(node_off) - 1
    out = []
    for n, st in zip(nodes, statuses):
        if n >= n_node:
            out.append((Y.WHY_NO_NODE, Y.WHY_CLAIM_NONE))
            continue
        S = g
        V = [r for r in alive if effects[r][0] == n and int(run_prio[r]) < prio_p]
        if st in (NO, SEARCH_LIMIT) and V:
            S = g.copy()
            for r in V:
                _release(S, effects[r][1])
        out.append(PW.pair_reason(S, node_off, table, claims, c0, c1, n, attrs, sels, backtrack, True))
    return out


def _tally(n_pod, n_claim, pair_pods, reasons, blocking):
    pod_why = np.zeros((n_pod, Y.WHY_N), np.uint32)
    blocks = np.zeros(n_claim, np.uint32)
    for p, r, c in zip(pair_pods, reasons, blocking):
        pod_why[p, r] += 1
        if c != Y.WHY_CLAIM_NONE:
            blocks[c] += 1
    return pod_why, blocks


def preempt_why(gpus, node_off, table, claims, pod_off, prio, run_claims, run_pod_off, run_prio, run_out, run_out_off=None,
                cand_nodes=None, cand_off=None, flags: int = 0, attrs=None, sels=None):
    """spec §19, the §14 form.  The selectors must also be set in the C oracle (`set_selectors`).  Returns (pair_status u8,
    pair_why u8, pair_claim u32, pod_why u32 [n_pod, WHY_N], claim_blocks u32 [n_claim]).  Raises ValueError on the
    arguments §14 rejects."""
    g = np.ascontiguousarray(gpus, dtype=O.GPU_DTYPE)
    claims = np.ascontiguousarray(claims, dtype=O.CLAIM_DTYPE) if claims is not None and len(claims) else \
        np.zeros(0, O.CLAIM_DTYPE)
    st = P.preempt(g, node_off, table, claims, pod_off, prio, run_claims, run_pod_off, run_prio, run_out, run_out_off,
                   cand_nodes, cand_off, 0, flags)[0]
    n_node, n_pod = len(node_off) - 1, len(pod_off) - 1
    if not n_pod:                                      # the running pods are not examined
        return (np.asarray(st, np.uint8), np.zeros(0, np.uint8), np.zeros(0, np.uint32), np.zeros((0, Y.WHY_N), np.uint32),
                np.zeros(len(claims), np.uint32))
    effects = _run_effects(g, node_off, run_claims, run_pod_off, run_out, run_out_off)
    alive = list(range(len(run_pod_off) - 1))
    lists = _cand_lists(n_pod, n_node, cand_nodes, cand_off)
    reasons, blocking, pair_pods, k = [], [], [], 0
    for p in range(n_pod):
        nodes = lists[p]
        for r, c in _pod_pairs(g, node_off, table, claims, int(pod_off[p]), int(pod_off[p + 1]), int(prio[p]), nodes,
                               [int(x) for x in st[k:k + len(nodes)]], effects, run_prio, alive,
                               bool(flags & Y.F_EXHAUSTIVE), attrs, sels):
            reasons.append(r); blocking.append(c); pair_pods.append(p)
        k += len(nodes)
    pod_why, blocks = _tally(n_pod, len(claims), pair_pods, reasons, blocking)
    return (np.asarray(st, np.uint8), np.array(reasons, np.uint8), np.array(blocking, np.uint32), pod_why, blocks)


def preempt_place_why(gpus, node_off, table, claims, pod_off, prio, run_claims, run_pod_off, run_prio, run_out,
                      run_out_off=None, cand_nodes=None, cand_off=None, out_off=None, n_out=None, flags: int = 0,
                      attrs=None, sels=None):
    """spec §19, the §15 form.  Returns preempt_place_oracle.preempt_place's (out, pod_node, pod_status, evicted_by,
    gpus_after), then (pair_status, pair_why, pair_claim, pod_why, claim_blocks) as preempt_why.  Raises ValueError on the
    arguments §15 rejects."""
    g0 = np.ascontiguousarray(gpus, dtype=O.GPU_DTYPE)
    claims = np.ascontiguousarray(claims, dtype=O.CLAIM_DTYPE) if claims is not None and len(claims) else \
        np.zeros(0, O.CLAIM_DTYPE)
    whole = PP.preempt_place(g0, node_off, table, claims, pod_off, prio, run_claims, run_pod_off, run_prio, run_out,
                             run_out_off, cand_nodes, cand_off, out_off, n_out, flags)
    n_node, n_pod, n_run = len(node_off) - 1, len(pod_off) - 1, len(run_pod_off) - 1
    have_off = out_off is not None
    effects = _run_effects(g0, node_off, run_claims, run_pod_off, run_out, run_out_off) if n_pod else []
    lists = _cand_lists(n_pod, n_node, cand_nodes, cand_off)
    backtrack = bool(flags & Y.F_EXHAUSTIVE)
    statuses, reasons, blocking, pair_pods = [], [], [], []
    for p in range(n_pod):
        c0, c1 = int(pod_off[p]), int(pod_off[p + 1])
        nodes = lists[p]
        # W_p: §15 on the pods before p (their slots stay inside n_out)
        if p:
            pre = PP.preempt_place(g0, node_off, table, claims[:c0], pod_off[:p + 1], prio[:p], run_claims, run_pod_off,
                                   run_prio, run_out, run_out_off,
                                   None if cand_off is None else cand_nodes[:cand_off[p]],
                                   None if cand_off is None else cand_off[:p + 1],
                                   None if out_off is None else out_off[:c0], whole[0].shape[0] if have_off else c0, flags)
            W, ev = pre[4], pre[3]
        else:
            W, ev = g0.copy(), np.full(n_run, NONE, np.uint32)
        alive = [r for r in range(n_run) if ev[r] == NONE]
        pod = claims[c0:c1]
        # never judged: invalid in the call's slot mode, or empty
        if c1 - c0 > Y.MAX_POD:
            bad = True
        elif c1 == c0 or not n_node:
            bad = False
        else:                                          # validity does not depend on the node
            bad = PW.pair_reason(W, node_off, table, claims, c0, c1, 0, attrs, sels, False, have_off)[0] == Y.ST_INVALID
        if bad or c1 == c0:
            for n in nodes:
                if n >= n_node:
                    statuses.append(NO); reasons.append(Y.WHY_NO_NODE); blocking.append(Y.WHY_CLAIM_NONE)
                elif c1 == c0:
                    statuses.append(FITS); reasons.append(Y.ST_OK); blocking.append(Y.WHY_CLAIM_NONE)
                else:
                    statuses.append(INVALID)
                    r, c = PW.pair_reason(W, node_off, table, claims, c0, c1, n, attrs, sels, False, have_off)
                    reasons.append(r); blocking.append(c)
                pair_pods.append(p)
            continue
        # judged: §14 with this one pod against W_p and the running pods not evicted yet (their order kept)
        idx = [i for r in alive for i in range(int(run_pod_off[r]), int(run_pod_off[r + 1]))]
        rpo = np.zeros(len(alive) + 1, np.uint32)
        rpo[1:] = np.cumsum([int(run_pod_off[r + 1]) - int(run_pod_off[r]) for r in alive])
        sub_rc = run_claims[idx] if len(idx) else np.zeros(0, O.CLAIM_DTYPE)
        sub_ro = run_out if run_out_off is not None else (run_out[idx] if len(idx) else np.zeros(0, O.OUT_DTYPE))
        sub_roo = None if run_out_off is None else np.asarray(run_out_off, np.uint32)[idx]
        one = P.preempt(W, node_off, table, pod, np.array([0, c1 - c0], np.uint32), np.array([prio[p]], np.int32), sub_rc,
                        rpo, np.asarray([run_prio[r] for r in alive], np.int32), sub_ro, sub_roo,
                        None if cand_off is None else np.array(nodes, np.uint32),
                        None if cand_off is None else np.array([0, len(nodes)], np.uint32), 0, flags)[0]
        st = [int(x) for x in one]
        for r, c in _pod_pairs(W, node_off, table, claims, c0, c1, int(prio[p]), nodes, st, effects, run_prio, alive,
                               backtrack, attrs, sels):
            reasons.append(r); blocking.append(c); pair_pods.append(p)
        statuses += st
    pod_why, blocks = _tally(n_pod, len(claims), pair_pods, reasons, blocking)
    return whole + (np.array(statuses, np.uint8), np.array(reasons, np.uint8), np.array(blocking, np.uint32), pod_why,
                    blocks)


# ---- the second statement, on oracle/naive.py -----------------------------------------------------------------------
def _naive_effects(gpus, node_off, run_claims, run_pod_off, run_out, run_out_off):
    """per running pod: (node or None, OK slots as (gpu, kind, start, size, mem_limit)); run_out: (gpu, start, size,
    profile, status) tuples"""
    n_node = len(node_off) - 1
    res = []
    for r in range(len(run_pod_off) - 1):
        eff = []
        for i in range(run_pod_off[r], run_pod_off[r + 1]):
            c = run_claims[i]
            n = c["count"] if (c["kind"] == 0 and c["node"] < n_node and 1 <= c["count"] <= 32
                               and (run_out_off is not None or c["count"] == 1)) else 1
            base = i if run_out_off is None else run_out_off[i]
            eff += [(o[0], c["kind"], o[1], o[2], c["mem_limit_mib"]) for o in run_out[base:base + n] if o[4] == 0]
        nodes = {bisect.bisect_right(list(node_off), e[0]) - 1 for e in eff}
        res.append((nodes.pop() if nodes else None, eff))
    return res


def _naive_release(W, g0, eff):
    for gpu, kind, start, size, lim in eff:
        g = W[gpu - g0]
        if kind == 0:
            g["full"] = False
        elif kind == 1:
            g["used"] -= set(range(start, min(start + size, 16))) if start < 16 else set()
        elif kind == 2:
            g["mem"] = (g["mem"] + lim) % (1 << 32)
            g["share"] = (g["share"] - 1) % (1 << 16)


def _naive_pod(N, G, node_off, table, pod, c0, prio_p, nodes, statuses, effects, run_prio, alive, exhaustive):
    n_node = len(node_off) - 1
    out = []
    for n, st in zip(nodes, statuses):
        if n >= n_node:
            out.append((Y.WHY_NO_NODE, Y.WHY_CLAIM_NONE))
            continue
        W = copy.deepcopy(G[node_off[n]:node_off[n + 1]])
        if st in (NO, SEARCH_LIMIT):                   # S': every lower-priority running pod on n gone
            for r in alive:
                if effects[r][0] == n and run_prio[r] < prio_p:
                    _naive_release(W, node_off[n], effects[r][1])
        r, b = PW.naive_pod_reason(N, W, table, [dict(c, node=n) for c in pod], n_node, exhaustive, True)
        out.append((r, Y.WHY_CLAIM_NONE if b is None else c0 + b))
    return out


def preempt_why_naive(gpus, node_off, table, claims, pod_off, prio, cands, exhaustive, run_claims, run_pod_off, run_prio,
                      run_out, run_out_off=None):
    """spec §19's §14 form on preempt_naive and naive_pod_reason (small cases, no selectors); arguments as
    preempt_oracle.preempt_naive takes them.  Returns (pair_status, pair_why, pair_claim, pod_why, claim_blocks) as
    lists."""
    from oracle import naive as N
    if len(pod_off) == 1:
        return [], [], [], [], [0] * len(claims)
    st = P.preempt_naive(gpus, node_off, table, claims, pod_off, prio, cands, exhaustive, run_claims, run_pod_off,
                         run_prio, run_out, run_out_off, 1)[0]
    n_node = len(node_off) - 1
    G = N._state(gpus)
    effects = _naive_effects(gpus, node_off, run_claims, run_pod_off, run_out, run_out_off)
    alive = list(range(len(run_pod_off) - 1))
    why, claim, pod_why, blocks, k = [], [], [], [0] * len(claims), 0
    for p in range(len(pod_off) - 1):
        nodes = list(range(n_node)) if cands is None else list(cands[p])
        row = [0] * Y.WHY_N
        for r, b in _naive_pod(N, G, node_off, table, claims[pod_off[p]:pod_off[p + 1]], pod_off[p], prio[p], nodes,
                               st[k:k + len(nodes)], effects, run_prio, alive, exhaustive):
            why.append(r); claim.append(b); row[r] += 1
            if b != Y.WHY_CLAIM_NONE:
                blocks[b] += 1
        pod_why.append(row)
        k += len(nodes)
    return list(st), why, claim, pod_why, blocks


def preempt_place_why_naive(gpus, node_off, table, claims, pod_off, prio, cands, exhaustive, run_claims, run_pod_off,
                            run_prio, run_out, out_off=None, run_out_off=None):
    """spec §19's §15 form as the host loop on the naive restatements: W_p from preempt_place_naive on the pods before
    p, then pod p's pairs from preempt_naive against W_p and the running pods not evicted yet, answered by naive_pod_reason.
    Returns (pair_status, pair_why, pair_claim, pod_why, claim_blocks) as lists."""
    from oracle import naive as N
    n_node, n_run = len(node_off) - 1, len(run_pod_off) - 1
    have_off = out_off is not None
    effects = _naive_effects(gpus, node_off, run_claims, run_pod_off, run_out, run_out_off)
    status, why, claim, pod_why, blocks = [], [], [], [], [0] * len(claims)
    for p in range(len(pod_off) - 1):
        c0, c1 = pod_off[p], pod_off[p + 1]
        pod = claims[c0:c1]
        nodes = list(range(n_node)) if cands is None else list(cands[p])
        _, _, _, ev, after = PP.preempt_place_naive(gpus, node_off, table, claims[:c0], pod_off[:p + 1], prio[:p],
                                                     None if cands is None else cands[:p], exhaustive, run_claims,
                                                     run_pod_off, run_prio, run_out,
                                                     None if out_off is None else out_off[:c0], run_out_off)
        G = N._state(after)
        alive = [r for r in range(n_run) if ev[r] == NONE]
        row = [0] * Y.WHY_N
        inv = len(pod) > N.MAX_POD or any(N._invalid(dict(c, node=0), 1, have_off) for c in pod)
        if inv or not pod:
            recs = []
            for n in nodes:
                if n >= n_node:
                    recs.append((NO, Y.WHY_NO_NODE, Y.WHY_CLAIM_NONE))
                elif not pod:
                    recs.append((FITS, Y.ST_OK, Y.WHY_CLAIM_NONE))
                elif len(pod) > N.MAX_POD:
                    recs.append((INVALID, Y.ST_INVALID, Y.WHY_CLAIM_NONE))
                else:
                    i = next(i for i, c in enumerate(pod) if N._invalid(dict(c, node=0), 1, have_off))
                    recs.append((INVALID, Y.ST_INVALID, c0 + i))
        else:
            rpo, idx = [0], []
            for r in alive:
                idx += list(range(run_pod_off[r], run_pod_off[r + 1]))
                rpo.append(len(idx))
            st = P.preempt_naive(after, node_off, table, pod, [0, len(pod)], [prio[p]], None if cands is None else [nodes],
                                 exhaustive, [run_claims[i] for i in idx], rpo, [run_prio[r] for r in alive],
                                 [run_out[i] for i in idx] if run_out_off is None else run_out,
                                 None if run_out_off is None else [run_out_off[i] for i in idx], 1)[0]
            recs = [(s, r, b) for s, (r, b) in zip(st, _naive_pod(N, G, node_off, table, pod, c0, prio[p], nodes, st,
                                                                  effects, run_prio, alive, exhaustive))]
        for s, r, b in recs:
            status.append(s); why.append(r); claim.append(b); row[r] += 1
            if b != Y.WHY_CLAIM_NONE:
                blocks[b] += 1
        pod_why.append(row)
    return status, why, claim, pod_why, blocks
