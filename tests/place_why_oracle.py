"""Spec §18 (why place pods put each pod where it did) restated in Python — TEST INFRASTRUCTURE ONLY.

`place_why` walks the pods in input order.  It answers each pod's pairs with `pair_reason` (§17's §12 branch, on
why_oracle's helpers, with backtracking only under DRA_F_EXHAUSTIVE and validity in the call's slot mode) on the state
the pods before it left, then advances that state with place_oracle's `place_pods` run on that one pod.
`place_why_naive` states the same thing a second time on `place_pods_naive` and `naive_pod_reason` (oracle/naive.py, no
selectors), sharing no code with the first; the CPU suite checks that the two agree."""
from __future__ import annotations

import numpy as np

import place_oracle as P
import why_oracle as Y
from oracle import oracle as O


def _slots(c, have_off):
    """OutRec slots of claim c in a place pods call: counted as if it named a node of the inventory"""
    return int(c["count"]) if have_off and c["kind"] == Y.KIND_GPU and 1 <= c["count"] <= Y.MAX_COUNT else 1


def _search(gpus, g0, g1, table, pod, mig, attrs, sels, backtrack):
    """The §12 search over the MIG claims `mig` (positions in pod) in canonical order: (status, d).  backtrack False:
    each level takes its first admissible choice, and a level with none fails the search (POD)."""
    used = [int(gpus[g]["busy"]) for g in range(g0, g1)]
    choice = {}
    state = {"descents": 0, "depth": 0, "d": 0}

    def options(level):
        c = pod[mig[level]]
        want = None
        if c["group"]:
            for j in range(level):
                if pod[mig[j]]["group"] == c["group"]:
                    want = choice[j][0]
                    break
        for k in range(g1 - g0):
            g = gpus[g0 + k]
            e = table[g["model"]][c["profile"]]
            size, mask = int(e["size"]), int(e["start_mask"])
            if want is not None and k != want:
                continue
            if (g["flags"] & (Y._MIG | Y._FULL | Y._UNAVAIL)) != Y._MIG or not mask:
                continue
            if not Y.sel_pass(attrs, sels, int(c["mem_limit_mib"]), g0 + k):
                continue
            for s in range(16):
                cells = ((1 << size) - 1) << s
                if (mask >> s) & 1 and s + size <= 16 and not (used[k] & cells):
                    yield k, s, cells

    def rec(level):
        if level == len(mig):
            return Y.ST_OK
        for k, s, cells in options(level):
            if state["descents"] == Y.EXH_BUDGET:
                return Y.ST_SEARCH_LIMIT
            state["descents"] += 1
            used[k] |= cells
            choice[level] = (k, s)
            state["depth"] += 1
            state["d"] = max(state["d"], state["depth"])
            r = rec(level + 1)
            if r != Y.ST_POD or not backtrack:
                return r
            used[k] &= ~cells
            state["depth"] -= 1
        return Y.ST_POD

    return rec(0), state["d"]


def pair_reason(gpus, node_off, table, claims, c0, c1, node, attrs, sels, backtrack, have_off):
    """One pair's (reason, blocking claim) by §17's §12 steps on the state `gpus`.  backtrack False: the search does not
    backtrack; have_off False: validity as a call without out_off judges it (a GPU claim of count != 1 is invalid)."""
    n_node = len(node_off) - 1
    if node >= n_node:
        return Y.WHY_NO_NODE, Y.WHY_CLAIM_NONE
    pod = np.array(claims[c0:c1], dtype=O.CLAIM_DTYPE)
    pod["node"] = node
    if len(pod) > Y.MAX_POD:
        return Y.ST_INVALID, Y.WHY_CLAIM_NONE
    if len(pod) == 0:
        return Y.ST_OK, Y.WHY_CLAIM_NONE
    # step 1: the invalid claims, in the call's slot mode (Allocate marks exactly those INVALID)
    if have_off:
        sl = [Y._slots(c) for c in pod]
        off = np.concatenate([[0], np.cumsum(sl)[:-1]]).astype(np.uint32)
        out, _ = O.allocate(gpus, node_off, table, pod, out_off=off, n_out=int(sum(sl)))
    else:
        off = np.arange(len(pod), dtype=np.uint32)
        out, _ = O.allocate(gpus, node_off, table, pod, n_out=len(pod))
    for i in range(len(pod)):
        if out[off[i]]["status"] == Y.ST_INVALID:
            return Y.ST_INVALID, c0 + i
    # step 2: the GPU / SHARED claims in order
    other = [i for i in range(len(pod)) if pod[i]["kind"] != Y.KIND_MIG]
    bad = Y._first_bad(gpus, node_off, table, pod[other])
    if bad is not None:
        return bad[1], c0 + other[bad[0]]
    # step 3: the pre-check, each MIG claim alone on the node as it stands (GPU / SHARED claims take no MIG GPU)
    mig = [i for i in range(len(pod)) if pod[i]["kind"] == Y.KIND_MIG]
    for i in mig:
        one = pod[i:i + 1].copy()
        one["group"] = 0
        bad = Y._first_bad(gpus, node_off, table, one)
        if bad is not None:
            return bad[1], c0 + i
    st, d = _search(gpus, int(node_off[node]), int(node_off[node + 1]), table, pod, mig, attrs, sels, backtrack)
    return (Y.ST_OK, Y.WHY_CLAIM_NONE) if st == Y.ST_OK else (st, c0 + mig[d])


def place_why(gpus, node_off, table, claims, pod_off, cand_nodes=None, cand_off=None, out_off=None, n_out=None,
              flags: int = 0, attrs=None, sels=None):
    """spec §18 from the start state `gpus` (DRA_F_FRESH_INVENTORY is the caller's: pass the pristine inventory).  The
    selectors must also be set in the C oracle (`set_selectors`).  Returns (out, pod_node, gpus_after, pair_why u8,
    pair_claim u32, pod_why u32 [n_pod, WHY_N], claim_blocks u32 [n_claim])."""
    g = np.ascontiguousarray(gpus, dtype=O.GPU_DTYPE).copy()
    claims = np.ascontiguousarray(claims, dtype=O.CLAIM_DTYPE) if claims is not None and len(claims) else \
        np.zeros(0, O.CLAIM_DTYPE)
    have_off = out_off is not None
    if n_out is None:
        n_out = len(claims) if not have_off else 0
    n_node, n_pod = len(node_off) - 1, len(pod_off) - 1
    out = np.zeros(n_out, dtype=O.OUT_DTYPE)
    pod_node = np.full(n_pod, P.NONE, np.uint32)
    backtrack = bool(flags & Y.F_EXHAUSTIVE)
    reasons, blocking = [], []
    pod_why = np.zeros((n_pod, Y.WHY_N), np.uint32)
    blocks = np.zeros(len(claims), np.uint32)
    for p in range(n_pod):
        c0, c1 = int(pod_off[p]), int(pod_off[p + 1])
        nodes = list(range(n_node)) if cand_off is None else [int(x) for x in cand_nodes[cand_off[p]:cand_off[p + 1]]]
        for n in nodes:                                  # every pair on W_p
            r, c = pair_reason(g, node_off, table, claims, c0, c1, n, attrs, sels, backtrack, have_off)
            reasons.append(r)
            blocking.append(c)
            pod_why[p, r] += 1
            if c != Y.WHY_CLAIM_NONE:
                blocks[c] += 1
        # W_{p+1}: the pod placed alone on W_p, its slots copied into the call's out
        sub = claims[c0:c1]
        oo = None if not have_off else np.asarray(out_off[c0:c1], np.uint32)
        o1, pn, g = P.place_pods(g, node_off, table, sub, np.array([0, c1 - c0], np.uint32),
                                 None if cand_off is None else np.array(nodes, np.uint32),
                                 None if cand_off is None else np.array([0, len(nodes)], np.uint32),
                                 oo, n_out if have_off else c1 - c0, flags & Y.F_EXHAUSTIVE)
        pod_node[p] = pn[0]
        for i in range(c1 - c0):
            b = int(oo[i]) if have_off else i
            d = b if have_off else c0 + i
            k = _slots(sub[i], have_off)
            out[d:d + k] = o1[b:b + k]
    return (out, pod_node, g, np.array(reasons, np.uint8), np.array(blocking, np.uint32), pod_why, blocks)


def place_why_naive(gpus, node_off, table, claims, pod_off, cands, exhaustive, out_off=None):
    """spec §18 restated on oracle/naive.py (small cases, no selectors): place_pods_naive one pod at a time, each pod's
    pairs answered by naive_pod_reason on the state before it.  gpus / claims: lists of dicts as naive.py takes them; cands:
    one list of nodes per pod, or None for every node ascending.  Returns (out list, pod_node list, gpus_after, pair_why,
    pair_claim, pod_why, claim_blocks) as lists."""
    import copy

    from oracle import naive as N
    n_node = len(node_off) - 1
    have_off = out_off is not None
    cur = [dict(g) for g in gpus]
    out, pod_node, reasons, blocking, pod_why, blocks = {}, [], [], [], [], [0] * len(claims)
    for p in range(len(pod_off) - 1):
        c0, c1 = pod_off[p], pod_off[p + 1]
        nodes = list(range(n_node)) if cands is None else list(cands[p])
        row = [0] * Y.WHY_N
        G = N._state(cur)
        for n in nodes:
            if n >= n_node:
                r, b = Y.WHY_NO_NODE, None
            else:
                pod = [dict(c, node=n) for c in claims[c0:c1]]
                r, b = naive_pod_reason(N, copy.deepcopy(G[node_off[n]:node_off[n + 1]]), table, pod, n_node,
                                        exhaustive, have_off)
            reasons.append(r)
            blocking.append(Y.WHY_CLAIM_NONE if b is None else c0 + b)
            row[r] += 1
            if b is not None:
                blocks[c0 + b] += 1
        pod_why.append(row)
        o1, pn, cur = place_pods_naive_one(cur, node_off, table, claims[c0:c1], nodes, exhaustive,
                                           None if not have_off else out_off[c0:c1])
        pod_node.append(pn)
        out.update(o1 if have_off else {c0 + i: r for i, r in o1.items()})
    n_out = max(out, default=-1) + 1
    return [out.get(i) for i in range(n_out)], pod_node, cur, reasons, blocking, pod_why, blocks


def place_pods_naive_one(gpus, node_off, table, pod, nodes, exhaustive, out_off):
    """place_pods_naive on one pod: ({slot: record}, node or NONE, gpus_after)"""
    out, pn, after = P.place_pods_naive(gpus, node_off, table, pod, [0, len(pod)], [nodes], exhaustive, out_off)
    return {i: r for i, r in enumerate(out) if r is not None}, pn[0], after


def naive_pod_reason(N, W, table, pod, n_node, backtrack, have_off):
    """One pod's (reason, position or None) by §17's §12 steps on the node's GPUs W (naive.py's state dicts).
    backtrack / have_off as in pair_reason."""
    if len(pod) > Y.MAX_POD:
        return Y.ST_INVALID, None
    for i, c in enumerate(pod):                                    # step 1
        if N._invalid(c, n_node, have_off):
            return Y.ST_INVALID, i
    for i, c in enumerate(pod):                                    # step 2, in order
        if c["kind"] == Y.KIND_GPU:
            el = [g for g in W if not (g["mig"] or g["full"] or g["unavail"]) and g["share"] == 0]
            if len(el) < c["count"]:
                return Y.ST_NO_CAPACITY, i
            for g in el[: c["count"]]:
                g["full"] = True
        elif c["kind"] == Y.KIND_SHARED:
            g = next((g for g in W if not (g["mig"] or g["full"] or g["unavail"]) and g["share"] < 0xFFFF
                      and g["mem"] >= c["mem_limit_mib"]), None)
            if g is None:
                return Y.ST_MEM_LIMIT, i
            g["mem"] -= c["mem_limit_mib"]
            g["share"] += 1
    mig = [i for i, c in enumerate(pod) if c["kind"] == Y.KIND_MIG]

    def free_starts(g, prof, used):
        size, mask = table[g["model"]][prof]
        return [s for s in range(16) if (mask >> s) & 1 and s + size <= 16 and not set(range(s, s + size)) & used]

    for i in mig:                                                  # step 3: the pre-check
        prof = pod[i]["profile"]
        usable = [g for g in W if g["mig"] and not g["unavail"] and table[g["model"]][prof][1]]
        if not any(free_starts(g, prof, g["used"]) for g in usable if not g["full"]):
            return (Y.ST_NO_CAPACITY if usable else Y.ST_BAD_PROFILE), i
    held, deepest, descents, placed = [], [0], [0], {}

    def search(level):
        if level == len(mig):
            return Y.ST_OK
        c = pod[mig[level]]
        same = [j for j in range(level) if c["group"] and pod[mig[j]]["group"] == c["group"]]
        for k, g in enumerate(W):
            if same and placed[same[0]] != k:
                continue
            if not g["mig"] or g["unavail"] or g["full"]:
                continue
            for s in free_starts(g, c["profile"], g["used"]):
                if descents[0] == Y.EXH_BUDGET:
                    return Y.ST_SEARCH_LIMIT
                descents[0] += 1
                cells = set(range(s, s + table[g["model"]][c["profile"]][0]))
                g["used"] |= cells
                placed[level] = k
                held.append(level)
                deepest[0] = max(deepest[0], len(held))
                r = search(level + 1)
                if r != Y.ST_POD or not backtrack:
                    return r
                held.pop()
                g["used"] -= cells
        return Y.ST_POD

    r = search(0)
    return (Y.ST_OK, None) if r == Y.ST_OK else (r, mig[deepest[0]])
