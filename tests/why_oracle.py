"""Spec §17 (why each node is unsuitable) restated in Python — TEST INFRASTRUCTURE ONLY.

`why` answers every (pod, candidate) pair with a reason and a blocking claim, and sums the per-pod and per-claim tallies.
Without DRA_F_EXHAUSTIVE the answer is read off oracle/dra_oracle.c's Allocate of the pod on the node's snapshot (the
first claim whose slot is not OK), which is §17's definition.  With it, steps 1-3 of §12 are stated here: the invalid
claims and the GPU / SHARED claims again through that Allocate, the pre-check per MIG claim as an Allocate of the claim
alone, and the MIG search as a plain recursion that counts its descents and the most levels it held at once (d).
Selectors (spec §10) are evaluated here too; the C oracle takes them through `set_selectors`.

`why_naive` states §17 a second time on oracle/naive.py's Allocate and state dicts (no selectors), sharing no code with
the C oracle or with `why`; the CPU suite checks that the two agree."""
from __future__ import annotations

import numpy as np

from oracle import oracle as O

ST_OK, ST_NO_CAPACITY, ST_BAD_PROFILE, ST_GROUP, ST_MEM_LIMIT, ST_INVALID, ST_POD, ST_SEARCH_LIMIT = range(8)
WHY_NO_NODE, WHY_N, WHY_CLAIM_NONE = 8, 9, 0xFFFFFFFF
F_EXHAUSTIVE = O.F_EXHAUSTIVE
KIND_GPU, KIND_MIG, KIND_SHARED = 0, 1, 2
MAX_POD, EXH_BUDGET, MAX_COUNT, MAX_PROFILES = 32, 4096, 32, 16
_MIG, _FULL, _UNAVAIL = 1, 2, 4


def _slots(c):
    return int(c["count"]) if c["kind"] == KIND_GPU and 1 <= c["count"] <= MAX_COUNT else 1


def _sel_id(c):
    return int(c["mem_limit_mib"]) if c["kind"] in (KIND_GPU, KIND_MIG) else int(c["group"]) if c["kind"] == KIND_SHARED else 0


def sel_pass(attrs, sels, sid, gpu):
    """Spec §10: does GPU `gpu` pass selector `sid` (1-based; 0 = none)?"""
    if sid == 0:
        return True
    if sels is None or sid > len(sels):
        return False
    a = attrs[gpu] if attrs is not None and len(attrs) else None
    val = {0: a["mem_total_mib"], 1: a["cc"], 2: a["index"], 3: a["product"], 4: a["driver_major"]} if a is not None \
        else {k: 0 for k in range(5)}
    stack = []
    for ins in sels[sid - 1]:
        op, attr, cmp, v2 = int(ins["op"]), int(ins["attr"]), int(ins["cmp"]), int(ins["value"])
        if op == 0:
            break
        if op == 1:
            if attr not in val:
                return False
            v = int(val[attr])
            r = {0: v == v2, 1: v != v2, 2: v < v2, 3: v <= v2, 4: v > v2, 5: v >= v2,
                 6: v < 32 and (v2 >> v) & 1 == 1}.get(cmp)
            if r is None:
                return False
            stack.append(bool(r))
        elif op in (2, 3):
            if len(stack) < 2:
                return False
            b, a_ = stack.pop(), stack.pop()
            stack.append((a_ and b) if op == 2 else (a_ or b))
        elif op == 4:
            if not stack:
                return False
            stack.append(not stack.pop())
        else:
            return False
    return not stack or stack[-1]


def _first_bad(gpus, node_off, table, pod):
    """(index, status) of the first claim of `pod` whose slot an Allocate on the snapshot leaves not OK, or None."""
    if len(pod) == 0:
        return None
    sl = [_slots(c) for c in pod]
    off = np.concatenate([[0], np.cumsum(sl)[:-1]]).astype(np.uint32)
    out, _ = O.allocate(gpus, node_off, table, pod, out_off=off, n_out=int(sum(sl)))
    for i in range(len(pod)):
        st = int(out[off[i]]["status"])
        if st != ST_OK:
            return i, st
    return None


def _search(gpus, g0, g1, table, pod, mig, attrs, sels):
    """The §12 search over the MIG claims `mig` (positions in pod) in canonical order.  Returns (status, d)."""
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
            if (g["flags"] & (_MIG | _FULL | _UNAVAIL)) != _MIG or not mask:
                continue
            if not sel_pass(attrs, sels, int(c["mem_limit_mib"]), g0 + k):
                continue
            for s in range(16):
                cells = ((1 << size) - 1) << s
                if (mask >> s) & 1 and s + size <= 16 and not (used[k] & cells):
                    yield k, s, cells

    def rec(level):
        if level == len(mig):
            return ST_OK
        for k, s, cells in options(level):
            if state["descents"] == EXH_BUDGET:
                return ST_SEARCH_LIMIT
            state["descents"] += 1
            used[k] |= cells
            choice[level] = (k, s)
            state["depth"] += 1
            state["d"] = max(state["d"], state["depth"])
            r = rec(level + 1)
            if r != ST_POD:
                return r
            used[k] &= ~cells
            state["depth"] -= 1
        return ST_POD

    return rec(0), state["d"]


def _pair(gpus, node_off, table, claims, c0, c1, node, flags, attrs, sels):
    n_node = len(node_off) - 1
    if node >= n_node:
        return WHY_NO_NODE, WHY_CLAIM_NONE
    pod = np.array(claims[c0:c1], dtype=O.CLAIM_DTYPE)
    pod["node"] = node
    if not flags & F_EXHAUSTIVE:
        bad = _first_bad(gpus, node_off, table, pod)
        return (ST_OK, WHY_CLAIM_NONE) if bad is None else (bad[1], c0 + bad[0])
    if len(pod) > MAX_POD:
        return ST_INVALID, WHY_CLAIM_NONE
    if len(pod) == 0:
        return ST_OK, WHY_CLAIM_NONE
    # step 1: the invalid claims (Allocate marks exactly those INVALID)
    sl = [_slots(c) for c in pod]
    off = np.concatenate([[0], np.cumsum(sl)[:-1]]).astype(np.uint32)
    out, _ = O.allocate(gpus, node_off, table, pod, out_off=off, n_out=int(sum(sl)))
    for i in range(len(pod)):
        if out[off[i]]["status"] == ST_INVALID:
            return ST_INVALID, c0 + i
    # step 2: the GPU / SHARED claims in order
    other = [i for i in range(len(pod)) if pod[i]["kind"] != KIND_MIG]
    bad = _first_bad(gpus, node_off, table, pod[other])
    if bad is not None:
        return bad[1], c0 + other[bad[0]]
    # step 3: the pre-check, each MIG claim alone on the node as it stands (GPU / SHARED claims take no MIG GPU)
    mig = [i for i in range(len(pod)) if pod[i]["kind"] == KIND_MIG]
    for i in mig:
        one = pod[i:i + 1].copy()
        one["group"] = 0
        bad = _first_bad(gpus, node_off, table, one)
        if bad is not None:
            return bad[1], c0 + i
    st, d = _search(gpus, int(node_off[node]), int(node_off[node + 1]), table, pod, mig, attrs, sels)
    return (ST_OK, WHY_CLAIM_NONE) if st == ST_OK else (st, c0 + mig[d])


def why(gpus, node_off, table, claims, pod_off, cand_nodes=None, cand_off=None, flags: int = 0, attrs=None, sels=None):
    """spec §17.  cand_nodes/cand_off None = every pod against every node (pair = pod * n_node + node).  The selectors
    must also be set in the C oracle (`set_selectors`).  Returns (pair_why u8, pair_claim u32, pod_why u32 [n_pod, 9],
    claim_blocks u32 [n_claim])."""
    gpus = np.ascontiguousarray(gpus, dtype=O.GPU_DTYPE)
    claims = np.ascontiguousarray(claims, dtype=O.CLAIM_DTYPE) if claims is not None and len(claims) else \
        np.zeros(0, O.CLAIM_DTYPE)
    n_node, n_pod = len(node_off) - 1, len(pod_off) - 1
    reasons, blocking = [], []
    pod_why = np.zeros((n_pod, WHY_N), np.uint32)
    blocks = np.zeros(len(claims), np.uint32)
    for p in range(n_pod):
        nodes = range(n_node) if cand_off is None else [int(x) for x in cand_nodes[cand_off[p]:cand_off[p + 1]]]
        for n in nodes:
            r, c = _pair(gpus, node_off, table, claims, int(pod_off[p]), int(pod_off[p + 1]), n, flags, attrs, sels)
            reasons.append(r)
            blocking.append(c)
            pod_why[p, r] += 1
            if c != WHY_CLAIM_NONE:
                blocks[c] += 1
    return np.array(reasons, np.uint8), np.array(blocking, np.uint32), pod_why, blocks


def why_naive(gpus, node_off, table, claims, pod_off, cands, exhaustive):
    """spec §17 restated a second time on oracle/naive.py (small cases, no selectors), sharing no code with the C oracle
    or with `why` above.  gpus / claims: lists of dicts as naive.py takes them; table[model][profile] = (size,
    start_mask); cands: one list of nodes per pod, or None for every node ascending.  Returns the four outputs as lists
    (pod_why as one list of WHY_N counts per pod)."""
    import copy

    from oracle import naive as N
    n_node = len(node_off) - 1
    reasons, blocking, pod_why, blocks = [], [], [], [0] * len(claims)
    for p in range(len(pod_off) - 1):
        c0, c1 = pod_off[p], pod_off[p + 1]
        row = [0] * WHY_N
        for n in (range(n_node) if cands is None else cands[p]):
            pod = [dict(c, node=n) for c in claims[c0:c1]]
            if n >= n_node:
                r, b = WHY_NO_NODE, None
            elif not exhaustive:
                # the first slot of the pod's own Allocate, slots as with out_off, that is not OK
                sl = [N._slots(c, n_node, True) for c in pod]
                out, _ = N.allocate(gpus, node_off, table, pod, [sum(sl[:i]) for i in range(len(pod))])
                first = [out[sum(sl[:i])][4] for i in range(len(pod))]
                bad = [i for i, st in enumerate(first) if st != ST_OK]
                r, b = (first[bad[0]], bad[0]) if bad else (ST_OK, None)
            else:
                r, b = _naive_pod(N, copy.deepcopy(N._state(gpus)[node_off[n]:node_off[n + 1]]), table, pod, n_node)
            reasons.append(r)
            blocking.append(WHY_CLAIM_NONE if b is None else c0 + b)
            row[r] += 1
            if b is not None:
                blocks[c0 + b] += 1
        pod_why.append(row)
    return reasons, blocking, pod_why, blocks


def _naive_pod(N, W, table, pod, n_node):
    """§17 with DRA_F_EXHAUSTIVE for one pod on the node's GPUs W (naive.py's state dicts): (reason, position or None)"""
    if len(pod) > MAX_POD:
        return ST_INVALID, None
    for i, c in enumerate(pod):                                    # step 1
        if N._invalid(c, n_node, True):
            return ST_INVALID, i
    for i, c in enumerate(pod):                                    # step 2, in order
        if c["kind"] == KIND_GPU:
            el = [g for g in W if not (g["mig"] or g["full"] or g["unavail"]) and g["share"] == 0]
            if len(el) < c["count"]:
                return ST_NO_CAPACITY, i
            for g in el[: c["count"]]:
                g["full"] = True
        elif c["kind"] == KIND_SHARED:
            g = next((g for g in W if not (g["mig"] or g["full"] or g["unavail"]) and g["share"] < 0xFFFF
                      and g["mem"] >= c["mem_limit_mib"]), None)
            if g is None:
                return ST_MEM_LIMIT, i
            g["mem"] -= c["mem_limit_mib"]
            g["share"] += 1
    mig = [i for i, c in enumerate(pod) if c["kind"] == KIND_MIG]

    def free_starts(g, prof, used):
        size, mask = table[g["model"]][prof]
        return [s for s in range(16) if (mask >> s) & 1 and s + size <= 16 and not set(range(s, s + size)) & used]

    for i in mig:                                                  # step 3: the pre-check
        prof = pod[i]["profile"]
        usable = [g for g in W if g["mig"] and not g["unavail"] and table[g["model"]][prof][1]]
        if not any(free_starts(g, prof, g["used"]) for g in usable if not g["full"]):
            return (ST_NO_CAPACITY if usable else ST_BAD_PROFILE), i
    held, deepest, descents, placed = [], [0], [0], {}

    def search(level):
        if level == len(mig):
            return ST_OK
        c = pod[mig[level]]
        same = [j for j in range(level) if c["group"] and pod[mig[j]]["group"] == c["group"]]
        for k, g in enumerate(W):
            if same and placed[same[0]] != k:
                continue
            if not g["mig"] or g["unavail"] or g["full"]:
                continue
            for s in free_starts(g, c["profile"], g["used"]):
                if descents[0] == EXH_BUDGET:
                    return ST_SEARCH_LIMIT
                descents[0] += 1
                cells = set(range(s, s + table[g["model"]][c["profile"]][0]))
                g["used"] |= cells
                placed[level] = k
                held.append(level)
                deepest[0] = max(deepest[0], len(held))
                r = search(level + 1)
                if r != ST_POD:
                    return r
                held.pop()
                g["used"] -= cells
        return ST_POD

    r = search(0)
    return (ST_OK, None) if r == ST_OK else (r, mig[deepest[0]])
