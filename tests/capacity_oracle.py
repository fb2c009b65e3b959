"""ctypes wrapper of the CPU oracle of spec §16 (pod capacity) — TEST INFRASTRUCTURE ONLY.

pod_oracle_capacity (tests/pod_oracles.c, loaded by tests/pod_oracles.py) counts the copies of each pod a candidate
node takes with the §12 evaluation of oracle/dra_oracle.c.  `capacity_naive` below is the independent restatement on
top of oracle/naive.py's `eval_pod`: the two share no code, and the CPU suite checks one against the other."""
from __future__ import annotations

import copy

import numpy as np

from oracle import oracle as O
from pod_oracles import _nz, _p, lib, set_selectors  # noqa: F401  (set_selectors: the selectors of every pod oracle)

F_EXHAUSTIVE = O.F_EXHAUSTIVE
ST_OK, ST_INVALID, ST_POD, ST_SEARCH_LIMIT = 0, 5, 6, 7


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
    rc = lib().pod_oracle_capacity(_p(g), len(g), _p(off), n_node, _p(t), _p(c), n_claim, _p(po), n_pod, _p(cn), _p(co),
                                   max_copies, _p(copies), _p(stop), _p(total), _p(nodes), flags)
    if rc != 0:
        raise ValueError(f"pod_oracle_capacity: rc={rc}")
    return copies[:n_pair], stop[:n_pair], total[:n_pod], nodes[:n_pod]


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
