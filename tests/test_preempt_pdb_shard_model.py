"""CPU suite: the partition-and-merge of the sharded preemption call with disruption budgets, modelled in Python as
test_preempt_shard_model.py models it without them.

Each (pod, candidate) pair is judged alone (preempt_pdb_oracle.preempt_naive_pdb with one pod and one candidate: every pair
copies the budgets afresh) by the rank that owns the candidate's node.  Each rank keeps per pod its first FITS position
and its best EVICT pair under the order with the fewest violations first, then the list position; the merge takes the
minimum over the ranks.  For every partition, worlds 1 to 5, the answer must be the single-inventory one of both
oracles."""
import numpy as np
import pytest

from test_oracle_properties import _dicts
from test_pod_mode import _mig, _tbl
from test_preempt import _flat, _outs, _small_world, mig_running, occupied
from test_preempt_shard_model import _partitions

import importlib
import preempt_oracle as P
import preempt_pdb_oracle as PB
from oracle import naive as N

R = importlib.import_module("k8s-dra-driver_b200").records
NONE = 0xFFFFFFFF
BIG = 1 << 16


def _judge(g, off, t, claims, pod_off, prio, rc, rpo, rpr, ro, run_pdb, allowed, p, node, exhaustive):
    """pair (p, node) alone: (status, victims in eviction order, violating victims)"""
    c = claims[pod_off[p]: pod_off[p + 1]]
    a = PB.preempt_naive_pdb(_dicts(g), list(off), _tbl(t), _dicts(c), [0, len(c)], [int(prio[p])], [[int(node)]],
                            exhaustive, _dicts(rc), list(rpo), list(rpr), _outs(ro), run_pdb, allowed, None, BIG)
    st, nv = a[0][0], a[1][0]
    return st, [int(v) for v in a[5][0][:nv]], a[6][0]


def _key(judged, rpr, pos):
    """the merge's order of EVICT pairs: fewest violations, then pre_better's keys, then list position"""
    _, v, viol = judged
    hi = max(int(rpr[r]) for r in v)
    last = min(r for r in v if int(rpr[r]) == hi)
    return (viol, hi, sum(int(rpr[r]) + (1 << 31) for r in v), len(v), -last, pos)


def _sharded(g, off, t, claims, pod_off, prio, rc, rpo, rpr, ro, run_pdb, allowed, cands, exhaustive, max_victims, bounds):
    n_node, world = len(off) - 1, len(bounds) - 1
    n_pod = len(pod_off) - 1
    lists = [list(range(n_node)) if cands is None else [int(n) for n in cands[p]] for p in range(n_pod)]
    base = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(int)

    def owner(n):
        for r in range(world):
            if bounds[r] <= n < bounds[r + 1]:
                return r
        return None

    judged = {}
    for p in range(n_pod):
        for i, n in enumerate(lists[p]):
            if owner(n) is not None:
                judged[base[p] + i] = _judge(g, off, t, claims, pod_off, prio, rc, rpo, rpr, ro, run_pdb, allowed, p, n,
                                             exhaustive)
    parts = []
    for r in range(world):
        pr = []
        for p in range(n_pod):
            fit, best, lim = None, None, False
            for i, n in enumerate(lists[p]):
                k = base[p] + i
                if owner(n) != r:
                    continue
                st = judged[k][0]
                if st == P.FITS and fit is None:
                    fit = k
                elif st == P.SEARCH_LIMIT:
                    lim = True
                elif st == P.EVICT and (best is None or _key(judged[k], rpr, k) < _key(judged[best], rpr, best)):
                    best = k
            if fit is not None:
                best = None
            pr.append((fit, best, lim, judged[best][1][:max_victims] if best is not None else []))
        parts.append(pr)
    pod_node, pod_status, n_victims, rows, pod_viol = [], [], [], [], []
    for p in range(n_pod):
        fits = [parts[r][p][0] for r in range(world) if parts[r][p][0] is not None]
        evict = [(r, parts[r][p][1]) for r in range(world) if parts[r][p][1] is not None]
        row = [NONE] * max_victims
        if fits:
            k = min(fits)
            pod_status.append(P.FITS); pod_node.append(lists[p][k - base[p]]); n_victims.append(0); pod_viol.append(0)
        elif evict:
            r, k = min(evict, key=lambda e: _key(judged[e[1]], rpr, e[1]))
            _, v, viol = judged[k]
            pod_status.append(P.EVICT); pod_node.append(lists[p][k - base[p]]); n_victims.append(len(v))
            pod_viol.append(viol)
            got = parts[r][p][3]
            row[:len(got)] = got
        else:
            c = claims[pod_off[p]: pod_off[p + 1]]
            inv = len(c) > 32 or any(N._invalid(dict(x, node=0), 1, True) for x in _dicts(c))
            lim = any(parts[r][p][2] for r in range(world))
            pod_status.append(P.INVALID if inv else P.SEARCH_LIMIT if lim else P.NO)
            pod_node.append(NONE); n_victims.append(0); pod_viol.append(0)
        rows.append(row)
    pair_status, pair_victims, pair_viol = [], [], []
    for p in range(n_pod):
        for i in range(len(lists[p])):
            st, v, viol = judged.get(base[p] + i, (P.NO, [], 0))
            pair_status.append(st)
            pair_victims.append(len(v) if st == P.EVICT else 0)
            pair_viol.append(viol if st == P.EVICT else 0)
    return pair_status, pair_victims, pod_node, pod_status, n_victims, rows, pair_viol, pod_viol


def _check(g, off, t, c, pod_off, prio, rc, rpo, rpr, ro, run_pdb, allowed, cands, flags, max_victims, partitions):
    exh = bool(flags & P.F_EXHAUSTIVE)
    cn, co = (None, None) if cands is None else _flat(cands)
    ref = PB.preempt_pdb(g, off, t, c, pod_off, prio, rc, rpo, rpr, ro, run_pdb, allowed, None, cn, co, max_victims, flags)
    naive = PB.preempt_naive_pdb(_dicts(g), list(off), _tbl(t), _dicts(c), list(pod_off), list(prio), cands, exh,
                                _dicts(rc), list(rpo), list(rpr), _outs(ro), run_pdb, allowed, None, max_victims)
    for i in (0, 1, 2, 3, 4, 6, 7):
        assert [int(x) for x in ref[i]] == naive[i], i
    assert ref[5].tolist() == [list(r) for r in naive[5]]
    for bounds in partitions:
        got = _sharded(g, off, t, c, pod_off, prio, rc, rpo, rpr, ro, run_pdb, allowed, cands, exh, max_victims, bounds)
        for i in (0, 1, 2, 3, 4, 6, 7):
            assert list(got[i]) == list(naive[i]), (i, bounds)
        assert got[5] == [list(r) for r in naive[5]], ("victims", bounds)
    return ref


@pytest.mark.parametrize("seed", range(30))
def test_random_partitions_give_the_single_inventory_answer(seed):
    w, c, po, prio, cands = _small_world(seed)
    rng = np.random.default_rng(200 + seed)
    n_node, n_run = len(w.node_off) - 1, len(w.run_prio)
    n_pdb = int(rng.integers(1, 4))
    allowed = [int(x) for x in rng.choice([-(1 << 31), -1, 0, 1, 2, (1 << 31) - 1], n_pdb)]
    run_pdb = [int(x) if x < n_pdb else NONE for x in rng.integers(0, n_pdb + 1, n_run)]
    parts = _partitions(rng, n_node, 4)
    for flags in (0, P.F_EXHAUSTIVE):
        _check(w.gpus, w.node_off, w.table, c, po, prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, run_pdb,
               allowed, cands, flags, int(seed % 4), parts)


def test_violations_decide_across_ranks():
    """Node 0's pair has the lower victim priority but violates its budget; node 2's does not.  Every split of the three
    nodes chooses node 2, wherever the two pairs fall."""
    g, off = R.make_inventory([1, 1, 1], mig=True)
    t = R.default_table()
    rc, rpo, rpr, ro = mig_running([(0, 0, 8, R.GI_7_SLICE, 1), (1, 0, 8, R.GI_7_SLICE, 6), (2, 0, 8, R.GI_7_SLICE, 5)],
                                   off)
    g = occupied(g, rc, ro)
    c = _mig(R, [R.GI_7_SLICE])
    parts = [[0, 3], [0, 1, 3], [0, 2, 3], [0, 1, 2, 3], [0, 0, 1, 3, 3], [0, 3, 3]]
    for cands in ([[0, 2]], [[2, 0]], [[0, 1, 2, 0]], [[5, 2, NONE, 0]]):
        ref = _check(g, off, t, c, np.array([0, 1], np.uint32), [9], rc, rpo, rpr, ro, [0, NONE, NONE], [0], cands, 0, 2,
                     parts)
        assert ref[3][0] == P.EVICT and ref[2][0] == 2 and ref[7][0] == 0
