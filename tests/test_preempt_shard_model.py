"""CPU suite: the partition-and-merge of the sharded preemption call (spec §14, "Sharded form"), modelled in Python.

Each (pod, candidate) pair is judged alone — preempt_oracle.preempt_naive with one pod and one candidate — as the rank
that owns the candidate's node judges it.  The pairs are split over random node ranges (empty and uneven ones included,
worlds 1 to 5); each rank reduces its own pairs per pod as k_spre_reduce does (first FITS position, best EVICT pair with
its list position, SEARCH_LIMIT seen), and the merge takes, per pod, the minimum over the ranks as k_spre_merge does.
The answer must be the single-inventory one of both oracles, for every partition."""
import numpy as np
import pytest

from test_oracle_properties import _dicts
from test_pod_mode import _mig, _tbl
from test_preempt import _outs, _small_world, mig_running, occupied

import importlib
import preempt_oracle as P
from oracle import naive as N

R = importlib.import_module("k8s-dra-driver_b200").records
NONE = 0xFFFFFFFF
BIG = 1 << 16


def _judge(g, off, t, claims, pod_off, prio, rc, rpo, rpr, ro, p, node, exhaustive):
    """pair (p, node) alone: (status, victims in eviction order)"""
    c = claims[pod_off[p]: pod_off[p + 1]]
    a = P.preempt_naive(_dicts(g), list(off), _tbl(t), _dicts(c), [0, len(c)], [int(prio[p])], [[int(node)]], exhaustive,
                        _dicts(rc), list(rpo), list(rpr), _outs(ro), None, BIG)
    st, nv = a[0][0], a[1][0]
    return st, [int(v) for v in a[5][0][:nv]]


def _key(victims, rpr, pos):
    """pre_better's order, then list position (smaller is better)"""
    hi = int(rpr[victims[0]])
    return (hi, sum(int(rpr[v]) + (1 << 31) for v in victims), len(victims), -victims[0], pos)


def _sharded(g, off, t, claims, pod_off, prio, rc, rpo, rpr, ro, cands, exhaustive, max_victims, bounds):
    n_node, world = len(off) - 1, len(bounds) - 1
    n_pod = len(pod_off) - 1
    lists = [list(range(n_node)) if cands is None else [int(n) for n in cands[p]] for p in range(n_pod)]
    base = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(int)

    def owner(n):
        for r in range(world):
            if bounds[r] <= n < bounds[r + 1]:
                return r
        return None                                       # a stray: nobody judges it

    judged = {}                                           # pair position -> (status, victims), by its owner only
    for p in range(n_pod):
        for i, n in enumerate(lists[p]):
            if owner(n) is not None:
                judged[base[p] + i] = _judge(g, off, t, claims, pod_off, prio, rc, rpo, rpr, ro, p, n, exhaustive)
    # step 3: each rank's partial per pod
    parts = []
    for r in range(world):
        pr = []
        for p in range(n_pod):
            fit, best, lim = None, None, False
            for i, n in enumerate(lists[p]):
                k = base[p] + i
                if owner(n) != r:
                    continue
                st, v = judged[k]
                if st == P.FITS and fit is None:
                    fit = k
                elif st == P.SEARCH_LIMIT:
                    lim = True
                elif st == P.EVICT and (best is None or _key(v, rpr, k) < _key(judged[best][1], rpr, best)):
                    best = k
            if fit is not None:
                best = None
            row = judged[best][1][:max_victims] if best is not None else []
            pr.append((fit, best, lim, row))
        parts.append(pr)
    # step 5: the merge
    pod_node, pod_status, n_victims, rows = [], [], [], []
    for p in range(n_pod):
        fits = [parts[r][p][0] for r in range(world) if parts[r][p][0] is not None]
        evict = [(r, parts[r][p][1]) for r in range(world) if parts[r][p][1] is not None]
        row = [NONE] * max_victims
        if fits:
            k = min(fits)
            pod_status.append(P.FITS); pod_node.append(lists[p][k - base[p]]); n_victims.append(0)
        elif evict:
            r, k = min(evict, key=lambda e: _key(judged[e[1]][1], rpr, e[1]))
            v = judged[k][1]
            pod_status.append(P.EVICT); pod_node.append(lists[p][k - base[p]]); n_victims.append(len(v))
            got = parts[r][p][3]
            row[:len(got)] = got
        else:
            c = claims[pod_off[p]: pod_off[p + 1]]
            inv = len(c) > 32 or any(N._invalid(dict(x, node=0), 1, True) for x in _dicts(c))
            lim = any(parts[r][p][2] for r in range(world))
            pod_status.append(P.INVALID if inv else P.SEARCH_LIMIT if lim else P.NO)
            pod_node.append(NONE); n_victims.append(0)
        rows.append(row)
    pair_status, pair_victims = [], []
    for p in range(n_pod):
        for i in range(len(lists[p])):
            st, v = judged.get(base[p] + i, (P.NO, []))
            pair_status.append(st); pair_victims.append(len(v) if st == P.EVICT else 0)
    return pair_status, pair_victims, pod_node, pod_status, n_victims, rows


def _partitions(rng, n_node, count):
    out = [[0, n_node]]
    for _ in range(count):
        world = int(rng.integers(1, 6))
        cuts = sorted(int(x) for x in rng.integers(0, n_node + 1, world - 1))
        out.append([0] + cuts + [n_node])
    if n_node >= 1:
        out.append([0, 0, n_node, n_node])               # empty first and last ranges
    return out


def _check(g, off, t, c, pod_off, prio, rc, rpo, rpr, ro, cands, flags, max_victims, partitions):
    exh = bool(flags & P.F_EXHAUSTIVE)
    cn, co = (None, None) if cands is None else _flat(cands)
    ref = P.preempt(g, off, t, c, pod_off, prio, rc, rpo, rpr, ro, None, cn, co, max_victims, flags)
    naive = P.preempt_naive(_dicts(g), list(off), _tbl(t), _dicts(c), list(pod_off), list(prio), cands, exh,
                            _dicts(rc), list(rpo), list(rpr), _outs(ro), None, max_victims)
    assert [list(x) for x in ref[:5]] == [list(x) for x in naive[:5]] and ref[5].tolist() == [list(r) for r in naive[5]]
    for bounds in partitions:
        got = _sharded(g, off, t, c, pod_off, prio, rc, rpo, rpr, ro, cands, exh, max_victims, bounds)
        for name, x, y in zip(("pair_status", "pair_victims", "pod_node", "pod_status", "n_victims"), got[:5], naive[:5]):
            assert list(x) == list(y), (name, bounds)
        assert got[5] == [list(r) for r in naive[5]], ("victims", bounds)
    return ref


def _flat(cands):
    off = np.zeros(len(cands) + 1, np.uint32)
    off[1:] = np.cumsum([len(x) for x in cands])
    return np.array([n for x in cands for n in x], dtype=np.uint32), off


@pytest.mark.parametrize("seed", range(40))
def test_random_partitions_give_the_single_inventory_answer(seed):
    w, c, po, prio, cands = _small_world(seed)
    rng = np.random.default_rng(100 + seed)
    n_node = len(w.node_off) - 1
    parts = _partitions(rng, n_node, 4)
    for flags in (0, P.F_EXHAUSTIVE):
        _check(w.gpus, w.node_off, w.table, c, po, prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, cands,
               flags, int(seed % 4), parts)


def test_ties_between_ranks_and_duplicates():
    """Node 0 and node 2 tie on the highest victim priority, the sum and the count, and differ only in the victim's
    start (its index); node 1's victim ranks higher.  Candidate lists repeat nodes and name strays.  Every split of the
    three nodes over one to three ranks answers as one inventory does."""
    g, off = R.make_inventory([1, 1, 1], mig=True)
    t = R.default_table()
    rc, rpo, rpr, ro = mig_running([(0, 0, 8, R.GI_7_SLICE, 5), (1, 0, 8, R.GI_7_SLICE, 6), (2, 0, 8, R.GI_7_SLICE, 5)],
                                   off)
    g = occupied(g, rc, ro)
    c = _mig(R, [R.GI_7_SLICE])
    parts = [[0, 3], [0, 1, 3], [0, 2, 3], [0, 1, 2, 3], [0, 0, 1, 3, 3], [0, 3, 3]]
    for cands in ([[0, 2]], [[2, 0]], [[0, 0, 2, 2]], [[1, 0, 2, 0]], [[5, 2, NONE, 0]]):
        ref = _check(g, off, t, c, np.array([0, 1], np.uint32), [9], rc, rpo, rpr, ro, cands, 0, 2, parts)
        assert ref[3][0] == P.EVICT and ref[2][0] == 2           # the later start wins: pod 2 on node 2


def test_invalid_search_limit_and_zero_row():
    g, off = R.make_inventory([1, 1], mig=True)
    t = R.default_table()
    rc, rpo, rpr, ro = mig_running([(0, 0, 1, R.GI_1_SLICE, 0), (1, 0, 8, R.GI_7_SLICE, 0)], off)
    g = occupied(g, rc, ro)
    c = np.concatenate([_mig(R, [R.GI_1_SLICE] * 7 + [R.GI_7_SLICE]),            # search limit on node 0, exhaustive
                        _mig(R, [R.GI_1_SLICE, 200]),                             # an invalid claim
                        _mig(R, [R.GI_1_SLICE] * 33),                             # more than 32 claims
                        _mig(R, [R.GI_7_SLICE])])
    pod_off = np.array([0, 8, 10, 43, 44], np.uint32)
    parts = [[0, 2], [0, 1, 2], [0, 0, 2], [0, 2, 2], [0, 1, 1, 2]]
    for flags in (0, P.F_EXHAUSTIVE):
        for mv in (0, 1, 4):
            ref = _check(g, off, t, c, pod_off, [5, 5, 5, 5], rc, rpo, rpr, ro, [[0], [0, 1, 7], [1, 0], [0, 1, 0]],
                         flags, mv, parts)
            assert list(ref[3][1:3]) == [P.INVALID, P.INVALID] and ref[3][3] == P.EVICT
            if flags:
                assert ref[3][0] == P.SEARCH_LIMIT
