"""CPU suite: spec §14 with disruption budgets — V's members whose eviction would take their budget below zero are
reprieved first, and the pod's EVICT pair is the one with the fewest such victims before any other key.

The C oracle (pod_oracle_preempt in tests/pod_oracles.c, budgets in the "members of V up to v" form) and the naive
restatement (preempt_oracle.preempt_naive_pdb, kube-scheduler's decrement-then-below-zero loop) share no code, so
agreement between them pins the rule."""
import importlib

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from preempt_problems import I32_MAX, I32_MIN, _Hyp, build
from test_oracle_properties import _dicts
from test_pod_mode import _mig, _tbl
from test_preempt import _flat, _outs, _small_world, mig_running, occupied

import preempt_oracle as P
import preempt_oracle as PB

R = importlib.import_module("k8s-dra-driver_b200").records
NONE = 0xFFFFFFFF
ALLOWED = (I32_MIN, -1, 0, 1, 2, I32_MAX)


def run_both(g, off, t, c, pod_off, prio, rc, rpo, rpr, ro, run_pdb, allowed, cands=None, flags=0, max_victims=8,
             run_out_off=None):
    """both oracles with budgets; they must agree in all eight outputs"""
    cn, co = (None, None) if cands is None else _flat(cands)
    a = PB.preempt_pdb(g, off, t, c, pod_off, prio, rc, rpo, rpr, ro, run_pdb, allowed, run_out_off, cn, co, max_victims,
                      flags)
    b = PB.preempt_naive_pdb(_dicts(g), list(off), _tbl(t), _dicts(c), list(pod_off), list(prio), cands,
                            bool(flags & P.F_EXHAUSTIVE), _dicts(rc), list(rpo), list(rpr), _outs(ro), run_pdb, allowed,
                            None if run_out_off is None else [int(x) for x in run_out_off], max_victims)
    for i in (0, 1, 2, 3, 4, 6, 7):
        assert [int(x) for x in a[i]] == b[i], i
    assert a[5].tolist() == [list(r) for r in b[5]]
    return a


# ---- hand-written fixtures -----------------------------------------------------------------------------------------
def _two_nodes():
    """Node 0 holds one 7g pod of priority 1; node 1 two 3g pods of priority 5.  A 7g pod of priority 10 needs node 0's
    one pod or node 1's two gone."""
    g, off = R.make_inventory([1, 1], mig=True)
    rc, rpo, rpr, ro = mig_running([(0, 0, 8, R.GI_7_SLICE, 1), (1, 0, 4, R.GI_3_SLICE, 5), (1, 4, 4, R.GI_3_SLICE, 5)], off)
    return occupied(g, rc, ro), off, R.default_table(), rc, rpo, rpr, ro


def test_a_pair_with_violations_loses_to_one_without():
    g, off, t, rc, rpo, rpr, ro = _two_nodes()
    c, po = _mig(R, [R.GI_7_SLICE]), np.array([0, 1], np.uint32)
    free = run_both(g, off, t, c, po, [10], rc, rpo, rpr, ro, None, None, cands=[[0, 1]])
    assert list(free[2]) == [0] and list(free[4]) == [1]           # without budgets: the lower victim priority wins
    got = run_both(g, off, t, c, po, [10], rc, rpo, rpr, ro, [0, NONE, NONE], [0], cands=[[0, 1]])
    assert list(got[0]) == [P.EVICT, P.EVICT] and list(got[6]) == [1, 0]
    assert list(got[2]) == [1] and list(got[4]) == [2] and list(got[5][0][:3]) == [1, 2, NONE] and list(got[7]) == [0]


def _one_node_two_3g(p0=5, p1=4):
    g, off = R.make_inventory([1], mig=True)
    rc, rpo, rpr, ro = mig_running([(0, 0, 4, R.GI_3_SLICE, p0), (0, 4, 4, R.GI_3_SLICE, p1)], off)
    return occupied(g, rc, ro), off, R.default_table(), rc, rpo, rpr, ro


def test_a_violating_member_is_tried_first_and_stays():
    """V = (pod 0, pod 1); a 3g pod needs one of them gone.  Without budgets pod 0 is reprieved first and pod 1 goes.
    With pod 1 under a budget that allows nothing, pod 1 is tried first and stays, so pod 0 goes."""
    g, off, t, rc, rpo, rpr, ro = _one_node_two_3g()
    c, po = _mig(R, [R.GI_3_SLICE]), np.array([0, 1], np.uint32)
    free = run_both(g, off, t, c, po, [10], rc, rpo, rpr, ro, None, None)
    assert list(free[5][0][:2]) == [1, NONE]
    got = run_both(g, off, t, c, po, [10], rc, rpo, rpr, ro, [NONE, 0], [0])
    assert list(got[3]) == [P.EVICT] and list(got[5][0][:2]) == [0, NONE] and list(got[7]) == [0]


@pytest.mark.parametrize("allowed, viol", [(I32_MIN, 2), (-1, 2), (0, 2), (1, 1), (2, 0), (I32_MAX, 0)])
def test_allowed_counts_the_members_in_v_order(allowed, viol):
    """Both 3g pods must go for a 7g pod and both count against one budget: the first is violating only when the budget
    allows nothing, the second when it allows fewer than two."""
    g, off, t, rc, rpo, rpr, ro = _one_node_two_3g()
    got = run_both(g, off, t, _mig(R, [R.GI_7_SLICE]), np.array([0, 1], np.uint32), [10], rc, rpo, rpr, ro, [0, 0],
                   [allowed])
    assert list(got[4]) == [2] and list(got[6]) == [viol] and list(got[7]) == [viol]


def test_budget_counts_members_before_the_reprieve():
    """Pod 0 (3g, slices 0-3) and pod 1 (2g, slices 4-5) share a budget that allows one eviction; pod 2 (2g, slices 6-7)
    has none.  A 3g pod needs slices 0-3 or 4-7.  Pod 1 is violating because pod 0 before it counts, so pod 1 is tried
    first and stays, then pod 0 goes and pod 2 stays: one victim where the budget-free answer has two."""
    g, off = R.make_inventory([1], mig=True)
    rc, rpo, rpr, ro = mig_running([(0, 0, 4, R.GI_3_SLICE, 6), (0, 4, 2, R.GI_2_SLICE, 5), (0, 6, 2, R.GI_2_SLICE, 4)], off)
    g, t = occupied(g, rc, ro), R.default_table()
    c, po = _mig(R, [R.GI_3_SLICE]), np.array([0, 1], np.uint32)
    free = run_both(g, off, t, c, po, [10], rc, rpo, rpr, ro, None, None, max_victims=3)
    assert free[5][0].tolist() == [1, 2, NONE]
    got = run_both(g, off, t, c, po, [10], rc, rpo, rpr, ro, [0, 0, NONE], [1], max_victims=3)
    assert got[5][0].tolist() == [0, NONE, NONE] and list(got[7]) == [0]


@pytest.mark.parametrize("allowed", [0, 1])
def test_a_budget_spanning_two_nodes_starts_full_on_each_pair(allowed):
    """Each node holds one 7g pod of the same budget.  Every pair copies the budget afresh, so with one eviction allowed
    neither pair violates it, and with none both do."""
    g, off = R.make_inventory([1, 1], mig=True)
    rc, rpo, rpr, ro = mig_running([(0, 0, 8, R.GI_7_SLICE, 5), (1, 0, 8, R.GI_7_SLICE, 5)], off)
    g, t = occupied(g, rc, ro), R.default_table()
    got = run_both(g, off, t, _mig(R, [R.GI_7_SLICE]), np.array([0, 1], np.uint32), [9], rc, rpo, rpr, ro, [0, 0],
                   [allowed], cands=[[0, 1]])
    assert list(got[6]) == [1 - allowed] * 2 and list(got[7]) == [1 - allowed] and list(got[2]) == [1]


@pytest.mark.parametrize("seed", range(12))
def test_no_budgets_is_preempt_byte_for_byte(seed):
    w, c, po, prio, cands = _small_world(seed)
    cn, co = (None, None) if cands is None else _flat(cands)
    args = (w.gpus, w.node_off, w.table, c, po, prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out)
    n_run = len(w.run_prio)
    for flags in (0, P.F_EXHAUSTIVE):
        ref = P.preempt(*args, None, cn, co, 4, flags)
        for run_pdb, allowed in ((None, None), ([NONE] * n_run, None), ([NONE] * n_run, []), ([NONE] * n_run, [0, -1])):
            got = PB.preempt_pdb(*args, run_pdb, allowed, None, cn, co, 4, flags)
            for x, y in zip(got[:6], ref):
                assert x.tobytes() == y.tobytes()
            assert not got[6].any() and not got[7].any()


def test_call_level_errors():
    g, off, t, rc, rpo, rpr, ro = _one_node_two_3g()
    c, po = _mig(R, [R.GI_7_SLICE]), np.array([0, 1], np.uint32)
    args = (g, off, t, c, po, [10], rc, rpo, rpr, ro)
    for run_pdb, allowed, n_pdb in (([0, 1], [0], None),            # a budget index >= n_pdb
                                    ([NONE, 0], [], None),          # any index with no budgets
                                    ([0, NONE], None, 1),           # n_pdb > 0 without allowed
                                    (None, [0], None)):             # running pods and budgets without run_pdb
        with pytest.raises(ValueError):
            PB.preempt_pdb(*args, run_pdb, allowed, n_pdb=n_pdb)
    # no pending pods: the running pods, run_pdb with them, are not examined; the budget arguments themselves are
    none = (g, off, t, c[:0], np.array([0], np.uint32), [], rc, rpo, rpr, ro)
    assert len(PB.preempt_pdb(*none, [0, 1], [0])[3]) == 0
    assert len(PB.preempt_pdb(*none, None, [0])[3]) == 0
    with pytest.raises(ValueError):
        PB.preempt_pdb(*none, [0, 0], None, n_pdb=1)


# ---- random problems -----------------------------------------------------------------------------------------------
def draw_budgets(D, n_run):
    """(run_pdb, allowed): up to four budgets, allowed at the int32 ends and around zero, NONE mixed in; now and then
    one budget for most running pods, so that it spans nodes and holds many members of one node"""
    n_pdb = D.pick((0, 1, 1, 2, 3, 4))
    allowed = [D.pick(ALLOWED) for _ in range(n_pdb)]
    if not n_pdb:
        return ([NONE] * n_run if D.int(0, 1) else None), allowed
    crowd = D.int(0, 2) == 0
    run_pdb = [(0 if D.int(0, 5) else NONE) if crowd else D.pick(list(range(n_pdb)) + [NONE]) for _ in range(n_run)]
    return run_pdb, allowed


@st.composite
def pdb_problems(draw):
    D = _Hyp(draw)
    pb = build(D)
    return pb, *draw_budgets(D, len(pb.run_prio))


@settings(max_examples=200, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True)
@given(pdb_problems())
def test_oracle_agrees_with_naive_on_random_problems(x):
    pb, run_pdb, allowed = x
    cn, co = pb.cand_arrays()
    try:
        a = PB.preempt_pdb(pb.gpus, pb.node_off, pb.table, pb.claims, pb.pod_off, pb.prio, pb.run_claims, pb.run_pod_off,
                          pb.run_prio, pb.run_out, run_pdb, allowed, pb.run_out_off, cn, co, pb.max_victims, pb.flags)
    except ValueError:
        assert pb.error, pb.what
        return
    assert not pb.error, pb.what
    b = PB.preempt_naive_pdb(_dicts(pb.gpus), list(pb.node_off), _tbl(pb.table), _dicts(pb.claims), list(pb.pod_off),
                            list(pb.prio), pb.cands, bool(pb.flags & P.F_EXHAUSTIVE), _dicts(pb.run_claims),
                            list(pb.run_pod_off), list(pb.run_prio), _outs(pb.run_out), run_pdb, allowed,
                            None if pb.run_out_off is None else [int(v) for v in pb.run_out_off], pb.max_victims)
    for i in (0, 1, 2, 3, 4, 6, 7):
        assert [int(v) for v in a[i]] == b[i], (i, pb.what)
    assert a[5].tolist() == [list(r) for r in b[5]], pb.what
    pst, pvi, pviol = a[0], a[1], a[6]
    assert ((pviol <= pvi) & ((pst == P.EVICT) | (pviol == 0))).all()
