"""CPU suite: spec §15 — preempt and place: the pods of a batch in input order, each judged as §14 judges it on the
inventory the pods before it left (their placements held, their victims gone), then applied.

The C oracle (tests/preempt_place_oracle.c, on tests/preempt_oracle.c's pair judgement and oracle/dra_oracle.c's pod
evaluation) and the Python restatement (preempt_place_oracle.preempt_place_naive: the host loop over
preempt_oracle.preempt_naive, §9 and oracle/naive.py's eval_pod) share no code, so agreement between them pins the rule."""
import importlib

import numpy as np
import pytest

from test_oracle_properties import _dicts
from test_pod_mode import _mig, _tbl
from test_preempt import _flat, _outs, _small_world, error_cases, mig_running, occupied

import place_oracle as PL
import preempt_oracle as P
import preempt_place_oracle as PP

R = importlib.import_module("k8s-dra-driver_b200").records
synth = importlib.import_module("k8s-dra-driver_b200").synth
NONE = 0xFFFFFFFF


def _inv(g):
    return [(int(x["busy"]), int(x["flags"]), int(x["mem_free_mib"]), int(x["share_cnt"])) for x in g]


def _inv_naive(gs):
    return [(x["busy"], x["flags"], x["mem_free_mib"], x["share_cnt"]) for x in gs]


def run_both(g, off, t, c, pod_off, prio, rc, rpo, rpr, ro, cands=None, flags=0, out_off=None):
    """the C oracle, checked against the naive host loop"""
    cn, co = (None, None) if cands is None else _flat(cands)
    a = PP.preempt_place(g, off, t, c, pod_off, prio, rc, rpo, rpr, ro, None, cn, co, out_off, None, flags)
    b = PP.preempt_place_naive(_dicts(g), [int(x) for x in off], _tbl(t), _dicts(c), [int(x) for x in pod_off],
                               [int(x) for x in prio], cands, bool(flags & PP.F_EXHAUSTIVE), _dicts(rc),
                               [int(x) for x in rpo], [int(x) for x in rpr], _outs(ro),
                               None if out_off is None else [int(x) for x in out_off])
    assert _outs(a[0]) == b[0]
    assert list(a[1]) == b[1] and list(a[2]) == b[2] and list(a[3]) == b[3]
    assert _inv(a[4]) == _inv_naive(b[4])
    return a


def _pods(*pods):
    """pods: lists of MIG profiles -> (claims, pod_off)"""
    c = _mig(R, [p for pod in pods for p in pod])
    off = np.zeros(len(pods) + 1, np.uint32)
    off[1:] = np.cumsum([len(p) for p in pods])
    return c, off


# ---- hand-written fixtures -----------------------------------------------------------------------------------------
def _two_nodes_one_hole():
    """Node 0: a 1g pod at slice 0 (prio 1) and a 3g pod at 4 (prio 100).  Node 1: 1g pods at 0 (prio 2) and 4 (prio 3).
    A 3g pod of priority 10 fits on node 0 once the prio-1 pod goes, on node 1 once the prio-2 pod goes; node 0 wins
    (lower highest victim priority)."""
    g, off = R.make_inventory([1, 1], mig=True)
    rc, rpo, rpr, ro = mig_running([(0, 0, 1, R.GI_1_SLICE, 1), (0, 4, 4, R.GI_3_SLICE, 100),
                                    (1, 0, 1, R.GI_1_SLICE, 2), (1, 4, 1, R.GI_1_SLICE, 3)], off)
    return occupied(g, rc, ro), off, R.default_table(), rc, rpo, rpr, ro


def test_two_pods_one_victim():
    """§14 sends both pods to node 0 to evict the same pod; §15 sends the second one to node 1, with its own victim."""
    g, off, t, rc, rpo, rpr, ro = _two_nodes_one_hole()
    c, po = _pods([R.GI_3_SLICE], [R.GI_3_SLICE])
    pre = P.preempt(g, off, t, c, po, [10, 10], rc, rpo, rpr, ro)
    assert list(pre[2]) == [0, 0] and list(pre[3]) == [P.EVICT, P.EVICT] and list(pre[5][:, 0]) == [0, 0]
    for flags in (0, PP.F_EXHAUSTIVE):
        out, node, st, ev, after = run_both(g, off, t, c, po, [10, 10], rc, rpo, rpr, ro, flags=flags)
        assert list(node) == [0, 1] and list(st) == [PP.EVICT, PP.EVICT] and list(ev) == [0, NONE, 1, NONE]
        assert _outs(out) == [(0, 0, 4, R.GI_3_SLICE, R.ST_OK), (1, 0, 4, R.GI_3_SLICE, R.ST_OK)]
        assert list(after["busy"]) == [0xFF, 0x1F]            # node 1: the prio-3 pod at slice 4 stays


def test_evicted_pod_is_not_counted_again_and_placed_pods_are_never_victims():
    """A 7g pod (prio 1) fills the GPU.  Pod 0 (1g, prio 10) evicts it and takes slice 0.  Pod 1 (7g, prio 20) then
    finds pod 0's 1g in the way: pod 0 is not a victim and the 7g pod is gone already, so there is nothing to evict."""
    g, off = R.make_inventory([1], mig=True)
    t = R.default_table()
    rc, rpo, rpr, ro = mig_running([(0, 0, 8, R.GI_7_SLICE, 1)], off)
    g = occupied(g, rc, ro)
    c, po = _pods([R.GI_1_SLICE], [R.GI_7_SLICE])
    out, node, st, ev, after = run_both(g, off, t, c, po, [10, 20], rc, rpo, rpr, ro)
    assert list(node) == [0, NONE] and list(st) == [PP.EVICT, PP.NO] and list(ev) == [0]
    assert _outs(out) == [(0, 0, 1, R.GI_1_SLICE, R.ST_OK), (NONE, 0, 0, R.GI_7_SLICE, R.ST_POD)]
    assert int(after["busy"][0]) == 0x1


def test_fits_anywhere_beats_evict():
    """Node 0 (listed first) needs an eviction, node 1 fits as it is: node 1, nothing evicted."""
    g, off, t, rc, rpo, rpr, ro = _two_nodes_one_hole()
    g2, off2 = R.make_inventory([1, 1, 1], mig=True)
    g2[:2] = g
    c, po = _pods([R.GI_3_SLICE])
    out, node, st, ev, after = run_both(g2, off2, t, c, po, [10], rc, rpo, rpr, ro, cands=[[0, 1, 2]])
    assert list(node) == [2] and list(st) == [PP.FITS] and list(ev) == [NONE] * 4


def test_equal_priority_is_not_evictable():
    g, off = R.make_inventory([1], mig=True)
    t = R.default_table()
    rc, rpo, rpr, ro = mig_running([(0, 0, 8, R.GI_7_SLICE, 10)], off)
    g = occupied(g, rc, ro)
    c, po = _pods([R.GI_1_SLICE])
    out, node, st, ev, after = run_both(g, off, t, c, po, [10], rc, rpo, rpr, ro)
    assert list(st) == [PP.NO] and list(ev) == [NONE] and _outs(out) == [(NONE, 0, 0, R.GI_1_SLICE, R.ST_POD)]
    assert _inv(after) == _inv(g)


def test_empty_pod_invalid_claims_and_33_claims():
    """An empty pod is FITS on its first candidate naming a node and writes nothing; a pod with an invalid claim is
    INVALID (that claim INVALID, the other POD); a pod of 33 claims is INVALID in every slot."""
    g, off = R.make_inventory([1], mig=True)
    t = R.default_table()
    rc, rpo, rpr, ro = mig_running([(0, 0, 8, R.GI_7_SLICE, 0)], off)
    g = occupied(g, rc, ro)
    c = _mig(R, [R.GI_1_SLICE, 200] + [R.GI_1_SLICE] * 33)
    po = np.array([0, 2, 2, 2, 35], np.uint32)
    out, node, st, ev, after = run_both(g, off, t, c, po, [5, 5, 5, 5], rc, rpo, rpr, ro, cands=[[0], [4, 0], [4], [0]])
    assert list(st) == [PP.INVALID, PP.FITS, PP.NO, PP.INVALID] and list(node) == [NONE, 0, NONE, NONE]
    assert list(out["status"][:2]) == [R.ST_POD, R.ST_INVALID] and (out["status"][2:] == R.ST_INVALID).all()
    assert list(ev) == [NONE] and _inv(after) == _inv(g)


def test_node_listed_twice():
    """The same node twice after a stray: judged once per entry on the same state, applied once."""
    g, off = R.make_inventory([1], mig=True)
    t = R.default_table()
    rc, rpo, rpr, ro = mig_running([(0, 0, 8, R.GI_7_SLICE, 5)], off)
    g = occupied(g, rc, ro)
    c, po = _pods([R.GI_7_SLICE], [R.GI_1_SLICE])
    out, node, st, ev, after = run_both(g, off, t, c, po, [9, 9], rc, rpo, rpr, ro, cands=[[3, 0, 0], [0, 0]])
    assert list(node) == [0, NONE] and list(st) == [PP.EVICT, PP.NO] and list(ev) == [0]
    assert _outs(out)[0] == (0, 0, 8, R.GI_7_SLICE, R.ST_OK)


def test_search_limit():
    """7 x 1g + 7g on a one-GPU node with a lower-priority 1g pod in the way: with it removed the search runs out of
    budget, so the pod is SEARCH_LIMIT and its slots too."""
    g, off = R.make_inventory([1], mig=True)
    t = R.default_table()
    rc, rpo, rpr, ro = mig_running([(0, 0, 1, R.GI_1_SLICE, 0)], off)
    g = occupied(g, rc, ro)
    c, po = _pods([R.GI_1_SLICE] * 7 + [R.GI_7_SLICE])
    out, node, st, ev, after = PP.preempt_place(g, off, t, c, po, [5], rc, rpo, rpr, ro, flags=PP.F_EXHAUSTIVE)
    assert list(st) == [PP.SEARCH_LIMIT] and (out["status"] == R.ST_SEARCH_LIMIT).all() and list(ev) == [NONE]
    out, node, st, ev, after = PP.preempt_place(g, off, t, c, po, [5], rc, rpo, rpr, ro)
    assert list(st) == [PP.NO] and (out["status"] == R.ST_POD).all()


def test_call_errors():
    g, off = R.make_inventory([1, 1], mig=True)
    t = R.default_table()
    ok, cases = error_cases(g, off)
    cases = [x for x in cases if "fl" not in x[1]] + [("unknown flags", dict(fl=0x1)), ("unknown flags", dict(fl=0x8)),
                                                      ("slot outside n_out", dict(oo=np.array([3], np.uint32)))]

    def call(a):
        return PP.preempt_place(g, off, t, a["c"], a["po"], a["prio"], a["rc"], a["rpo"], a["rpr"], a["ro"], a["roo"],
                                a["cn"], a["co"], a.get("oo"), 1, a["fl"])
    call(ok)
    for name, kw in cases:
        with pytest.raises(ValueError):
            call(dict(ok, **kw))
            pytest.fail(name)
    # no pending pods: the running pods are not examined
    bad = dict(ok, c=np.zeros(0, R.CLAIM_DTYPE), po=np.zeros(1, np.uint32), prio=[], rpo=np.array([0, 2, 1], np.uint32))
    PP.preempt_place(g, off, t, bad["c"], bad["po"], bad["prio"], bad["rc"], bad["rpo"], bad["rpr"], bad["ro"])


def test_dense_form_over_two_to_the_32_pairs():
    n = 1 << 16
    g, off = R.make_inventory([1] * n, mig=True)
    with pytest.raises(ValueError):
        PP.preempt_place(g, off, R.default_table(), np.zeros(0, R.CLAIM_DTYPE), np.zeros(n + 1, np.uint32),
                         np.zeros(n, np.int32), np.zeros(0, R.CLAIM_DTYPE), np.zeros(1, np.uint32), np.zeros(0, np.int32),
                         np.zeros(0, R.OUT_DTYPE))


# ---- the C oracle against the naive host loop ----------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(120))
def test_oracle_agrees_with_naive(seed):
    w, c, po, prio, cands = _small_world(seed)
    n_node = len(w.node_off) - 1
    rng = np.random.default_rng(1000 + seed)
    if cands is None:
        cands = [list(rng.integers(0, n_node + 2, size=int(rng.integers(0, 5)))) for _ in range(len(po) - 1)]
    out_off = None
    if seed % 2:                                     # out_off given: GPU claims of count > 1 are valid
        sl = [int(x["count"]) if x["kind"] == R.KIND_GPU and 1 <= x["count"] <= 32 else 1 for x in c]
        out_off = np.concatenate([[0], np.cumsum(sl)[:-1]]).astype(np.uint32) if len(sl) else np.zeros(0, np.uint32)
    for flags in (0, PP.F_EXHAUSTIVE):
        for form in (None, cands):
            run_both(w.gpus, w.node_off, w.table, c, po, prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out,
                     cands=form, flags=flags, out_off=out_off)


# ---- properties on seeded synth.preempt worlds ----------------------------------------------------------------------
def _world(seed, **kw):
    w = synth.preempt(n_node=10, gpus_per_node=4 + 4 * (seed % 2), n_pending=40, seed=seed, **kw)
    oo, n_out = R.out_offsets(w.claims, len(w.node_off) - 1)
    return w, oo, n_out


def _host_loop(w, oracle, oo, n_out, flags, cands=None):
    """per pod: §14 with that one pod and the running pods not evicted yet, §9 for its victims, §12 on the chosen node"""
    n_node, n_run = len(w.node_off) - 1, len(w.run_pod_off) - 1
    g = w.gpus.copy()
    out = np.zeros(n_out, R.OUT_DTYPE)
    ev = np.full(n_run, NONE, np.uint32)
    node, st = [], []
    for p in range(len(w.pod_off) - 1):
        c0, c1 = int(w.pod_off[p]), int(w.pod_off[p + 1])
        alive = np.flatnonzero(ev == NONE)
        keep = np.zeros(len(w.run_claims), bool)
        for r in alive:
            keep[w.run_pod_off[r]: w.run_pod_off[r + 1]] = True
        rpo = np.concatenate([[0], np.cumsum(w.run_pod_off[alive + 1] - w.run_pod_off[alive])]).astype(np.uint32)
        cn, co = (None, None) if cands is None else _flat([cands[p]])
        _, _, pn, ps, nv, vic = P.preempt(g, w.node_off, w.table, w.claims[c0:c1], np.array([0, c1 - c0], np.uint32),
                                          w.prio[p:p + 1], w.run_claims[keep], rpo, w.run_prio[alive], w.run_out[keep],
                                          cand_nodes=cn, cand_off=co, max_victims=max(len(alive), 1), flags=flags)
        node.append(int(pn[0])); st.append(int(ps[0]))
        victims = alive[vic[0][: nv[0]]]
        ev[victims] = p
        vk = np.zeros(len(w.run_claims), bool)
        for r in victims:
            vk[w.run_pod_off[r]: w.run_pod_off[r + 1]] = True
        if vk.any():
            g = oracle.deallocate(g, w.run_claims[vk], w.run_out[vk], n_node=n_node)
        pod = w.claims[c0:c1].copy()
        if pn[0] != NONE:
            if c1 > c0:
                pod["node"] = pn[0]
                po_, g = oracle.allocate_pods(g, w.node_off, w.table, pod, np.array([0, c1 - c0], np.uint32),
                                              oo[c0:c1] - oo[c0], n_out - int(oo[c0]), flags=flags)
                for i in range(c0, c1):
                    n = int(R.claim_slots(pod[i - c0: i - c0 + 1], n_node)[0])
                    out[oo[i]: oo[i] + n] = po_[oo[i] - oo[c0]: oo[i] - oo[c0] + n]
        else:
            for i in range(c0, c1):
                placed = w.claims[i: i + 1].copy(); placed["node"] = 0
                n = int(R.claim_slots(placed, 1)[0])
                out[oo[i]: oo[i] + n] = (NONE, 0, 0, R.PROFILE_GPU if placed["kind"][0] == R.KIND_GPU else
                                         R.PROFILE_SHARED if placed["kind"][0] == R.KIND_SHARED else placed["profile"][0],
                                         R.ST_SEARCH_LIMIT if ps[0] == P.SEARCH_LIMIT else R.ST_POD)
    return out, np.array(node, np.uint32), np.array(st, np.uint8), ev, g


@pytest.mark.parametrize("seed", range(4))
def test_host_loop_equivalence(seed, oracle):
    w, oo, n_out = _world(seed)
    n_node = len(w.node_off) - 1
    rng = np.random.default_rng(seed)
    cands = [list(rng.permutation(n_node)[: int(rng.integers(1, n_node + 1))]) for _ in range(len(w.pod_off) - 1)]
    for flags in (0, PP.F_EXHAUSTIVE):
        for form in (None, cands):
            cn, co = (None, None) if form is None else _flat(form)
            a = PP.preempt_place(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off,
                                 w.run_prio, w.run_out, None, cn, co, oo, n_out, flags)
            b = _host_loop(w, oracle, oo, n_out, flags, form)
            assert a[0].tobytes() == b[0].tobytes()
            assert list(a[1]) == list(b[1]) and list(a[2]) == list(b[2]) and list(a[3]) == list(b[3])
            assert a[4].tobytes() == b[4].tobytes()
            assert (a[2] == PP.EVICT).any()


@pytest.mark.parametrize("seed", range(4))
def test_place_pods_equivalence_when_nothing_is_evictable(seed):
    w, oo, n_out = _world(seed, prio_lo=100, prio_hi=200, pending_prio=100)
    for flags in (0, PP.F_EXHAUSTIVE):
        out, node, st, ev, after = PP.preempt_place(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims,
                                                    w.run_pod_off, w.run_prio, w.run_out, None, None, None, oo, n_out, flags)
        pout, pnode, pafter = PL.place_pods(w.gpus, w.node_off, w.table, w.claims, w.pod_off, None, None, oo, n_out, flags)
        assert out.tobytes() == pout.tobytes() and after.tobytes() == pafter.tobytes()
        nonempty = np.diff(w.pod_off) > 0
        assert (node[nonempty] == pnode[nonempty]).all() and (ev == NONE).all()


def _apply(g, claims, out, have_off, oo, add):
    """the Allocate updates (add) or §9 for OK slots, in numpy"""
    g = g.copy()
    for i, c in enumerate(claims):
        n = int(c["count"]) if c["kind"] == R.KIND_GPU and 1 <= c["count"] <= 32 and have_off else 1
        base = int(oo[i]) if have_off else i
        for o in out[base: base + n]:
            if o["status"] != R.ST_OK:
                continue
            x = g[o["gpu"]]
            if c["kind"] == R.KIND_GPU:
                f = int(x["flags"])
                x["flags"] = (f | R.GPU_FULL_ALLOCATED) if add else (f & ~R.GPU_FULL_ALLOCATED & 0xFF)
            elif c["kind"] == R.KIND_MIG:
                m = (((1 << int(o["size"])) - 1) << int(o["start"])) & 0xFFFF
                x["busy"] = (int(x["busy"]) | m) if add else (int(x["busy"]) & ~m)
            else:
                x["mem_free_mib"] = (int(x["mem_free_mib"]) + (-1 if add else 1) * int(c["mem_limit_mib"])) % (1 << 32)
                x["share_cnt"] = (int(x["share_cnt"]) + (1 if add else -1)) % (1 << 16)
            g[o["gpu"]] = x
    return g


@pytest.mark.parametrize("seed", range(4))
def test_properties(seed):
    w, oo, n_out = _world(seed)
    n_node = len(w.node_off) - 1
    node_of = np.searchsorted(w.node_off, np.arange(len(w.gpus)), side="right") - 1
    for flags in (0, PP.F_EXHAUSTIVE):
        out, node, st, ev, after = PP.preempt_place(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims,
                                                    w.run_pod_off, w.run_prio, w.run_out, None, None, None, oo, n_out, flags)
        assert (st == PP.EVICT).any()
        # every victim is on its evictor's node, at a lower priority
        for r in np.flatnonzero(ev != NONE):
            p = ev[r]
            assert st[p] == PP.EVICT and w.run_prio[r] < w.prio[p]
            gpus = w.run_out["gpu"][w.run_pod_off[r]: w.run_pod_off[r + 1]][w.run_out["status"][w.run_pod_off[r]: w.run_pod_off[r + 1]] == R.ST_OK]
            assert (node_of[gpus] == node[p]).all()
        # final inventory = initial, with §9 for the victims and the Allocate updates for the OutRecs (they commute)
        vk = np.zeros(len(w.run_claims), bool)
        for r in np.flatnonzero(ev != NONE):
            vk[w.run_pod_off[r]: w.run_pod_off[r + 1]] = True
        g = _apply(w.gpus, w.run_claims[vk], w.run_out[vk], False, None, False)
        g = _apply(g, w.claims, out, True, oo, True)
        assert g.tobytes() == after.tobytes()
        # no two MIG placements overlap: the placed pods' and the running pods that stay
        used = {}
        keep = ~vk
        recs = [(o, c) for c, o in zip(w.run_claims[keep], w.run_out[keep])]
        recs += [(out[oo[i]], w.claims[i]) for i in range(len(w.claims)) if w.claims[i]["kind"] == R.KIND_MIG]
        for o, c in recs:
            if c["kind"] != R.KIND_MIG or o["status"] != R.ST_OK:
                continue
            m = (((1 << int(o["size"])) - 1) << int(o["start"])) & 0xFFFF
            assert used.get(int(o["gpu"]), 0) & m == 0
            used[int(o["gpu"])] = used.get(int(o["gpu"]), 0) | m
        assert all(node[p] < n_node for p in np.flatnonzero(st <= PP.EVICT))
