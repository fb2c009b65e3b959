"""CPU suite: spec §14 — preemption: for a pod that fits nowhere, the lower-priority running pods to evict on each
candidate node, and the node to evict them on (kube-scheduler's DefaultPreemption without PodDisruptionBudgets).

The C oracle (pod_oracle_preempt in tests/pod_oracles.c, on oracle/dra_oracle.c's pod evaluation) and the pure-Python
restatement (preempt_oracle.preempt_naive, on oracle/naive.py's) share no code, so agreement between them pins the
rule."""
import importlib

import numpy as np
import pytest

from test_oracle_properties import _dicts
from test_pod_mode import _mig, _tbl

import preempt_oracle as P

R = importlib.import_module("k8s-dra-driver_b200").records
synth = importlib.import_module("k8s-dra-driver_b200").synth
NONE = 0xFFFFFFFF
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1


def _flat(cands):
    off = np.zeros(len(cands) + 1, np.uint32)
    off[1:] = np.cumsum([len(x) for x in cands])
    return np.array([n for x in cands for n in x], dtype=np.uint32), off


def _outs(recs):
    return [tuple(int(o[k]) for k in ("gpu", "start", "size", "profile", "status")) for o in recs]


def mig_running(pods, node_off):
    """pods: [(gpu, start, size, profile, prio)] one MIG claim each.  Returns (gpus-independent) running arrays."""
    c = np.zeros(len(pods), R.CLAIM_DTYPE)
    o = np.zeros(len(pods), R.OUT_DTYPE)
    for i, (gpu, s, size, prof, _) in enumerate(pods):
        c[i]["kind"], c[i]["profile"], c[i]["count"] = R.KIND_MIG, prof, 1
        c[i]["node"] = int(np.searchsorted(node_off, gpu, side="right") - 1)
        o[i]["gpu"], o[i]["start"], o[i]["size"], o[i]["profile"], o[i]["status"] = gpu, s, size, prof, R.ST_OK
    return c, np.arange(len(pods) + 1, dtype=np.uint32), np.array([p[4] for p in pods], np.int32), o


def occupied(g, run_c, run_o):
    g = g.copy()
    for c, o in zip(run_c, run_o):
        if o["status"] == R.ST_OK and c["kind"] == R.KIND_MIG:
            g["busy"][o["gpu"]] |= ((1 << int(o["size"])) - 1) << int(o["start"])
    return g


def run_both(g, off, t, c, pod_off, prio, rc, rpo, rpr, ro, cands=None, flags=0, max_victims=8):
    cn, co = (None, None) if cands is None else _flat(cands)
    a = P.preempt(g, off, t, c, pod_off, prio, rc, rpo, rpr, ro, None, cn, co, max_victims, flags)
    b = P.preempt_naive(_dicts(g), list(off), _tbl(t), _dicts(c), list(pod_off), list(prio), cands,
                        bool(flags & P.F_EXHAUSTIVE), _dicts(rc), list(rpo), list(rpr), _outs(ro), None, max_victims)
    assert list(a[0]) == b[0] and list(a[1]) == b[1] and list(a[2]) == b[2]
    assert list(a[3]) == b[3] and list(a[4]) == b[4] and a[5].tolist() == [list(r) for r in b[5]]
    return a


# ---- hand-written fixtures -----------------------------------------------------------------------------------------
def test_seven_slivers_four_victims():
    """Seven 1g pods at slices 0..6 with priorities 1..7; a 3g pod (4 slices, starts 0 or 4) at priority 10.  Removing
    all seven makes room; the reprieve keeps 7, 6, 5 (slices 6, 5, 4) and evicts 4, 3, 2, 1 (slices 3..0)."""
    g, off = R.make_inventory([1], mig=True)
    t = R.default_table()
    rc, rpo, rpr, ro = mig_running([(0, s, 1, R.GI_1_SLICE, s + 1) for s in range(7)], off)
    g = occupied(g, rc, ro)
    c = _mig(R, [R.GI_3_SLICE])
    for flags in (0, P.F_EXHAUSTIVE):
        st, pv, node, pst, nv, vic = run_both(g, off, t, c, np.array([0, 1], np.uint32), [10], rc, rpo, rpr, ro, flags=flags)
        assert list(st) == [P.EVICT] and list(pv) == [4] and list(node) == [0] and list(pst) == [P.EVICT]
        assert list(nv) == [4] and list(vic[0]) == [3, 2, 1, 0, NONE, NONE, NONE, NONE]


def test_equal_priority_never_evicts():
    g, off = R.make_inventory([1], mig=True)
    t = R.default_table()
    rc, rpo, rpr, ro = mig_running([(0, 0, 8, R.GI_7_SLICE, 10)], off)
    g = occupied(g, rc, ro)
    st, pv, node, pst, nv, vic = run_both(g, off, t, _mig(R, [R.GI_1_SLICE]), np.array([0, 1], np.uint32), [10],
                                          rc, rpo, rpr, ro)
    assert list(st) == [P.NO] and list(pst) == [P.NO] and list(node) == [NONE] and list(nv) == [0]
    st, *_ = run_both(g, off, t, _mig(R, [R.GI_1_SLICE]), np.array([0, 1], np.uint32), [11], rc, rpo, rpr, ro)
    assert list(st) == [P.EVICT]


@pytest.mark.parametrize("which", ["highest", "sum", "count", "latest"])
def test_tie_breaks(which):
    """Two one-GPU nodes, a 7g pod at priority 100; each criterion alone decides between them (node 1 wins)."""
    g, off = R.make_inventory([1, 1], mig=True)
    t = R.default_table()
    # node 0's and node 1's running pods: (start, size, profile, prio); node 0's come first in index order
    a, b = {
        "highest": ([(0, 8, R.GI_7_SLICE, 5)], [(0, 8, R.GI_7_SLICE, 4)]),
        "sum": ([(0, 4, R.GI_3_SLICE, 5), (4, 4, R.GI_3_SLICE, 5)], [(0, 4, R.GI_3_SLICE, 5), (4, 4, R.GI_3_SLICE, 1)]),
        "count": ([(0, 4, R.GI_3_SLICE, 5), (4, 4, R.GI_3_SLICE, I32_MIN)], [(0, 8, R.GI_7_SLICE, 5)]),
        "latest": ([(0, 8, R.GI_7_SLICE, 5)], [(0, 8, R.GI_7_SLICE, 5)]),
    }[which]
    rc, rpo, rpr, ro = mig_running([(0, s, z, p, q) for s, z, p, q in a] + [(1, s, z, p, q) for s, z, p, q in b], off)
    g = occupied(g, rc, ro)
    st, pv, node, pst, nv, vic = run_both(g, off, t, _mig(R, [R.GI_7_SLICE]), np.array([0, 1], np.uint32), [100],
                                          rc, rpo, rpr, ro, cands=[[0, 1]])
    assert list(st) == [P.EVICT, P.EVICT] and list(node) == [1] and list(pst) == [P.EVICT]


def test_tie_break_position():
    """Equal in every other criterion: the earlier candidate wins (here one node listed twice, after a stray)."""
    g, off = R.make_inventory([1], mig=True)
    t = R.default_table()
    rc, rpo, rpr, ro = mig_running([(0, 0, 8, R.GI_7_SLICE, 5)], off)
    g = occupied(g, rc, ro)
    st, pv, node, pst, nv, vic = run_both(g, off, t, _mig(R, [R.GI_7_SLICE]), np.array([0, 1], np.uint32), [9],
                                          rc, rpo, rpr, ro, cands=[[3, 0, 0]])
    assert list(st) == [P.NO, P.EVICT, P.EVICT] and list(node) == [0] and list(vic[0][:2]) == [0, NONE]


def test_int32_extremes():
    g, off = R.make_inventory([1, 1], mig=True)
    t = R.default_table()
    rc, rpo, rpr, ro = mig_running([(0, 0, 4, R.GI_3_SLICE, I32_MIN), (0, 4, 4, R.GI_3_SLICE, I32_MIN),
                                    (1, 0, 8, R.GI_7_SLICE, I32_MAX - 1)], off)
    g = occupied(g, rc, ro)
    st, pv, node, pst, nv, vic = run_both(g, off, t, _mig(R, [R.GI_7_SLICE]), np.array([0, 1], np.uint32), [I32_MAX],
                                          rc, rpo, rpr, ro)
    assert list(st) == [P.EVICT, P.EVICT] and list(node) == [0] and list(vic[0][:2]) == [0, 1]
    st, *_ = run_both(g, off, t, _mig(R, [R.GI_7_SLICE]), np.array([0, 1], np.uint32), [I32_MIN], rc, rpo, rpr, ro)
    assert list(st) == [P.NO, P.NO]


def test_exhaustive_only():
    """The order dependence of spec §12: {1g, 3g} on a GPU with slice 4 held (by a pod of priority 20) fits only with the
    search (3g at 0, 1g at 5).  A pod of priority 0 at slice 0 has to go first; in order, 1g takes slice 0 and 3g fails."""
    g, off = R.make_inventory([1], mig=True)
    t = R.default_table()
    rc, rpo, rpr, ro = mig_running([(0, 0, 1, R.GI_1_SLICE, 0), (0, 4, 1, R.GI_1_SLICE, 20)], off)
    g = occupied(g, rc, ro)
    c = _mig(R, [R.GI_1_SLICE, R.GI_3_SLICE])
    st, pv, node, pst, nv, vic = run_both(g, off, t, c, np.array([0, 2], np.uint32), [10], rc, rpo, rpr, ro,
                                          flags=P.F_EXHAUSTIVE)
    assert list(pst) == [P.EVICT] and list(node) == [0] and list(vic[0][:2]) == [0, NONE]
    st, pv, node, pst, nv, vic = run_both(g, off, t, c, np.array([0, 2], np.uint32), [10], rc, rpo, rpr, ro)
    assert list(pst) == [P.NO]


def test_search_limit():
    """The search-limit shape of the exhaustive search: 7 x 1g + 7g on a one-GPU node (every arrangement of the 1g claims
    is tried before the 7g claim fails).  A 1g running pod of lower priority keeps the pod out as the node stands (the
    pre-check fails the 7g); with it removed the search runs out of budget."""
    g, off = R.make_inventory([1], mig=True)
    t = R.default_table()
    rc, rpo, rpr, ro = mig_running([(0, 0, 1, R.GI_1_SLICE, 0)], off)
    g = occupied(g, rc, ro)
    c = _mig(R, [R.GI_1_SLICE] * 7 + [R.GI_7_SLICE])
    pod_off = np.array([0, 8], np.uint32)
    a = P.preempt(g, off, t, c, pod_off, [5], rc, rpo, rpr, ro, flags=P.F_EXHAUSTIVE)
    assert list(a[0]) == [P.SEARCH_LIMIT] and list(a[3]) == [P.SEARCH_LIMIT] and list(a[2]) == [NONE]
    a = P.preempt(g, off, t, c, pod_off, [5], rc, rpo, rpr, ro)
    assert list(a[0]) == [P.NO] and list(a[3]) == [P.NO]


def test_max_victims_shorter_than_the_count():
    g, off = R.make_inventory([1], mig=True)
    t = R.default_table()
    rc, rpo, rpr, ro = mig_running([(0, s, 1, R.GI_1_SLICE, 1) for s in range(7)], off)
    g = occupied(g, rc, ro)
    for mv in (0, 1, 3, 7, 9):
        a = P.preempt(g, off, t, _mig(R, [R.GI_7_SLICE]), np.array([0, 1], np.uint32), [2], rc, rpo, rpr, ro,
                      max_victims=mv)
        assert list(a[4]) == [7] and a[5].shape == (1, mv)
        assert list(a[5][0]) == list(range(min(mv, 7))) + [NONE] * max(0, mv - 7)


def test_invalid_and_empty_pods():
    g, off = R.make_inventory([1], mig=True)
    t = R.default_table()
    rc, rpo, rpr, ro = mig_running([(0, 0, 8, R.GI_7_SLICE, 0)], off)
    g = occupied(g, rc, ro)
    c = _mig(R, [R.GI_1_SLICE, 200] + [R.GI_1_SLICE] * 33)
    pod_off = np.array([0, 2, 2, 35], np.uint32)
    st, pv, node, pst, nv, vic = run_both(g, off, t, c, pod_off, [5, 5, 5], rc, rpo, rpr, ro, cands=[[0, 4], [4], [0]])
    assert list(st) == [P.INVALID, P.NO, P.NO, P.INVALID] and list(pst) == [P.INVALID, P.NO, P.INVALID]
    st, *_ = run_both(g, off, t, c, pod_off, [5, 5, 5], rc, rpo, rpr, ro, cands=[[4], [0], [4]])
    assert list(st) == [P.NO, P.FITS, P.NO]


def error_cases(g, off):
    """(name, changes to a valid call) for every DRA_E_INVAL condition of spec §14"""
    rc, rpo, rpr, ro = mig_running([(0, 0, 1, R.GI_1_SLICE, 0), (1, 0, 1, R.GI_1_SLICE, 0)], off)
    c = _mig(R, [R.GI_1_SLICE])
    bad_gpu = ro.copy(); bad_gpu[1]["gpu"] = len(g)
    ok = dict(c=c, po=np.array([0, 1], np.uint32), prio=[1], rc=rc, rpo=rpo, rpr=rpr, ro=ro, roo=None, cn=None, co=None,
              mv=4, fl=0)
    return ok, [
        ("unknown flags", dict(fl=0x1)), ("unknown flags", dict(fl=0x8)),
        ("pod_off not spanning", dict(po=np.array([1, 1], np.uint32))),
        ("pod_off not monotone", dict(c=np.concatenate([c, c]), po=np.array([0, 2, 1, 2], np.uint32), prio=[1, 1, 1])),
        ("cand_off not starting at 0", dict(cn=np.array([0, 1], np.uint32), co=np.array([1, 2], np.uint32))),
        ("cand_off not monotone", dict(c=np.concatenate([c, c]), po=np.array([0, 1, 2], np.uint32), prio=[1, 1],
                                       cn=np.array([0, 1], np.uint32), co=np.array([0, 2, 1], np.uint32))),
        ("running pod_off not monotone", dict(rpo=np.array([0, 2, 1], np.uint32))),
        ("running pod_off not spanning", dict(rpo=np.array([0, 1], np.uint32), rpr=rpr[:1])),
        ("slot range outside n_out", dict(roo=np.array([0, 5], np.uint32))),
        ("slot range outside n_out", dict(ro=ro[:1])),
        ("GPU index >= n_gpu", dict(ro=bad_gpu)),
        ("GPUs of two nodes", dict(rpo=np.array([0, 2], np.uint32), rpr=rpr[:1])),
    ]


def test_call_errors():
    g, off = R.make_inventory([1, 1], mig=True)
    t = R.default_table()
    ok, cases = error_cases(g, off)

    def call(a):
        return P.preempt(g, off, t, a["c"], a["po"], a["prio"], a["rc"], a["rpo"], a["rpr"], a["ro"], a["roo"], a["cn"],
                         a["co"], a["mv"], a["fl"])
    call(ok)
    for name, kw in cases:
        with pytest.raises(ValueError):
            call(dict(ok, **kw))
            pytest.fail(name)
    # max_victims > 0 without a victims buffer
    out = [np.zeros(4, np.uint32) for _ in range(5)]
    prio = np.array([1], np.int32)
    assert P.lib().pod_oracle_preempt(P._p(g), len(g), P._p(off), len(off) - 1, P._p(t), P._p(ok["c"]), 1,
                                      P._p(ok["po"]), P._p(prio), 1, None, None, P._p(ok["rc"]), 2, P._p(ok["rpo"]),
                                      P._p(ok["rpr"]), 2, None, P._p(ok["ro"]), 2, None, None, 0, P._p(out[0]),
                                      P._p(out[1]), None, P._p(out[2]), P._p(out[3]), P._p(out[4]), None, None, 3,
                                      0) == -1


def test_dense_form_over_two_to_the_32_pairs():
    n = 1 << 16
    g, off = R.make_inventory([1] * n, mig=True)
    with pytest.raises(ValueError):
        P.preempt(g, off, R.default_table(), np.zeros(0, R.CLAIM_DTYPE), np.zeros(n + 1, np.uint32), np.zeros(n, np.int32),
                  np.zeros(0, R.CLAIM_DTYPE), np.zeros(1, np.uint32), np.zeros(0, np.int32), np.zeros(0, R.OUT_DTYPE),
                  max_victims=0)


# ---- the C oracle against the naive restatement --------------------------------------------------------------------
def _small_world(seed):
    rng = np.random.default_rng(seed)
    w = synth.preempt(n_node=int(rng.integers(1, 4)), gpus_per_node=int(rng.integers(1, 4)), n_pending=int(rng.integers(1, 5)),
                      seed=seed, fill=int(rng.integers(50, 101)), mig_nodes=int(rng.integers(1, 5)), prio_lo=-20, prio_hi=40,
                      shared_per_gpu=3)
    c, po, prio = w.claims.copy(), list(w.pod_off), list(w.prio)
    extra = rng.integers(0, 4)
    if extra == 1:                                    # a mixed pod: 1g + SHARED
        e = np.zeros(2, R.CLAIM_DTYPE)
        e["kind"], e["profile"], e["count"], e["mem_limit_mib"] = [R.KIND_MIG, R.KIND_SHARED], [R.GI_1_SLICE, 0], 1, [0, 2048]
    elif extra == 2:                                  # an invalid claim
        e = np.zeros(1, R.CLAIM_DTYPE); e["kind"] = 3
    elif extra == 3:                                  # an empty pod
        e = np.zeros(0, R.CLAIM_DTYPE)
    if extra:
        c = np.concatenate([c, e]); po.append(len(c)); prio.append(int(rng.integers(-30, 60)))
    n_node = w.n_node if hasattr(w, "n_node") else len(w.node_off) - 1
    cands = None
    if rng.integers(0, 2):
        cands = [list(rng.integers(0, n_node + 2, size=int(rng.integers(0, 5)))) for _ in range(len(po) - 1)]
    return w, c, np.array(po, np.uint32), prio, cands


@pytest.mark.parametrize("seed", range(120))
def test_oracle_agrees_with_naive(seed):
    w, c, po, prio, cands = _small_world(seed)
    for flags in (0, P.F_EXHAUSTIVE):
        run_both(w.gpus, w.node_off, w.table, c, po, prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out,
                 cands=cands, flags=flags, max_victims=int(seed % 5))


# ---- properties on seeded synth.preempt worlds ------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(4))
def test_properties(seed, oracle):
    w = synth.preempt(n_node=12, gpus_per_node=4 + 4 * (seed % 2), n_pending=40, seed=seed)
    # the generator is consistent: deallocating every running pod empties the inventory
    g = oracle.deallocate(w.gpus, w.run_claims, w.run_out, n_node=len(w.node_off) - 1)
    assert g.tobytes() == w.empty.tobytes()
    n_pod, n_node = len(w.pod_off) - 1, len(w.node_off) - 1
    for flags in (0, P.F_EXHAUSTIVE):
        st, pv, node, pst, nv, vic = P.preempt(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims,
                                               w.run_pod_off, w.run_prio, w.run_out, max_victims=64, flags=flags)
        if flags:
            cn = np.tile(np.arange(n_node, dtype=np.uint32), n_pod)
            co = (np.arange(n_pod + 1) * n_node).astype(np.uint32)
            bits = oracle.unsuitable(w.gpus, w.node_off, w.table, w.claims, w.pod_off, cn, co, flags=oracle.F_EXHAUSTIVE)
            fits = np.unpackbits(bits, bitorder="little")[: n_pod * n_node].astype(bool)
            assert (fits == (st == P.FITS)).all()
        assert (pst == P.EVICT).any()
        for p in np.flatnonzero(pst == P.EVICT):
            v = vic[p][: nv[p]]
            assert nv[p] <= 64 and (w.run_prio[v] < w.prio[p]).all()
            keep = np.zeros(len(w.run_claims), bool)
            for r in v:
                keep[w.run_pod_off[r]: w.run_pod_off[r + 1]] = True
            g = oracle.deallocate(w.gpus, w.run_claims[keep], w.run_out[keep], n_node=n_node)
            pod = w.claims[w.pod_off[p]: w.pod_off[p + 1]].copy()
            pod["node"] = node[p]
            oo, n_out = R.out_offsets(pod, n_node)
            out, _ = oracle.allocate_pods(g, w.node_off, w.table, pod, np.array([0, len(pod)], np.uint32), oo, n_out,
                                          flags=flags)
            assert (out["status"] == R.ST_OK).all()
