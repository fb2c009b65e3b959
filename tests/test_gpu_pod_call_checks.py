"""GPU suite: what the synchronous pod calls (UnsuitableNodes, pods Allocate, place pods, preemption, preempt and place)
promise about their arguments — the return code of every rejected call, with no output byte and no inventory word
written, the kernels each call launches and the chain bits it reports, and the kernel times it leaves under profiling.

The per-pod candidate limit and the node limit of place pods and preempt and place (PL_POS, 2^30 - 1) are checked by
the calls but cannot be reached here."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

from test_preempt import mig_running

import place_oracle as PL
import preempt_oracle as PR
import preempt_place_oracle as PP

pytestmark = pytest.mark.gpu
SENTINEL = 0xAB
UNS, PODS, PLACE, PRE, PREPL = "unsuitable", "allocate_pods", "place_pods", "preempt", "preempt_place"
ALL = (UNS, PODS, PLACE, PRE, PREPL)
CANDS = (UNS, PLACE, PRE, PREPL)
CN, CO = [0, 1, 1], [0, 2, 3]                               # a valid candidate form for the two pending pods


@pytest.fixture(scope="module")
def ctx(pkg):
    c = pkg.api.Context(device=0)
    yield c
    c.close()


def _world(R):
    """Two 1-GPU MIG nodes; two pending pods of one 1g claim each (node 0); one running 1g pod on each GPU."""
    g, off = R.make_inventory([1, 1], mig=True)
    c = np.zeros(2, R.CLAIM_DTYPE)
    c["kind"], c["profile"], c["count"] = R.KIND_MIG, R.GI_1_SLICE, 1
    rc, rpo, rpr, ro = mig_running([(0, 0, 1, R.GI_1_SLICE, 0), (1, 0, 1, R.GI_1_SLICE, 0)], off)
    return SimpleNamespace(g=g, off=off, t=R.default_table(), c=c, po=np.array([0, 1, 2], np.uint32),
                           prio=np.array([1, 1], np.int32), rc=rc, rpo=rpo, rpr=rpr, ro=ro)


def _load(ctx, w):
    ctx.set_table(w.t)
    ctx.set_inventory(w.g, w.off)


def _base(w):
    return dict(c=w.c, po=w.po, prio=w.prio, cn=None, co=None, oo=None, n_out=len(w.c), mv=4, victims=True, fl=0)


def _raw(pkg, ctx, w, fn, a):
    """dra_<fn> through ctypes on outputs of 64 sentinel-filled elements each; returns (rc, outputs)"""
    A = pkg.api
    def arr(k, dt):
        return None if a.get(k) is None else np.ascontiguousarray(a[k], dtype=dt)
    c, po, prio = arr("c", A.R.CLAIM_DTYPE), arr("po", np.uint32), arr("prio", np.int32)
    cn, co, oo = arr("cn", np.uint32), arr("co", np.uint32), arr("oo", np.uint32)
    n_pod, n_out, fl = len(po) - 1, a["n_out"], a["fl"]
    dts = {UNS: [np.uint8], PODS: [A.R.OUT_DTYPE], PLACE: [A.R.OUT_DTYPE, np.uint32],
           PRE: [np.uint8, np.uint32, np.uint32, np.uint8, np.uint32, np.uint32],
           PREPL: [A.R.OUT_DTYPE, np.uint32, np.uint8, np.uint32]}[fn]
    o = [np.full(64 * np.dtype(d).itemsize, SENTINEL, np.uint8).view(d) for d in dts]
    run = A.RunningPods(w.rc.ctypes.data, len(w.rc), w.rpo.ctypes.data, len(w.rpo) - 1, w.rpr.ctypes.data, None,
                        w.ro.ctypes.data, len(w.ro))
    p = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)      # noqa: E731
    L, h = ctx._lib, ctx._h
    if fn == UNS:
        rc = L.dra_unsuitable_batch(h, p(c), len(c), p(po), n_pod, p(cn), p(co), p(o[0]), fl)
    elif fn == PODS:
        rc = L.dra_allocate_pods_batch(h, p(c), len(c), p(po), n_pod, p(oo), p(o[0]), n_out, fl)
    elif fn == PLACE:
        rc = L.dra_place_pods_batch(h, p(c), len(c), p(po), n_pod, p(cn), p(co), p(oo), p(o[0]), n_out, p(o[1]), fl)
    elif fn == PRE:
        rc = L.dra_preempt_batch(h, p(c), len(c), p(po), p(prio), n_pod, p(cn), p(co), C.byref(run), *[p(x) for x in o[:5]],
                                 p(o[5]) if a["victims"] else None, a["mv"], fl)
    else:
        rc = L.dra_preempt_place_batch(h, p(c), len(c), p(po), p(prio), n_pod, p(cn), p(co), C.byref(run), p(oo), p(o[0]),
                                       n_out, p(o[1]), p(o[2]), p(o[3]), fl)
    return rc, o


def _valid(pkg, ctx, oracle, w, fn):
    """The valid base call through the Python API against its oracle, from the loaded inventory w.g"""
    _load(ctx, w)
    if fn == UNS:
        got = ctx.unsuitable(w.c, w.po, CN, CO)
        assert got.tobytes() == oracle.unsuitable(w.g, w.off, w.t, w.c, w.po, CN, CO).tobytes()
        return
    if fn == PODS:
        c = w.c.copy()
        c["node"] = [0, 1]
        got, ref = [ctx.allocate_pods(c, w.po)], oracle.allocate_pods(w.g, w.off, w.t, c, w.po)
    elif fn == PLACE:
        got, ref = ctx.place_pods(w.c, w.po), PL.place_pods(w.g, w.off, w.t, w.c, w.po, n_out=len(w.c))
    elif fn == PRE:
        got = ctx.preempt(w.c, w.po, w.prio, w.rc, w.rpo, w.rpr, w.ro, max_victims=4)
        ref = PR.preempt(w.g, w.off, w.t, w.c, w.po, w.prio, w.rc, w.rpo, w.rpr, w.ro, max_victims=4) + (w.g,)
    else:
        got = ctx.preempt_place(w.c, w.po, w.prio, w.rc, w.rpo, w.rpr, w.ro, n_out=len(w.c))
        ref = PP.preempt_place(w.g, w.off, w.t, w.c, w.po, w.prio, w.rc, w.rpo, w.rpr, w.ro, n_out=len(w.c))
    for x, y in zip(got, ref[:-1]):
        assert x.tobytes() == y.tobytes(), fn
    assert ctx.get_inventory().tobytes() == ref[-1].tobytes(), fn


CASES = [
    ("unknown flag", ALL, dict(fl=0x1)),                   # DRA_F_NODE_SORTED: none of the five takes it
    ("pod_off[0] != 0", ALL, dict(po=[1, 1, 2])),
    ("pod_off[n_pod] != n_claim", ALL, dict(po=[0, 1, 1])),
    ("pod_off decreasing", ALL, dict(po=[0, 2, 1, 2], prio=[1, 1, 1])),
    ("cand_nodes without cand_off", CANDS, dict(cn=[0])),
    ("cand_off listing candidates, cand_nodes NULL", CANDS, dict(co=[0, 1, 2])),
    ("cand_off[0] != 0", CANDS, dict(cn=[0, 1], co=[1, 1, 2])),
    ("cand_off decreasing", CANDS, dict(cn=[0, 1], co=[0, 2, 1])),
    ("n_out < n_claim without out_off", (PODS, PLACE, PREPL), dict(n_out=1)),
    ("a claim's slots past n_out", (PODS, PLACE, PREPL), dict(oo=[0, 5])),
    ("max_victims without victims", (PRE,), dict(victims=False)),
]


@pytest.mark.parametrize("fn", ALL)
def test_one_fault_calls_are_rejected_and_write_nothing(pkg, ctx, oracle, fn):
    A, R = pkg.api, pkg.records
    w = _world(R)
    _load(ctx, w)
    rc, _ = _raw(pkg, ctx, w, fn, _base(w))
    assert rc == A.OK, fn
    for name, fns, kw in CASES:
        if fn not in fns:
            continue
        _load(ctx, w)
        rc, outs = _raw(pkg, ctx, w, fn, dict(_base(w), **kw))
        assert rc == A.E_INVAL, name
        assert all((o.view(np.uint8) == SENTINEL).all() for o in outs), name
        assert ctx.get_inventory().tobytes() == w.g.tobytes(), name
        _valid(pkg, ctx, oracle, w, fn)


@pytest.mark.parametrize("fn", ALL)
def test_no_inventory_is_a_state_error_before_any_argument_error(pkg, fn):
    A, R = pkg.api, pkg.records
    w = _world(R)
    with A.Context(device=0) as c:
        c.set_table(w.t)
        for kw in ({}, dict(po=[1, 1, 2])):
            rc, outs = _raw(pkg, c, w, fn, dict(_base(w), **kw))
            assert rc == A.E_STATE, kw
            assert all((o.view(np.uint8) == SENTINEL).all() for o in outs), kw


def _call(ctx, w, fn, form):
    """One valid call in the given form: dense, cands, no pods, or (preemption) no running pods"""
    c, po, prio = (w.c[:0], np.zeros(1, np.uint32), w.prio[:0]) if form == "no pods" else (w.c, w.po, w.prio)
    cn, co = (CN, CO) if form == "cands" else (None, None)
    run = (w.rc[:0], np.zeros(1, np.uint32), w.rpr[:0], w.ro[:0]) if form == "no running" else (w.rc, w.rpo, w.rpr, w.ro)
    if fn == UNS:
        ctx.unsuitable(c, po, cn, co)
    elif fn == PODS:
        pc = c.copy()
        pc["node"] = np.arange(len(pc)) % 2
        ctx.allocate_pods(pc, po)
    elif fn == PLACE:
        ctx.place_pods(c, po, cn, co)
    elif fn == PRE:
        ctx.preempt(c, po, prio, *run, None, cn, co)
    else:
        ctx.preempt_place(c, po, prio, *run, None, cn, co)


# Launches and chain bits of one call on the two-node world (None: the call leaves the previous call's chain)
CHAINS = [
    (UNS, "dense", 1, None), (UNS, "cands", 1, None), (UNS, "no pods", 0, None),
    (PODS, "dense", 3, {"bucket_small"}), (PODS, "no pods", 0, set()),
    (PLACE, "dense", 2, {"place"}), (PLACE, "cands", 3, {"bucket_small", "place"}), (PLACE, "no pods", 0, set()),
    (PRE, "dense", 6, {"preempt", "bucket_small"}), (PRE, "cands", 6, {"preempt", "bucket_small"}),
    (PRE, "no pods", 0, {"preempt"}), (PRE, "no running", 5, {"preempt"}),
    (PREPL, "dense", 5, {"preempt_place", "bucket_small"}), (PREPL, "cands", 6, {"preempt_place", "bucket_small"}),
    (PREPL, "no pods", 0, {"preempt_place"}), (PREPL, "no running", 3, {"preempt_place"}),
]


@pytest.mark.parametrize("fn,form,launches,chain", CHAINS)
def test_launch_count_and_chain(pkg, ctx, fn, form, launches, chain):
    w = _world(pkg.records)
    _load(ctx, w)
    ctx.allocate_pods(w.c[:0], np.zeros(1, np.uint32))        # a known chain before the call: none
    before, n0 = ctx.last_chain(), ctx.launch_count()
    _call(ctx, w, fn, form)
    assert ctx.launch_count() - n0 == launches
    assert ctx.last_chain() == (before if chain is None else chain)


# The stages each call times: its sort's first stage ("bucket_hist", here one kernel) and its walk ("pack"); place pods'
# dense form sorts nothing, so its one stage spans the whole call
TIMED = [(PODS, "dense", {"bucket_hist", "pack"}), (PLACE, "dense", {"bucket_hist"}),
         (PLACE, "cands", {"bucket_hist", "pack"})]


@pytest.mark.parametrize("fn,form,stages", TIMED)
def test_profiling_times_the_call(pkg, fn, form, stages):
    """A fresh context, so no earlier call's times can stand in for this one's."""
    A = pkg.api
    w = _world(pkg.records)
    with A.Context(device=0) as c:
        c.set_profiling(True)
        _load(c, w)
        _call(c, w, fn, form)
        t = c.timings_us()
        assert {k for k, v in t.items() if v > 0} == stages, t
