"""GPU suite: preempt and place (spec §15) at its edges, on one inventory (dra_preempt_place_batch) and on a sharded world
of one device (dra_preempt_place_batch_global_device).  Every call's outputs (OutRecs, pod_node, pod_status, evicted_by)
and the live inventory afterwards are compared byte for byte with preempt_place_oracle.preempt_place on the same
inventory; nothing may be written past an output, and reset_inventory() must give back the inventory as loaded.  A
call-level error returns E_INVAL with no output and no inventory word written.

* the hand-written §15 fixtures of test_preempt_place.py, and every §14 fixture of test_preempt.py one pod at a time
  (a one-pod §15 call is §14's judgement, then applied)
* the 64-bit priority sum, and choices whose best pair sits past the first warp of a pod's candidates
* random problems (tests/preempt_problems.py): mismatched records, run_out_off, and the pending out_off absent, packed,
  permuted with gaps, or with spare slots
* the call's slot mode: without out_off a multi-GPU claim is INVALID, and its pod evicts nothing
* more nodes than the walk has warps: every warp owns several nodes, leaves a waiting one and comes back to it, along a
  serial chain of hand-offs across the whole inventory
* one context reused by calls that grow and shrink every size, interleaved with the calls sharing its buffers
* the sharded call on worlds of one to three contexts"""
import dataclasses
import functools
import inspect
import os
from types import SimpleNamespace

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

import preempt_oracle as P
import preempt_place_oracle as PP
import test_preempt_place as TP
from preempt_problems import NONE, PlaceProblem, Problem, _Rng, as_place, place_problems, random_place_problem
from test_gpu_preempt_edges import _call as _call14, _fixture_problems, _load, _n_sm, _sum_world, _warp_world
from test_gpu_preempt_place import _raw
from test_gpu_shard_preempt import Running
from test_gpu_shard_preempt_place import World
from test_gpu_shard_unsuitable import _bounds
from test_pod_mode import _mig
from test_preempt import mig_running, occupied
from test_preempt_place import check_matched

pytestmark = pytest.mark.gpu
SENT, SLACK = 0xA5, 16
NAMES = ("out", "pod_node", "pod_status", "evicted_by")
N_EX = int(os.environ.get("DRA_PROP_EXAMPLES", "0"))      # > 0: that many RANDOM examples instead of the fixed ones


@pytest.fixture(scope="module")
def pctx(pkg):
    c = pkg.api.Context(device=0)
    yield c
    c.close()


def _call(pkg, ctx, pb, pristine, flags=None, what=""):
    """dra_preempt_place_batch on pb against the oracle on the context's live inventory; then reset_inventory() must give
    back `pristine`.  Returns (out, pod_node, pod_status, evicted_by, inventory after), or None when the call must fail
    (E_INVAL, nothing written)."""
    A = pkg.api
    flags = pb.flags if flags is None else flags
    before = ctx.get_inventory()
    cn, co = pb.cand_arrays()
    a = dict(c=pb.claims, po=pb.pod_off, prio=pb.prio, rc=pb.run_claims, rpo=pb.run_pod_off, rpr=pb.run_prio,
             ro=pb.run_out, roo=pb.run_out_off, cn=cn, co=co, oo=pb.out_off, n_out=pb.n_out,
             fl=A.F_EXHAUSTIVE if flags else 0)
    rc_, outs = _raw(pkg, ctx, a, SENT, SLACK)
    try:
        # slots no claim owns come back zero; with no pending pods, evicted_by is not written
        ref = pb.pp_oracle(before, flags, fill=0 if len(pb.prio) else SENT)
    except ValueError:
        ref = None
    after = ctx.get_inventory()
    got = None
    if ref is None:
        assert rc_ == A.E_INVAL, what
        assert all((o.view(np.uint8) == SENT).all() for o in outs), f"{what}: an output was written"
        assert after.tobytes() == before.tobytes(), f"{what}: a failed call changed the inventory"
    else:
        assert rc_ == A.OK, what
        assert "preempt_place" in ctx.last_chain(), what
        got = []
        for name, o, y in zip(NAMES, outs, ref):
            x = o[: y.size]
            if x.tobytes() != y.tobytes():
                bad = np.flatnonzero(x.view(np.uint8) != y.view(np.uint8))[:5]
                pytest.fail(f"{what}: {name} differs at bytes {bad}")
            assert (o[y.size:].view(np.uint8) == SENT).all(), f"{what}: written past {name}"
            got.append(x)
        if after.tobytes() != ref[4].tobytes():
            bad = np.flatnonzero(after != ref[4])[:5]
            pytest.fail(f"{what}: inventory differs at GPUs {bad}: device {after[bad]} oracle {ref[4][bad]}")
        got.append(after)
    ctx.reset_inventory()
    assert ctx.get_inventory().tobytes() == pristine.tobytes(), f"{what}: reset did not give back the loaded inventory"
    return got


def _run(pkg, ctx, pb, **kw):
    _load(ctx, pb)
    return _call(pkg, ctx, pb, pb.gpus, **kw)


def _place(pb, form="packed", seed=0):
    """pb as a §15 problem (each call finds its own verdict from the oracle)"""
    return as_place(pb, _Rng(np.random.default_rng(seed)), form, judge=False)


# ---- 1. the hand-written fixtures -----------------------------------------------------------------------------------
FIXTURES = [TP.test_two_pods_one_victim, TP.test_evicted_pod_is_not_counted_again_and_placed_pods_are_never_victims,
            TP.test_fits_anywhere_beats_evict, TP.test_equal_priority_is_not_evictable,
            TP.test_empty_pod_invalid_claims_and_33_claims, TP.test_node_listed_twice, TP.test_search_limit,
            *[functools.partial(TP.test_slot_mode_decides_validity, c, f) for c in (None, [[0]], [[5, 0, 0]])
              for f in (0, PP.F_EXHAUSTIVE)]]


def _pp_fixture_problems(monkeypatch):
    """every preempt_place_oracle.preempt_place call the §15 fixtures make (each still checks its own answer)"""
    calls, orig = [], PP.preempt_place
    sig = inspect.signature(orig)

    def record(*args, **kw):
        res = orig(*args, **kw)
        b = sig.bind(*args, **kw)
        b.apply_defaults()
        calls.append(dict(b.arguments))
        return res
    monkeypatch.setattr(PP, "preempt_place", record)
    try:
        for f in FIXTURES:
            f()
    finally:
        monkeypatch.undo()
    out = []
    for a in calls:
        co, cn = a["cand_off"], a["cand_nodes"]
        cands = None if co is None else [[int(x) for x in cn[co[p]: co[p + 1]]] for p in range(len(co) - 1)]
        c = a["claims"]
        n_out = a["n_out"] if a["n_out"] is not None else PP.pending_slots(c, a["out_off"]) if len(c) else 0
        out.append(PlaceProblem(a["gpus"], np.asarray(a["node_off"], np.uint32), a["table"], c,
                                np.asarray(a["pod_off"], np.uint32), np.asarray(a["prio"], np.int32), cands,
                                a["run_claims"], np.asarray(a["run_pod_off"], np.uint32),
                                np.asarray(a["run_prio"], np.int32), a["run_out"], a["run_out_off"], 0, a["flags"], True,
                                False, out_off=a["out_off"], n_out=n_out))
    return out


def test_hand_written_fixtures(pkg, pctx, monkeypatch):
    pbs = _pp_fixture_problems(monkeypatch)
    assert len(pbs) >= 20
    for i, pb in enumerate(pbs):
        for flags in (0, PP.F_EXHAUSTIVE):
            _run(pkg, pctx, pb, flags=flags, what=f"fixture {i} f{flags}")


def test_preempt_fixtures_one_pod_at_a_time(pkg, pctx, monkeypatch):
    """A one-pod §15 call judges the pod as §14 does: its pod_node and pod_status are §14's, and when §14's victim row
    holds them all, evicted_by marks exactly those victims."""
    pbs = _fixture_problems(monkeypatch)
    assert len(pbs) >= 20
    n_calls = 0
    for i, pb in enumerate(pbs):
        for flags in (0, P.F_EXHAUSTIVE):
            _, _, node, status, nv, vic = pb.oracle(flags=flags)
            for p in range(len(pb.prio)):
                c0, c1 = int(pb.pod_off[p]), int(pb.pod_off[p + 1])
                one = dataclasses.replace(pb, claims=pb.claims[c0:c1], pod_off=np.array([0, c1 - c0], np.uint32),
                                          prio=pb.prio[p:p + 1], cands=None if pb.cands is None else [pb.cands[p]])
                got = _run(pkg, pctx, _place(one), flags=flags, what=f"fixture {i} pod {p} f{flags}")
                assert got[1][0] == node[p] and got[2][0] == status[p], (i, p, flags)
                if nv[p] <= pb.max_victims:
                    assert sorted(np.flatnonzero(got[3] == 0)) == sorted(vic[p][: nv[p]]), (i, p, flags)
                n_calls += 1
    assert n_calls >= 40


# ---- 2. the 64-bit priority sum, and choices past one warp ----------------------------------------------------------
def test_priority_sum_is_64_bit(pkg, pctx):
    R = pkg.records
    for a_first in (True, False):
        for cands in (None, [[0, 1]], [[1, 0]]):
            pb, nb, vic = _sum_world(R, a_first)
            for form in ("none", "packed"):
                x = _place(dataclasses.replace(pb, cands=cands), form)
                for flags in (0, P.F_EXHAUSTIVE):
                    out, node, st_, ev, after = _run(pkg, pctx, x, flags=flags, what=f"sum {a_first} {cands} {form}")
                    assert list(node) == [nb] and list(st_) == [PP.EVICT]
                    assert list(ev) == [NONE, NONE, 0, 0] and vic == [2, 3]
                    assert after[nb]["busy"] != 0 and after[1 - nb].tobytes() == pb.gpus[1 - nb].tobytes()


def test_choice_past_one_warp(pkg, pctx):
    """test_gpu_preempt_edges' world of three one-GPU nodes: pod 0's best pair (node 0) sits at positions 5, 6, 37 and
    69 of 70; then node 0 holds pod 0, which is no victim, so pod 1 takes node 2 (its victim of priority 5 beats node 1's
    of priority 6), found on lane 0 of the first warp among 70 entries."""
    R = pkg.records
    g, off, rc, rpo, rpr, ro = _warp_world(R)
    stray = [3, 4, NONE]
    a = [stray[k % 3] if k % 4 else 1 for k in range(70)]
    for k in (0, 2, 33, 36, 64):
        a[k] = 2
    for k in (5, 6, 37, 69):
        a[k] = 0
    b = [2 if k % 3 == 0 else 1 if k % 3 == 1 else stray[k % 2] for k in range(70)]
    b[63], b[64] = 0, 0
    pb = Problem(g, off, R.default_table(), _mig(R, [R.GI_7_SLICE, R.GI_7_SLICE]), np.array([0, 1, 2], np.uint32),
                 np.array([100, 100], np.int32), [a, b], rc, rpo, rpr, ro, None, 2, 0, True, False)
    for form in ("none", "gaps"):
        for flags in (0, P.F_EXHAUSTIVE):
            out, node, st_, ev, after = _run(pkg, pctx, _place(pb, form, flags), flags=flags, what=f"past one warp {form}")
            assert list(node) == [0, 2] and list(st_) == [PP.EVICT, PP.EVICT] and list(ev) == [1, NONE, 0]
            assert (out["status"] == R.ST_OK).all()


# ---- 3. random problems ---------------------------------------------------------------------------------------------
def _check_random(pkg, ctx, pb):
    got = _run(pkg, ctx, pb, what=pb.what)
    assert (got is None) == pb.error, pb.what
    if got is not None and pb.matched and len(pb.prio):
        out, node, st_, ev, _ = got
        check_matched(pb.gpus, pb.node_off, pb.claims, pb.pod_off, out, node, st_, ev, pb.out_off)
    return got


def test_random_problems(pkg, pctx):
    forms = {}

    @settings(max_examples=N_EX or 120, deadline=None, suppress_health_check=list(HealthCheck), derandomize=N_EX == 0,
              database=None)
    @given(place_problems())
    def run(pb):
        _check_random(pkg, pctx, pb)
        forms[pb.form] = forms.get(pb.form, 0) + 1
    run()
    assert len(forms) == 4, forms


def test_larger_random_problems(pkg, pctx):
    """the same builder at 8 and 32 times the nodes and running pods"""
    n = 0
    for seed in range(40):
        pb = random_place_problem(500 + seed, 8 if seed % 2 else 32)
        n += _check_random(pkg, pctx, pb) is not None
    assert n >= 30


# ---- 4. the call's slot mode ----------------------------------------------------------------------------------------
SHAPES = ("gpu1", "gpu2", "gpu3", "gpu4", "3g", "7g")


def _synth_problem(w, cands=None, flags=0):
    return Problem(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, cands, w.run_claims, w.run_pod_off,
                   w.run_prio, w.run_out, None, 0, flags, True, False)


@pytest.mark.parametrize("mig_nodes", [4, 0])
def test_slot_mode(pkg, pctx, mig_nodes):
    """1- to 4-GPU claims on a MIG and a non-MIG world, with and without out_off, dense and with candidates.  Without
    out_off a pod with a multi-GPU claim is INVALID and evicts nothing; with nothing evictable, pod_node is place pods'
    for every non-empty pod."""
    R = pkg.records
    rng = np.random.default_rng(mig_nodes)
    multi_evict = 0
    for prio_kw in ({}, dict(prio_lo=500, prio_hi=600, pending_prio=500)):
        w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=48, seed=3 + mig_nodes, mig_nodes=mig_nodes,
                              shapes=SHAPES, **prio_kw)
        n_pod = len(w.prio)
        multi = np.array([((w.claims["kind"][w.pod_off[p]:w.pod_off[p + 1]] == R.KIND_GPU) &
                           (w.claims["count"][w.pod_off[p]:w.pod_off[p + 1]] > 1)).any() for p in range(n_pod)])
        assert multi.any() and not multi.all()
        for cands in (None, [[int(x) for x in rng.integers(0, 14, 6)] for _ in range(n_pod)]):
            for form in ("none", "packed"):
                for flags in (0, P.F_EXHAUSTIVE):
                    pb = _place(_synth_problem(w, cands, flags), form)
                    what = f"slot mode mig {mig_nodes} {prio_kw} {form} cands {cands is not None} f{flags}"
                    out, node, st_, ev, after = _run(pkg, pctx, pb, what=what)
                    check_matched(pb.gpus, pb.node_off, pb.claims, pb.pod_off, out, node, st_, ev, pb.out_off)
                    if form == "none":
                        assert (st_[multi] == PP.INVALID).all() and not np.isin(ev, np.flatnonzero(multi)).any(), what
                    if prio_kw:
                        assert (ev == NONE).all()
                        cn, co = pb.cand_arrays()
                        _load(pctx, pb)
                        pout, pnode = pctx.place_pods(pb.claims, pb.pod_off, cn, co, pb.out_off, pb.n_out,
                                                      pkg.api.F_EXHAUSTIVE if flags else 0)
                        assert pout.tobytes() == out.tobytes() and pctx.get_inventory().tobytes() == after.tobytes(), what
                        assert (pnode == node).all(), what
                        pctx.reset_inventory()
                    elif form == "packed":
                        multi_evict += int((st_[multi] == PP.EVICT).sum())
    assert (multi_evict > 0) == (mig_nodes == 0)         # with out_off, multi-GPU pods do evict where GPUs are whole


# ---- 5. more nodes than the walk has warps --------------------------------------------------------------------------
def _n_wide():
    """every warp of the walk owns at least two nodes at any occupancy: at most 16 CTAs of 4 warps per SM"""
    return 128 * _n_sm() + 37


def _chain(R, n, mirror):
    """n one-GPU MIG nodes, node k (mirrored: n-1-k) held by running pod k, a 7g pod of priority 0.  Pending: n-1 7g pods
    of priority 1, pod i listing nodes i+1 and i.  Each pair is EVICT with one victim of priority 0, and the later
    running pod wins the tie, so pod i takes node i+1 from running pod i+1, and pod i+1 finds node i+1 held by a pod that
    is no victim: one hand-off per pod, along the whole inventory."""
    at = (lambda k: n - 1 - k) if mirror else (lambda k: k)
    g, off = R.make_inventory([1] * n, mig=True)
    rc = np.zeros(n, R.CLAIM_DTYPE)
    rc["kind"], rc["profile"], rc["count"] = R.KIND_MIG, R.GI_7_SLICE, 1
    rc["node"] = [at(k) for k in range(n)]
    ro = np.zeros(n, R.OUT_DTYPE)
    ro["gpu"], ro["start"], ro["size"], ro["profile"], ro["status"] = rc["node"], 0, 8, R.GI_7_SLICE, R.ST_OK
    g = occupied(g, rc, ro)
    c = _mig(R, [R.GI_7_SLICE] * (n - 1))
    cands = [[at(i + 1), at(i)] for i in range(n - 1)]
    pb = Problem(g, off, R.default_table(), c, np.arange(n, dtype=np.uint32), np.ones(n - 1, np.int32), cands, rc,
                 np.arange(n + 1, dtype=np.uint32), np.zeros(n, np.int32), ro, None, 1, 0, True, False)
    return pb, at


def test_serial_chain_across_more_nodes_than_warps(pkg, pctx):
    R = pkg.records
    n = _n_wide()
    for mirror in (False, True):
        pb, at = _chain(R, n, mirror)
        for form in ("packed", "none"):
            out, node, st_, ev, after = _run(pkg, pctx, _place(pb, form), what=f"chain mirror {mirror} {form}")
            assert (node == np.array([at(i + 1) for i in range(n - 1)], np.uint32)).all()
            assert (st_ == PP.EVICT).all() and ev[0] == NONE and (ev[1:] == np.arange(n - 1)).all()
            assert (out["status"] == R.ST_OK).all() and (after["busy"] == pb.gpus["busy"]).all()


def test_synthetic_world_wider_than_the_walk(pkg, pctx):
    n = _n_wide()
    w = pkg.synth.preempt(n_node=n, gpus_per_node=2, n_pending=3000, seed=17)
    rng = np.random.default_rng(17)
    cands = [[int(x) for x in rng.integers(0, n + 2, 8)] for _ in range(len(w.prio))]
    pb = _place(_synth_problem(w, cands))
    got = _run(pkg, pctx, pb, what="wide, 8 candidates")
    assert (got[2] == PP.EVICT).sum() > 100
    check_matched(w.gpus, w.node_off, w.claims, w.pod_off, got[0], got[1], got[2], got[3], pb.out_off)
    po = w.pod_off[:41]
    few = dataclasses.replace(_synth_problem(w, None, P.F_EXHAUSTIVE), claims=w.claims[: po[-1]], pod_off=po,
                              prio=w.prio[:40])
    got = _run(pkg, pctx, _place(few, "gaps"), what="wide, dense")
    assert (got[2] == PP.EVICT).any()


# ---- 6. one context, sizes growing and shrinking, shared buffers in between -----------------------------------------
def _pick(scale, want_off, start):
    """the first valid random §15 problem from seed `start` on with (or without) run_out_off"""
    s = start
    while True:
        pb = random_place_problem(s, scale)
        if (pb.run_out_off is not None) == want_off and not pb.error and len(pb.prio):
            return pb
        s += 1


def _on_two_nodes(pb):
    """pb with two consecutive running pods on different nodes merged into one (a call-level error found on the
    device), or None"""
    node_of = np.searchsorted(pb.node_off, np.arange(len(pb.gpus)), side="right") - 1
    roo = pb.run_out_off
    nodes = []
    for r in range(len(pb.run_prio)):
        s = set()
        for i in range(int(pb.run_pod_off[r]), int(pb.run_pod_off[r + 1])):
            b = int(roo[i]) if roo is not None else i
            o = pb.run_out[b]
            if o["status"] == 0 and o["gpu"] < len(pb.gpus):
                s.add(int(node_of[o["gpu"]]))
        nodes.append(s)
    for r in range(len(nodes) - 1):
        if len(nodes[r]) == 1 and len(nodes[r + 1]) == 1 and nodes[r] != nodes[r + 1]:
            return dataclasses.replace(pb, run_pod_off=np.delete(pb.run_pod_off, r + 1).astype(np.uint32),
                                       run_prio=np.delete(pb.run_prio, r + 1).astype(np.int32), error=True)
    return None


def test_context_reuse(pkg, oracle):
    import place_oracle
    R, A = pkg.records, pkg.api
    ctx = A.Context(device=0)
    rejected = 0
    try:
        for it, scale in enumerate((1, 4, 16, 2, 16, 1, 8, 1)):
            pb = _pick(scale, it % 2 == 0, 2000 * it)
            what = f"reuse {it} scale {scale}"
            _load(ctx, pb)
            _call(pkg, ctx, pb, pb.gpus, what=what)
            bad = _on_two_nodes(pb)
            if bad is not None:                          # rejected on the device, then a good call
                assert _call(pkg, ctx, bad, pb.gpus, what=what + " two nodes") is None
                rejected += 1
                _call(pkg, ctx, pb, pb.gpus, what=what + " after the rejection")
            # §14 on the same pods (it shares the running-pod buffers)
            _call14(pkg, ctx, pb, pb.gpus, what=what + " preempt")
            # the running claims through Allocate, which takes the live inventory on
            oo, n_out = R.out_offsets(pb.run_claims, pb.n_node)
            out = ctx.allocate(pb.run_claims, oo, n_out)
            ref, live = oracle.allocate(pb.gpus, pb.node_off, pb.table, pb.run_claims, oo, n_out)
            assert out.tobytes() == ref.tobytes() and ctx.get_inventory().tobytes() == live.tobytes(), what
            _call(pkg, ctx, dataclasses.replace(pb, flags=P.F_EXHAUSTIVE - pb.flags), pb.gpus, what=what + " after")
            # UnsuitableNodes and place pods on the pending pods
            cn, co = pb.cand_arrays()
            if cn is None:
                n_pod = len(pb.prio)
                cn = np.tile(np.arange(pb.n_node, dtype=np.uint32), n_pod)
                co = (np.arange(n_pod + 1) * pb.n_node).astype(np.uint32)
            bits = ctx.unsuitable(pb.claims, pb.pod_off, cn, co, flags=pb.flags)
            assert bits.tobytes() == oracle.unsuitable(pb.gpus, pb.node_off, pb.table, pb.claims, pb.pod_off, cn, co,
                                                       flags=pb.flags).tobytes(), what
            placed = pb.claims.copy()
            placed["node"] = 0
            po, n_po = R.out_offsets(placed, 1)
            out, node = ctx.place_pods(pb.claims, pb.pod_off, cn, co, po, n_po, flags=pb.flags)
            ref, rnode, after = place_oracle.place_pods(pb.gpus, pb.node_off, pb.table, pb.claims, pb.pod_off, cn, co,
                                                        po, n_po, flags=pb.flags)
            assert out.tobytes() == ref.tobytes() and node.tobytes() == rnode.tobytes(), what
            assert ctx.get_inventory().tobytes() == after.tobytes(), what
            _call(pkg, ctx, pb, pb.gpus, what=what + " after place")
        assert rejected >= 2
    finally:
        ctx.close()


# ---- 7. the sharded call on one device ------------------------------------------------------------------------------
CONFIGS = [(1, "even"), (2, "even"), (2, "uneven"), (3, "empty"), (3, "uneven")]


def _sharded(pkg, pb, world, kind, what=""):
    """pb on a world of `world` contexts, every rank against the oracle on the world's state; a call-level error must
    fail every rank with nothing written"""
    A = pkg.api
    w = SimpleNamespace(gpus=pb.gpus, node_off=pb.node_off, table=pb.table, run_claims=pb.run_claims)
    W = World(pkg, w, world, _bounds(pb.n_node, world, kind), sizes=(64, 4096, 512))
    what = f"{what} world {world} {kind}"
    fl = A.F_EXHAUSTIVE if pb.flags else 0
    cands = pb.cand_arrays() if pb.cands is not None else None
    ra = (pb.run_claims, pb.run_pod_off, pb.run_prio, pb.run_out)
    try:
        run = Running(pkg, *ra, out_off=pb.run_out_off)
        if pb.error:
            try:
                outs, _ = W.enqueue(pb.claims, pb.pod_off, pb.prio, run, cands, fl, (pb.out_off, pb.n_out))
            except A.DraError as e:                      # refused on the host: nothing was enqueued on any rank
                assert e.code == A.E_INVAL, what
                outs = None
            if outs is not None:
                for r, c in enumerate(W.ctxs):
                    with pytest.raises(A.DraError) as e:
                        c.sync()
                    assert e.value.code == A.E_INVAL, (what, r)
                for r, o in enumerate(outs):
                    assert all((t.cpu().numpy() == 0x5C).all() for t in o), f"{what}: rank {r} wrote an output"
        else:
            W.check(pb.claims, pb.pod_off, pb.prio, ra, run, cands, fl, what, (pb.out_off, pb.n_out), pb.run_out_off)
        for r, c in enumerate(W.ctxs):
            if pb.error:
                assert c.get_inventory().tobytes() == pb.gpus.tobytes(), f"{what}: rank {r}'s live inventory changed"
            c.reset_inventory()
            assert c.get_inventory().tobytes() == pb.gpus.tobytes(), f"{what}: rank {r}'s pristine inventory changed"
    finally:
        W.close()


def test_sharded_random_problems(pkg):
    @settings(max_examples=N_EX or 40, deadline=None, suppress_health_check=list(HealthCheck), derandomize=N_EX == 0,
              database=None)
    @given(place_problems(), st.sampled_from(CONFIGS))
    def run(pb, cfg):
        _sharded(pkg, pb, *cfg, what=pb.what)
    run()


def test_sharded_fixtures(pkg, monkeypatch):
    pbs = _pp_fixture_problems(monkeypatch)
    for i, pb in enumerate(pbs):
        for world, kind in CONFIGS:
            _sharded(pkg, pb, world, kind, what=f"fixture {i}")
