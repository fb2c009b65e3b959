"""GPU suite: preemption with disruption budgets on a sharded world (dra_preempt_pdb_batch_global_device).  World contexts
of this process on ONE device, as in test_gpu_shard_preempt.py.  Every rank's eight outputs must be byte for byte the
oracle's answer on the world's state; world 1 is the single-inventory call; a bad budget index fails every rank with
nothing written, and the next call on the world works."""
import numpy as np
import pytest

import preempt_oracle as P
import shard_world as S
from test_gpu_preempt_pdb import NAMES, budgets

pytestmark = pytest.mark.gpu
NONE = 0xFFFFFFFF
SENTINEL = 0x5C


class Budgets:
    """run_pdb and allowed on the device, and the dra_disruption_budgets struct pointing at them"""

    def __init__(self, pkg, run_pdb, allowed, n_pdb=None):
        self.keep = [S.dev(np.asarray(run_pdb, np.uint32)), S.dev(np.asarray(allowed, np.int32))]
        self.struct = pkg.api.DisruptionBudgets(self.keep[0].data_ptr() if len(run_pdb) else None,
                                                self.keep[1].data_ptr() if len(allowed) else None,
                                                len(allowed) if n_pdb is None else n_pdb)


def call(W, claims, pod_off, prio, run, bud, cands=None, max_victims=16, flags=0, pairs=True, expect=0):
    return S.preempt(W, claims, pod_off, prio, run, cands, max_victims, flags, pairs, pdb=True, bud=bud, sentinel=SENTINEL,
                     expect=expect)


def _world(pkg, w, world, bounds, **kw):
    """rank r serving [bounds[r], bounds[r+1]) of the inventory, preemption and its pairs reserved"""
    return S.World(pkg, w.table, w.node_off, w.gpus, world, bounds, n_out_max=max(1, len(w.run_claims)),
                   preempt=(4096, 200000, 64), pairs=200000, **kw)


def _running(pkg, w):
    return S.Running(pkg, w.run_claims, w.run_pod_off, w.run_prio, w.run_out)


def _oracle(pkg, gpus, w, cands, mv, flags, run_pdb, allowed):
    cn, co = (None, None) if cands is None else cands
    return P.preempt_pdb(gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off,
                         w.run_prio, w.run_out, run_pdb, allowed, None, cn, co, mv,
                         P.F_EXHAUSTIVE if flags & pkg.api.F_EXHAUSTIVE else 0)


COMBOS = [(0, "dense", 16, True), (1, "cands", 3, False), (0, "cands", 2, True), (1, "dense", 0, True)]


@pytest.mark.parametrize("world,kind", [(1, "even"), (2, "uneven"), (3, "empty"), (4, "even")])
@pytest.mark.parametrize("width", [8, 16, 32])
def test_matches_oracle(pkg, world, kind, width):
    w = pkg.synth.preempt(n_node=24, gpus_per_node=width, n_pending=60, seed=world * 10 + width)
    W = _world(pkg, w, world, S.bounds(S.nn(w), world, kind))
    rng = np.random.default_rng(world + width)
    try:
        run, viol = _running(pkg, w), 0
        for f, form, mv, pairs in COMBOS:
            flags = f * pkg.api.F_EXHAUSTIVE
            cands = None if form == "dense" else S.cands(rng, len(w.prio), S.nn(w), 16)
            run_pdb, allowed = budgets(rng, len(w.run_prio))
            ref = _oracle(pkg, W.state(), w, cands, mv, flags, run_pdb, allowed)
            viol += int(ref[7].sum())
            got = call(W, w.claims, w.pod_off, w.prio, run, Budgets(pkg, run_pdb, allowed), cands, mv, flags, pairs)
            for r, g in enumerate(got):
                S.same(g, ref, NAMES, f"w{world} {kind} width {width} rank {r} f{flags} {form} mv{mv}")
        assert viol > 0
    finally:
        W.close()


def test_world_one_is_the_single_inventory_call(pkg):
    w = pkg.synth.preempt(n_node=20, gpus_per_node=8, n_pending=80, seed=2)
    W = _world(pkg, w, 1, [0, S.nn(w)], export=False)
    rng = np.random.default_rng(5)
    try:
        run = _running(pkg, w)
        for flags in (0, pkg.api.F_EXHAUSTIVE):
            for cands in (None, S.cands(rng, len(w.prio), S.nn(w), 7)):
                run_pdb, allowed = budgets(rng, len(w.run_prio))
                cn, co = (None, None) if cands is None else cands
                single = W.ctxs[0].preempt_pdb(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio,
                                               w.run_out, run_pdb, allowed, None, cn, co, 8, flags)
                got = call(W, w.claims, w.pod_off, w.prio, run, Budgets(pkg, run_pdb, allowed), cands, 8, flags)[0]
                S.same(got, single, NAMES, f"world 1 f{flags}")
        assert "preempt_shard" in W.ctxs[0].last_chain()
    finally:
        W.close()


def test_no_budgets_is_the_budget_free_call(pkg):
    w = pkg.synth.preempt(n_node=24, gpus_per_node=8, n_pending=40, seed=9)
    W = _world(pkg, w, 3, S.bounds(S.nn(w), 3, "uneven"))
    try:
        run = _running(pkg, w)
        ref = _oracle(pkg, W.state(), w, None, 8, 0, None, None)
        for bud in (None, Budgets(pkg, [], []), Budgets(pkg, np.full(len(w.run_prio), NONE, np.uint32), [0])):
            for r, g in enumerate(call(W, w.claims, w.pod_off, w.prio, run, bud, None, 8)):
                S.same(g, ref, NAMES, f"no budgets rank {r}")
    finally:
        W.close()


def test_bad_budget_fails_every_rank(pkg):
    A = pkg.api
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=20, seed=17)
    W = _world(pkg, w, 3, S.bounds(S.nn(w), 3, "uneven"))
    try:
        run = _running(pkg, w)
        run_pdb = np.zeros(len(w.run_prio), np.uint32)
        run_pdb[-1] = 1                                   # n_pdb is 1
        outs = call(W, w.claims, w.pod_off, w.prio, run, Budgets(pkg, run_pdb, [0]), expect=A.E_INVAL)
        for r, o in enumerate(outs):
            assert all((h == SENTINEL).all() for h in o), f"rank {r} wrote an output"
        # host-side: n_pdb without allowed, running pods without run_pdb; nothing is enqueued
        for bud in (Budgets(pkg, run_pdb, [], n_pdb=1), Budgets(pkg, [], [0])):
            for c in W.ctxs:
                with pytest.raises(A.DraError) as e:
                    c.preempt_pdb_global_device(0, 0, 0, 0, 1, None, None, 0, run.struct, bud.struct, None, None, None,
                                                0, 0, 0, None, None, 0)
                assert e.value.code == A.E_INVAL
        # the next call on the world works
        run_pdb[-1] = 0
        ref = _oracle(pkg, W.state(), w, None, 16, 0, run_pdb, [0])
        for r, g in enumerate(call(W, w.claims, w.pod_off, w.prio, run, Budgets(pkg, run_pdb, [0]))):
            S.same(g, ref, NAMES, f"after the fault rank {r}")
    finally:
        W.close()
