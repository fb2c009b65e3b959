"""GPU suite: preemption with disruption budgets on a sharded world (dra_preempt_pdb_batch_global_device).  World contexts
of this process on ONE device, as in test_gpu_shard_preempt.py.  Every rank's eight outputs must be byte for byte the
oracle's answer on the world's state; world 1 is the single-inventory call; a bad budget index fails every rank with
nothing written, and the next call on the world works."""
import os
import subprocess
import sys

import numpy as np
import pytest

import preempt_oracle as P
import preempt_pdb_oracle as PB
from test_gpu_preempt_pdb import NAMES, budgets
from test_gpu_shard_preempt import World, _cands, _dev, _nn, _running
from test_gpu_shard_unsuitable import _bounds

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE = 0xFFFFFFFF
SENTINEL = 0x5C


class Budgets:
    """run_pdb and allowed on the device, and the dra_disruption_budgets struct pointing at them"""

    def __init__(self, pkg, run_pdb, allowed, n_pdb=None):
        self.keep = [_dev(np.asarray(run_pdb, np.uint32)), _dev(np.asarray(allowed, np.int32))]
        self.struct = pkg.api.DisruptionBudgets(self.keep[0].data_ptr() if len(run_pdb) else None,
                                                self.keep[1].data_ptr() if len(allowed) else None,
                                                len(allowed) if n_pdb is None else n_pdb)


def enqueue(W, claims, pod_off, prio, run, bud, cands=None, max_victims=16, flags=0, pairs=True):
    """the call on every rank; returns (per-rank sentinel-filled outputs, sizes, n_pod)"""
    import torch
    n_pod = len(pod_off) - 1
    cn, co = (None, None) if cands is None else cands
    n_pair = n_pod * _nn(W.w) if co is None else int(co[-1])
    keep = [_dev(claims), _dev(pod_off), _dev(prio)] + ([None, None] if cn is None else [_dev(cn), _dev(co)])
    sizes = (n_pair, n_pair * 4, n_pod * 4, n_pod, n_pod * 4, n_pod * max_victims * 4, n_pair * 4, n_pod * 4)
    outs = [[torch.full((s + 16,), SENTINEL, dtype=torch.uint8, device="cuda:0") for s in sizes] for _ in W.ctxs]
    torch.cuda.synchronize()
    ptr = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    for c, o in zip(W.ctxs, outs):
        c.preempt_pdb_global_device(keep[0].data_ptr(), len(claims), keep[1].data_ptr(), keep[2].data_ptr(), n_pod,
                                    ptr(keep[3]), ptr(keep[4]), n_pair, run.struct, None if bud is None else bud.struct,
                                    o[0].data_ptr() if pairs else None, o[1].data_ptr() if pairs else None,
                                    o[6].data_ptr() if pairs else None, o[2].data_ptr(), o[3].data_ptr(),
                                    o[4].data_ptr(), o[7].data_ptr(), o[5].data_ptr() if max_victims else None,
                                    max_victims, flags)
    return outs, (keep, sizes, n_pod)


def call(W, claims, pod_off, prio, run, bud, cands=None, max_victims=16, flags=0, pairs=True):
    outs, (keep, sizes, n_pod) = enqueue(W, claims, pod_off, prio, run, bud, cands, max_victims, flags, pairs)
    for c in W.ctxs:
        c.sync()
    res = []
    dt = (np.uint8, np.uint32, np.uint32, np.uint8, np.uint32, np.uint32, np.uint32, np.uint32)
    for r, o in enumerate(outs):
        hs = [t.cpu().numpy() for t in o]
        for i, (h, s) in enumerate(zip(hs, sizes)):
            assert (h[s:] == SENTINEL).all(), f"rank {r} wrote past {NAMES[i]}"
            if not pairs and i in (0, 1, 6):
                assert (h == SENTINEL).all(), f"rank {r} wrote {NAMES[i]} without being asked"
        got = [h[:s].view(d) for h, s, d in zip(hs, sizes, dt)]
        got[5] = got[5].reshape(n_pod, max_victims)
        res.append(got)
    return res


def _same(got, ref, what, pairs=True):
    for i, (name, x, y) in enumerate(zip(NAMES, got, ref)):
        if not pairs and i in (0, 1, 6):
            continue
        if x.tobytes() != y.tobytes():
            bad = np.flatnonzero(x.reshape(-1) != y.reshape(-1))[:5]
            pytest.fail(f"{what}: {name} differs at {bad}: device {x.reshape(-1)[bad]} oracle {y.reshape(-1)[bad]}")


def _oracle(pkg, gpus, w, cands, mv, flags, run_pdb, allowed):
    cn, co = (None, None) if cands is None else cands
    return PB.preempt_pdb(gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off,
                         w.run_prio, w.run_out, run_pdb, allowed, None, cn, co, mv,
                         P.F_EXHAUSTIVE if flags & pkg.api.F_EXHAUSTIVE else 0)


COMBOS = [(0, "dense", 16, True), (1, "cands", 3, False), (0, "cands", 2, True), (1, "dense", 0, True)]


@pytest.mark.parametrize("world,kind", [(1, "even"), (2, "uneven"), (3, "empty"), (4, "even")])
@pytest.mark.parametrize("width", [8, 16, 32])
def test_matches_oracle(pkg, world, kind, width):
    w = pkg.synth.preempt(n_node=24, gpus_per_node=width, n_pending=60, seed=world * 10 + width)
    W = World(pkg, w, world, _bounds(_nn(w), world, kind))
    rng = np.random.default_rng(world + width)
    try:
        run, viol = _running(pkg, w), 0
        for f, form, mv, pairs in COMBOS:
            flags = f * pkg.api.F_EXHAUSTIVE
            cands = None if form == "dense" else _cands(rng, len(w.prio), _nn(w), 16)
            run_pdb, allowed = budgets(rng, len(w.run_prio))
            ref = _oracle(pkg, W.state(), w, cands, mv, flags, run_pdb, allowed)
            viol += int(ref[7].sum())
            got = call(W, w.claims, w.pod_off, w.prio, run, Budgets(pkg, run_pdb, allowed), cands, mv, flags, pairs)
            for r, g in enumerate(got):
                _same(g, ref, f"w{world} {kind} width {width} rank {r} f{flags} {form} mv{mv}", pairs)
        assert viol > 0
    finally:
        W.close()


def test_world_one_is_the_single_inventory_call(pkg):
    w = pkg.synth.preempt(n_node=20, gpus_per_node=8, n_pending=80, seed=2)
    W = World(pkg, w, 1, [0, _nn(w)], export=False)
    rng = np.random.default_rng(5)
    try:
        run = _running(pkg, w)
        for flags in (0, pkg.api.F_EXHAUSTIVE):
            for cands in (None, _cands(rng, len(w.prio), _nn(w), 7)):
                run_pdb, allowed = budgets(rng, len(w.run_prio))
                cn, co = (None, None) if cands is None else cands
                single = W.ctxs[0].preempt_pdb(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio,
                                               w.run_out, run_pdb, allowed, None, cn, co, 8, flags)
                got = call(W, w.claims, w.pod_off, w.prio, run, Budgets(pkg, run_pdb, allowed), cands, 8, flags)[0]
                _same(got, single, f"world 1 f{flags}")
        assert "preempt_shard" in W.ctxs[0].last_chain()
    finally:
        W.close()


def test_no_budgets_is_the_budget_free_call(pkg):
    w = pkg.synth.preempt(n_node=24, gpus_per_node=8, n_pending=40, seed=9)
    W = World(pkg, w, 3, _bounds(_nn(w), 3, "uneven"))
    try:
        run = _running(pkg, w)
        ref = _oracle(pkg, W.state(), w, None, 8, 0, None, None)
        for bud in (None, Budgets(pkg, [], []), Budgets(pkg, np.full(len(w.run_prio), NONE, np.uint32), [0])):
            for r, g in enumerate(call(W, w.claims, w.pod_off, w.prio, run, bud, None, 8)):
                _same(g, ref, f"no budgets rank {r}")
    finally:
        W.close()


def test_bad_budget_fails_every_rank(pkg):
    A = pkg.api
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=20, seed=17)
    W = World(pkg, w, 3, _bounds(_nn(w), 3, "uneven"))
    try:
        run = _running(pkg, w)
        run_pdb = np.zeros(len(w.run_prio), np.uint32)
        run_pdb[-1] = 1                                   # n_pdb is 1
        outs, _ = enqueue(W, w.claims, w.pod_off, w.prio, run, Budgets(pkg, run_pdb, [0]))
        for r, c in enumerate(W.ctxs):
            with pytest.raises(A.DraError) as e:
                c.sync()
            assert e.value.code == A.E_INVAL, r
        for r, o in enumerate(outs):
            assert all((t.cpu().numpy() == SENTINEL).all() for t in o), f"rank {r} wrote an output"
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
            _same(g, ref, f"after the fault rank {r}")
    finally:
        W.close()


def test_multi_process_preempt_pdb():
    """tests/multi_gpu_shard_preempt_pdb_check.py under torchrun: one process per GPU, peers mapped with IPC handles."""
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = min(n, 4)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", "29647",
                        os.path.join(ROOT, "tests", "multi_gpu_shard_preempt_pdb_check.py")],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
