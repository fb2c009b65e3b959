"""GPU suite: pod capacity on a sharded world (dra_pod_capacity_batch_global_device, spec §16 "Sharded form").  World
contexts of this process on ONE device, wired with dra_comm_init_local / dra_peer_import_local like
test_gpu_shard_preempt.py.  Every rank's four outputs must be byte for byte the oracle's answer on the world's state: the
inventory each rank holds for its own node range."""
import numpy as np
import pytest

import capacity_oracle as K
import preempt_oracle as P
import shard_world as S
from test_pod_capacity import _flat, problem

pytestmark = pytest.mark.gpu
SENTINEL = 0x5C
ALL = (True, True, True)
EXH = 0x4                                                # DRA_F_EXHAUSTIVE


def _world(pkg, gpus, node_off, table, world, bounds, invs=None, max_pairs=1 << 16, n_out=64, **kw):
    """rank r serving [bounds[r], bounds[r+1]) of the inventory it was given; max_pairs None: exported without room for
    the call"""
    return S.World(pkg, table, node_off, gpus if invs is None else invs, world, bounds, n_out_max=n_out, capacity=max_pairs,
                   **kw)


def _check(W, claims, pod_off, cands, mc, flags, want, what):
    cn, co = (None, None) if cands is None else cands
    ref = K.capacity(W.state(), W.node_off, W.table, claims, pod_off, cn, co, mc, K.F_EXHAUSTIVE if flags else 0)
    for r, got in enumerate(S.capacity(W, claims, pod_off, cands, mc, flags, want, SENTINEL)):
        S.same(got, ref, S.CAPACITY_NAMES, f"{what} rank {r}")
    return ref


WANTS = [ALL, (False, True, False), (True, False, True), (False, False, False)]


@pytest.mark.parametrize("world,kind", [(1, "even"), (2, "even"), (2, "uneven"), (3, "empty"), (3, "uneven"),
                                        (4, "even"), (4, "empty")])
@pytest.mark.parametrize("width", [8, 16, 32])
def test_matches_oracle(pkg, world, kind, width):
    """Dense and candidate forms, both flags, every optional-output choice, rows of W = 8, 16 and 32 lanes: every rank's
    outputs against the oracle on the world's state; the chain bit and the launch count."""
    A = pkg.api
    w = pkg.synth.preempt(n_node=24, gpus_per_node=width, n_pending=60, seed=world * 10 + width)
    W = _world(pkg, w.gpus, w.node_off, w.table, world, S.bounds(S.nn(w), world, kind))
    try:
        rng = np.random.default_rng(world + width)
        n_pod = len(w.pod_off) - 1
        for i, (flags, form) in enumerate([(0, "dense"), (A.F_EXHAUSTIVE, "cands"), (0, "cands"), (A.F_EXHAUSTIVE, "dense")]):
            cands = None if form == "dense" else S.cands(rng, n_pod, S.nn(w), 16)
            ref = _check(W, w.claims, w.pod_off, cands, (64, 3, 1, 300)[i], flags, WANTS[i], f"w{world} {kind} {form} f{flags}")
            assert ref[0].max() > 0 and (ref[0] == 0).any()
        c = W.ctxs[0]
        before = c._lib.dra_launch_count(c._h)
        S.capacity(W, w.claims, w.pod_off)
        assert c._lib.dra_launch_count(c._h) - before == (4 if world > 1 else 3)
        assert c.last_chain() == {"pod_capacity_shard"}
    finally:
        W.close()


@pytest.mark.parametrize("world", [2, 3])
def test_random_problems(pkg, world):
    """The CPU suite's generator: fragmented nodes of every width, pods of 0 to 33 claims with invalid ones, candidate
    lists with duplicates and strays, or the dense form; random ranges."""
    stops = set()
    for seed in range(8):
        g, off, t, c, pod_off, cands = problem(500 * world + seed, n_node=9, n_run=60)
        rng = np.random.default_rng(seed)
        cuts = sorted(rng.integers(0, 10, world - 1).tolist())
        W = _world(pkg, g, off, t, world, [0] + cuts + [9])
        try:
            fc = None if cands is None else _flat(cands)
            for flags in (0, EXH):
                ref = _check(W, c, pod_off, fc, 2 if flags else 64, flags, WANTS[seed % 4], f"seed {seed} f{flags}")
                stops |= set(ref[1].tolist())
        finally:
            W.close()
    assert {K.ST_OK, K.ST_POD, K.ST_INVALID} <= stops


def test_diverged_copies(pkg):
    """Each rank holds the real world on its own range only, the empty inventory elsewhere: the sharded answer is the
    oracle's on the real world, while rank 0's dra_pod_capacity_batch (its own copy taken for the world) is not.  No
    inventory word changes."""
    w = pkg.synth.preempt(n_node=24, gpus_per_node=8, n_pending=60, seed=21)
    world = 3
    bounds = S.bounds(S.nn(w), world, "even")
    invs = []
    for r in range(world):
        g = w.empty.copy()
        a, b = int(w.node_off[bounds[r]]), int(w.node_off[bounds[r + 1]])
        g[a:b] = w.gpus[a:b]
        invs.append(g)
    W = _world(pkg, w.gpus, w.node_off, w.table, world, bounds, invs=invs)
    try:
        assert W.state().tobytes() == w.gpus.tobytes()
        cands = S.cands(np.random.default_rng(4), len(w.pod_off) - 1, S.nn(w), 9)
        for flags in (0, EXH):
            for cd in (None, cands):
                ref = _check(W, w.claims, w.pod_off, cd, 64, flags, ALL, f"diverged f{flags}")
                cn, co = (None, None) if cd is None else cd
                single = W.ctxs[0].pod_capacity(w.claims, w.pod_off, cn, co, 64, bool(flags))
                assert single[0].tobytes() != ref[0].tobytes(), "the workload does not expose stale copies"
        for r, c in enumerate(W.ctxs):
            assert c.get_inventory().tobytes() == invs[r].tobytes(), f"rank {r}'s live inventory changed"
            c.reset_inventory()
            assert c.get_inventory().tobytes() == invs[r].tobytes(), f"rank {r}'s pristine inventory changed"
    finally:
        W.close()


def test_the_real_flow(pkg):
    """Pods placed by the sharded pods Allocate, then the sharded capacity with no sync: the oracle's answer on the world's
    state, and the same as dra_pod_capacity_batch on rank 0 after the inventory sync."""
    import torch
    w = pkg.synth.preempt(n_node=24, gpus_per_node=8, n_pending=50, seed=13)
    world = 3
    bounds = S.bounds(S.nn(w), world, "uneven")
    n_out = len(w.run_claims)
    W = _world(pkg, w.empty, w.node_off, w.table, world, bounds, invs=[w.empty] * world, n_out=n_out)
    try:
        d_rc, d_rpo = S.dev(w.run_claims), S.dev(w.run_pod_off)
        torch.cuda.synchronize()
        for c in W.ctxs:
            c.allocate_pods_global_device(d_rc.data_ptr(), len(w.run_claims), d_rpo.data_ptr(), len(w.run_pod_off) - 1,
                                          None, n_out, 0)
        cands = S.cands(np.random.default_rng(6), len(w.pod_off) - 1, S.nn(w), 12)
        got_all = S.capacity(W, w.claims, w.pod_off, cands, 64, EXH)
        state = W.state()
        assert state.tobytes() != w.empty.tobytes()
        befores = [c.get_inventory() for c in W.ctxs]
        assert any(b.tobytes() != state.tobytes() for b in befores)          # no rank holds the world before the sync
        ref = K.capacity(state, w.node_off, w.table, w.claims, w.pod_off, *cands, 64, K.F_EXHAUSTIVE)
        for r, got in enumerate(got_all):
            S.same(got, ref, S.CAPACITY_NAMES, f"real flow rank {r}")
        for r, c in enumerate(W.ctxs):
            assert c.get_inventory().tobytes() == befores[r].tobytes(), f"rank {r}: live inventory changed"
        for c in W.ctxs:
            c.shard_sync_inventory_device()
        for c in W.ctxs:
            c.sync()
        single = W.ctxs[0].pod_capacity(w.claims, w.pod_off, *cands, 64, True)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(single, got_all[0]))
        for c in W.ctxs:
            c.reset_inventory()
            assert c.get_inventory().tobytes() == w.empty.tobytes(), "pristine inventory changed"
    finally:
        W.close()


def test_world_one_is_the_single_inventory_call(pkg):
    w = pkg.synth.preempt(n_node=20, gpus_per_node=16, n_pending=80, seed=2)
    W = _world(pkg, w.gpus, w.node_off, w.table, 1, [0, S.nn(w)], export=False)
    try:
        rng = np.random.default_rng(0)
        for flags in (0, EXH):
            for cands in (None, S.cands(rng, len(w.pod_off) - 1, S.nn(w), 7)):
                cn, co = (None, None) if cands is None else cands
                single = W.ctxs[0].pod_capacity(w.claims, w.pod_off, cn, co, 9, bool(flags))
                S.same(S.capacity(W, w.claims, w.pod_off, cands, 9, flags)[0], single, S.CAPACITY_NAMES, f"world 1 f{flags}")
        assert W.ctxs[0].last_chain() == {"pod_capacity_shard"}
    finally:
        W.close()


def test_consecutive_calls_of_changing_size(pkg):
    """Calls of growing and shrinking size, interleaved with sharded UnsuitableNodes and sharded preemption on the same
    world: call parity and the shared peer buffer."""
    w = pkg.synth.preempt(n_node=24, gpus_per_node=8, n_pending=120, seed=31, fill=60)
    world = 4
    n_pod_max = len(w.pod_off) - 1
    n_pair_max = n_pod_max * S.nn(w)
    W = _world(pkg, w.gpus, w.node_off, w.table, world, S.bounds(S.nn(w), world, "uneven"), max_pairs=n_pair_max,
               n_out=max(1, len(w.run_claims)), pairs=n_pair_max, preempt=(n_pod_max, n_pair_max, 16))
    try:
        run = S.Running(pkg, w.run_claims, w.run_pod_off, w.run_prio, w.run_out)
        rng = np.random.default_rng(8)
        for it, n in enumerate((40, 120, 7, 90, 1, 120)):
            po = w.pod_off[: n + 1]
            claims = w.claims[: int(po[-1])]
            flags = EXH * (it % 2)
            cands = None if it % 3 == 0 else S.cands(rng, n, S.nn(w), 1 + it)
            _check(W, claims, po, cands, (64, 5, 1)[it % 3], flags, WANTS[it % 4], f"call {it}")
            bits = S.unsuitable(W, claims, po, flags=flags)
            assert all(b.tobytes() == bits[0].tobytes() for b in bits)
            prio = w.prio[:n]
            got = S.preempt(W, claims, po, prio, run, None, 16, flags)
            ref = P.preempt(W.state(), w.node_off, w.table, claims, po, prio, w.run_claims, w.run_pod_off, w.run_prio,
                            w.run_out, None, None, None, 16, P.F_EXHAUSTIVE if flags else 0)
            for r, g in enumerate(got):
                S.same(g, ref, S.PREEMPT_NAMES, f"preemption after call {it} rank {r}")
    finally:
        W.close()


@pytest.mark.parametrize("kind", ["pod_off order", "pod_off span", "cand_off order", "cand_off span"])
def test_device_faults_fail_every_rank(pkg, kind):
    A = pkg.api
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=20, seed=17)
    world = 3
    W = _world(pkg, w.gpus, w.node_off, w.table, world, S.bounds(S.nn(w), world, "uneven"))
    try:
        po = w.pod_off.copy()
        cn, co = S.cands(np.random.default_rng(0), len(po) - 1, S.nn(w), 4)
        if kind == "pod_off order":
            po[5] = po[6] + 1
        elif kind == "pod_off span":
            po[-1] -= 1
        elif kind == "cand_off order":
            co[3] = co[4] + 2
        else:
            co[0] = 1
        outs = S.capacity(W, w.claims, po, (cn, co), 64, 0, sentinel=SENTINEL, expect=A.E_INVAL)
        for r, o in enumerate(outs):
            assert all((h == SENTINEL).all() for h in o), f"{kind}: rank {r} wrote an output"
        # the next valid call on the same world matches the oracle
        _check(W, w.claims, w.pod_off, S.cands(np.random.default_rng(2), len(po) - 1, S.nn(w), 4), 64, EXH, ALL, f"after {kind}")
    finally:
        W.close()


@pytest.mark.parametrize("world", [1, 2, 3])
def test_pods_without_candidates(pkg, world):
    """Every candidate list empty (n_pair 0, n_pod > 0): no pair is written, and every rank's pod_total and pod_nodes are
    0.  The exchange still runs, and the next call on the same world is right."""
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=20, seed=9, fill=40)   # room for copies
    n_pod = len(w.pod_off) - 1
    W = _world(pkg, w.gpus, w.node_off, w.table, world, S.bounds(S.nn(w), world, "uneven"))
    try:
        empty = (np.zeros(0, np.uint32), np.zeros(n_pod + 1, np.uint32))
        for flags in (0, EXH):
            ref = _check(W, w.claims, w.pod_off, empty, 64, flags, ALL, f"w{world} no candidates f{flags}")
            assert len(ref[0]) == 0 and not ref[2].any() and not ref[3].any()
            c = W.ctxs[0]
            before = c._lib.dra_launch_count(c._h)
            got = S.capacity(W, w.claims, w.pod_off, empty, 64, flags)
            assert c._lib.dra_launch_count(c._h) - before == (3 if world > 1 else 2)   # prep, (push,) merge
            for r, g in enumerate(got):
                assert g[2].tolist() == [0] * n_pod and g[3].tolist() == [0] * n_pod, f"rank {r}"
        # some pods with candidates, some without
        cn, co = S.cands(np.random.default_rng(3), n_pod, S.nn(w), 3)
        co[1:6] = co[1]                                   # pods 1..4: no candidates
        keep_n = np.concatenate([cn[: co[1]], cn[co[1] + 12:]]).astype(np.uint32)
        co[6:] -= 12
        ref = _check(W, w.claims, w.pod_off, (keep_n, co), 64, EXH, ALL, f"w{world} mixed")
        assert not ref[2][1:5].any() and ref[2].any()
    finally:
        W.close()


def test_host_side_errors(pkg):
    import torch
    A = pkg.api
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=20, seed=5)
    n_pod, n_node = len(w.pod_off) - 1, S.nn(w)
    W = _world(pkg, w.gpus, w.node_off, w.table, 2, S.bounds(n_node, 2, "even"), max_pairs=n_pod * n_node)
    try:
        c = W.ctxs[0]
        keep = [S.dev(w.claims), S.dev(w.pod_off)]
        cn, co = S.cands(np.random.default_rng(1), n_pod, n_node, 3)
        d_cn, d_co = S.dev(cn), S.dev(co)
        o = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda:0").data_ptr()
        launches = c._lib.dra_launch_count(c._h)

        def call(n_pair=n_pod * n_node, mc=4, flags=0, copies=o, cands=(None, None), n=n_pod):
            with pytest.raises(A.DraError) as e:
                c.pod_capacity_global_device(keep[0].data_ptr(), len(w.claims), keep[1].data_ptr(), n, *cands, n_pair, mc,
                                             copies, o, o, o, flags)
            return e.value.code

        assert call(flags=0x1) == A.E_INVAL                                   # unknown flags
        assert call(flags=A.F_FRESH_INVENTORY) == A.E_INVAL
        assert call(mc=0) == A.E_INVAL and call(mc=65536) == A.E_INVAL       # max_copies outside [1, 65535]
        assert call(cands=(d_cn.data_ptr(), None), n_pair=int(co[-1])) == A.E_INVAL   # one candidate array alone
        assert call(cands=(None, d_co.data_ptr()), n_pair=int(co[-1])) == A.E_INVAL
        assert call(n_pair=n_pod * n_node + 1) == A.E_INVAL                   # dense n_pair != n_pod * n_node
        assert call(cands=(d_cn.data_ptr(), d_co.data_ptr()), n_pair=0xFFFFFFF1) == A.E_INVAL
        assert call(cands=(d_cn.data_ptr(), d_co.data_ptr()), n_pair=n_pod * n_node + 1) == A.E_INVAL   # above max_pairs
        assert call(n=(1 << 26) + 1, cands=(d_cn.data_ptr(), d_co.data_ptr()), n_pair=int(co[-1])) == A.E_INVAL
        assert call(copies=None) == A.E_INVAL                                 # no pair_copies with pairs to answer
        assert c._lib.dra_launch_count(c._h) == launches
        with pytest.raises(A.DraError) as e:
            c.set_shard_capacity(10)                                          # after the export
        assert e.value.code == A.E_STATE
        # no pods: OK, nothing enqueued on any rank
        for ctx in W.ctxs:
            ctx.pod_capacity_global_device(keep[0].data_ptr(), 0, keep[1].data_ptr(), 0, None, None, 0, 4, None)
            ctx.sync()
        assert c._lib.dra_launch_count(c._h) == launches
    finally:
        W.close()
    # a bare dra_set_shard, a world with no export, one exported without dra_set_shard_capacity
    for kw in (dict(bare=True), dict(export=False), dict(max_pairs=None)):
        W = _world(pkg, w.gpus, w.node_off, w.table, 2, S.bounds(n_node, 2, "even"), **kw)
        try:
            with pytest.raises(A.DraError) as e:
                S.capacity(W, w.claims, w.pod_off)
            assert e.value.code == A.E_STATE, kw
            if kw == dict(max_pairs=None):                # also with no pairs at all: nothing reserved to push into
                c = W.ctxs[0]
                launches = c._lib.dra_launch_count(c._h)
                empty = (np.zeros(0, np.uint32), np.zeros(n_pod + 1, np.uint32))
                with pytest.raises(A.DraError) as e:
                    S.capacity(W, w.claims, w.pod_off, empty)
                assert e.value.code == A.E_STATE
                assert c._lib.dra_launch_count(c._h) == launches
        finally:
            W.close()
    with A.Context(device=0) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        keep = [S.dev(w.claims), S.dev(w.pod_off)]
        with pytest.raises(A.DraError) as e:
            c.pod_capacity_global_device(keep[0].data_ptr(), len(w.claims), keep[1].data_ptr(), n_pod, None, None,
                                         n_pod * n_node, 4, keep[0].data_ptr())
        assert e.value.code == A.E_STATE
    # a peer set up for a different max_pairs is refused at the import
    ctxs = [A.Context(device=0) for _ in range(2)]
    try:
        for r, c in enumerate(ctxs):
            c.comm_init_local(r, 2)
            c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
            c.set_shard_map(S.bounds(n_node, 2, "even"))
            c.set_shard_capacity(100 * (r + 1))
            c.shard_export(64, 0, want_handle=False)
        with pytest.raises(A.DraError) as e:
            ctxs[0].peer_import_local(ctxs)
        assert e.value.code == A.E_INVAL
    finally:
        for c in ctxs:
            c.close()
