"""CPU model of the sharded preempt-and-place exchange (dra_preempt_place_batch_global_device, spec §15 "Sharded form").

Each rank holds its own node range as authoritative and stale copies of the others.  The model runs the call's protocol
under random fair schedules: every rank pushes its own GPU range to every peer; deliveries are delayed and reordered at
random; a rank assembles the world's state only once every peer's range has arrived, runs §15 on that private copy with
the C oracle, and writes back its own range alone.  Against both oracles of tests/preempt_place_oracle.py, for worlds of
1 to 5 ranks and random partitions (empty ranges included): no deadlock, every rank's outputs equal and equal to §15 on
the world's state, the same result for every partition, no GPU written outside a rank's range, and every victim on its
evictor's chosen node, inside the range of the rank that released it."""
import importlib

import numpy as np
import pytest

from test_oracle_properties import _dicts
from test_pod_mode import _tbl
from test_preempt import _flat, _outs, mig_running, occupied

import preempt_place_oracle as PP

R = importlib.import_module("k8s-dra-driver_b200").records
synth = importlib.import_module("k8s-dra-driver_b200").synth
NONE = 0xFFFFFFFF


def _partition(rng, n_node, world):
    cuts = np.sort(rng.integers(0, n_node + 1, size=world - 1))
    return [0] + [int(x) for x in cuts] + [n_node]


def run_protocol(rng, state, stale, off, bounds, call):
    """One call on every rank under a random fair schedule.  Returns (per-rank outputs, per-rank inventories after)."""
    world = len(bounds) - 1
    rng_of = [(int(off[bounds[r]]), int(off[bounds[r + 1]])) for r in range(world)]
    held = []
    for r in range(world):                              # own range authoritative, the rest stale
        g = stale.copy()
        a, b = rng_of[r]
        g[a:b] = state[a:b]
        held.append(g)
    in_flight = [(src, dst) for src in range(world) for dst in range(world) if src != dst]
    staged = [dict() for _ in range(world)]
    done = [None] * world
    for _ in range(100000):
        if all(d is not None for d in done):
            break
        ready = [r for r in range(world) if done[r] is None and len(staged[r]) == world - 1]
        moves = [("deliver", i) for i in range(len(in_flight))] + [("run", r) for r in ready]
        assert moves, "deadlock: nothing can move"
        kind, x = moves[rng.integers(len(moves))]
        if kind == "deliver":
            src, dst = in_flight.pop(x)
            a, b = rng_of[src]
            staged[dst][src] = held[src][a:b].copy()      # the sender's own range as it holds it
            continue
        g = held[x].copy()                              # the private copy of the world's state
        for src, recs in staged[x].items():
            a, b = rng_of[src]
            g[a:b] = recs
        out = call(g)
        a, b = rng_of[x]
        after = held[x].copy()
        after[a:b] = out[4][a:b]                        # the own range back, nothing else
        done[x] = (out[:4], after, held[x])
    else:
        pytest.fail("no progress")
    return done, rng_of


def _check_world(rng, w_gpus, stale, off, table, claims, pod_off, prio, run, cands, flags, n_parts=4, out_off=None):
    rc, rpo, rpr, ro = run
    cn, co = (None, None) if cands is None else cands
    ref = PP.preempt_place(w_gpus, off, table, claims, pod_off, prio, rc, rpo, rpr, ro, None, cn, co, out_off, None, flags)
    call = lambda g: PP.preempt_place(g, off, table, claims, pod_off, prio, rc, rpo, rpr, ro, None, cn, co, out_off, None, flags)  # noqa: E731
    n_node = len(off) - 1
    for _ in range(n_parts):
        world = int(rng.integers(1, 6))
        bounds = _partition(rng, n_node, world)
        done, rng_of = run_protocol(rng, w_gpus, stale, off, bounds, call)
        world_after = w_gpus.copy()
        for r, (outs, after, before) in enumerate(done):
            for x, y in zip(outs, ref[:4]):
                assert x.tobytes() == y.tobytes(), f"rank {r} of {bounds}"
            a, b = rng_of[r]
            assert after[:a].tobytes() == before[:a].tobytes() and after[b:].tobytes() == before[b:].tobytes()
            world_after[a:b] = after[a:b]
        assert world_after.tobytes() == ref[4].tobytes(), f"world state after {bounds}"
        # every victim lies on its evictor's chosen node, inside the range of the rank that released it
        ev = ref[3]
        for v in np.flatnonzero(ev != NONE):
            node = int(ref[1][ev[v]])
            gpus = {int(ro["gpu"][i]) for i in range(rpo[v], rpo[v + 1]) if ro["status"][i] == 0}
            assert all(off[node] <= gg < off[node + 1] for gg in gpus)
            owner = next(r for r in range(len(bounds) - 1) if bounds[r] <= node < bounds[r + 1])
            a, b = rng_of[owner]
            assert all(a <= gg < b for gg in gpus)
    return ref


def _pods(*pods):
    from test_pod_mode import _mig
    c = _mig(R, [p for pod in pods for p in pod])
    off = np.zeros(len(pods) + 1, np.uint32)
    off[1:] = np.cumsum([len(p) for p in pods])
    return c, off


def _naive_agrees(g, off, t, c, po, prio, run, cands, flags):
    rc, rpo, rpr, ro = run
    cn, co = (None, None) if cands is None else _flat(cands)
    a = PP.preempt_place(g, off, t, c, po, prio, rc, rpo, rpr, ro, None, cn, co, None, None, flags)
    b = PP.preempt_place_naive(_dicts(g), [int(x) for x in off], _tbl(t), _dicts(c), [int(x) for x in po],
                               [int(x) for x in prio], cands, bool(flags & PP.F_EXHAUSTIVE), _dicts(rc),
                               [int(x) for x in rpo], [int(x) for x in rpr], _outs(ro))
    assert _outs(a[0]) == b[0] and list(a[1]) == b[1] and list(a[2]) == b[2] and list(a[3]) == b[3]


def _fixture_world():
    """four one-GPU MIG nodes: 1g pods at slice 0 on nodes 0 and 1 (prio 50, not evictable by prio 10), node 2 holds a 3g
    pod at 4 (prio 100) and a 1g at 0 (prio 1), node 3 a 1g at 0 (prio 2) and a 1g at 4 (prio 3)"""
    g, off = R.make_inventory([1, 1, 1, 1], mig=True)
    run = mig_running([(0, 0, 4, R.GI_3_SLICE, 50), (0, 4, 4, R.GI_3_SLICE, 50), (1, 0, 4, R.GI_3_SLICE, 50),
                       (1, 4, 4, R.GI_3_SLICE, 50), (2, 0, 1, R.GI_1_SLICE, 1), (2, 4, 4, R.GI_3_SLICE, 100),
                       (3, 0, 1, R.GI_1_SLICE, 2), (3, 4, 1, R.GI_1_SLICE, 3)], off)
    return occupied(g, run[0], run[3]), off, R.default_table(), run


@pytest.mark.parametrize("case", ["same_eviction", "evict_two_ranks", "tie", "search_limit", "duplicates_strays",
                                  "empty_33_invalid"])
def test_fixtures(case):
    g, off, t, run = _fixture_world()
    stale, _ = R.make_inventory([1, 1, 1, 1], mig=True)              # the stale copies: everything free
    rng = np.random.default_rng(len(case))
    flags = 0
    if case == "same_eviction":          # both need the prio-1 eviction on node 2; candidates list nodes 0, 1 first
        c, po = _pods([R.GI_3_SLICE], [R.GI_3_SLICE])
        cands = [[0, 1, 2, 3], [0, 1, 2, 3]]
    elif case == "evict_two_ranks":      # EVICT on node 2 and node 3, pre_better picks node 2 (lower victim priority)
        c, po = _pods([R.GI_3_SLICE])
        cands = [[3, 2]]
    elif case == "tie":                  # the same pair on two nodes: the earlier list position wins
        c, po = _pods([R.GI_1_SLICE])
        cands = [[3, 2]]
    elif case == "search_limit":
        c, po = _pods([R.GI_1_SLICE] * 6)
        cands = [[2, 0, 1]]
        flags = PP.F_EXHAUSTIVE
    elif case == "duplicates_strays":
        c, po = _pods([R.GI_3_SLICE], [R.GI_1_SLICE])
        cands = [[9, 2, 2, 7], [3, 3, 99]]
    else:
        c, po = _pods([], [R.GI_1_SLICE] * 33, [R.GI_1_SLICE])
        c["profile"][-1] = 0xEE                                          # an invalid claim
        cands = [[1, 2], [2], [0, 3]]
    prio = np.full(len(po) - 1, 10, np.int32)
    _naive_agrees(g, off, t, c, po, prio, run, cands, flags)
    cn, co = _flat(cands)
    ref = _check_world(rng, g, stale, off, t, c, po, prio, run, (cn, co), flags, n_parts=12)
    if case == "same_eviction":
        assert list(ref[1]) == [2, 3] and list(ref[2]) == [PP.EVICT, PP.EVICT]


@pytest.mark.parametrize("seed", range(8))
def test_random_worlds(seed):
    rng = np.random.default_rng(seed)
    w = synth.preempt(n_node=10, gpus_per_node=4 + 4 * (seed % 2), n_pending=30, seed=seed)
    stale = synth.preempt(n_node=10, gpus_per_node=4 + 4 * (seed % 2), n_pending=30, seed=seed + 100).gpus
    run = (w.run_claims, w.run_pod_off, w.run_prio, w.run_out)
    n_pod = len(w.pod_off) - 1
    for flags in (0, PP.F_EXHAUSTIVE):
        cands = None
        if flags:
            cn = rng.integers(0, 12, size=n_pod * 4).astype(np.uint32)       # duplicates and strays included
            cands = (cn, (np.arange(n_pod + 1) * 4).astype(np.uint32))
        _check_world(rng, w.gpus, stale, w.node_off, w.table, w.claims, w.pod_off, w.prio, run, cands, flags)
