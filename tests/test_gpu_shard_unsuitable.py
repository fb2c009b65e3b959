"""GPU suite: UnsuitableNodes on a sharded world (dra_unsuitable_batch_global_device).  World contexts of this process on
ONE device, wired with dra_comm_init_local / dra_peer_import_local like test_gpu_shard.py.  Every rank's bitmap must be
byte for byte the oracle's answer on the world's real state: the inventory each rank holds for its own node range."""
import numpy as np
import pytest

import shard_world as S

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5


def _world(pkg, w, world, bounds, max_pairs, inv=None, attrs=None, sels=None):
    """every rank holding the whole inventory, the table exported for w's records"""
    return S.World(pkg, w.table, w.node_off, w.gpus if inv is None else inv, world, bounds, attrs=attrs, sels=sels,
                   n_out_max=max(1, w.n_out), pairs=max_pairs)


def _call(W, claims, pod_off, cn=None, co=None, flags=0):
    return S.unsuitable(W, claims, pod_off, None if cn is None else (cn, co), flags, sentinel=SENTINEL)


@pytest.mark.parametrize("world", [1, 2, 3, 4])
@pytest.mark.parametrize("workload", ["pods", "mixed"])
def test_matches_oracle(pkg, oracle, world, workload):
    """Dense and candidate-list forms, first-fit and exhaustive, every rank's whole bitmap against the oracle."""
    R = pkg.records
    rng = np.random.default_rng(world * 10 + (workload == "mixed"))
    attrs = sels = None
    if workload == "pods":
        pw, pod_off = pkg.synth.pods(900, 29, world)
        w, claims = pw, pw.claims
        inv = pw.gpus
    else:
        w = pkg.synth.mixed(2400, 31, 50 + world)
        attrs, sels = pkg.synth.with_selectors(w, world)
        inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims[:800])[1]        # partly filled
        claims = w.claims.copy()
        pod_off = S.pod_cuts(rng, w.n_claim, 700, big=True)
        for p in range(len(pod_off) - 1):                 # most pods on one node, as a scheduler would ask
            if rng.integers(0, 10):
                claims["node"][pod_off[p]: pod_off[p + 1]] = claims["node"][pod_off[p]]
    n_pod, n_node = len(pod_off) - 1, w.n_node
    cn, co = S.candidates(rng, n_pod, n_node)
    dn, do = S.dense(n_pod, n_node)
    bounds = S.bounds(n_node, world, "uneven" if world == 3 else "even")
    W = _world(pkg, w, world, bounds, max(n_pod * n_node, int(co[-1])), inv, attrs, sels)
    oracle.set_selectors(attrs, sels)
    try:
        for flags, oflags in ((0, 0), (pkg.api.F_EXHAUSTIVE, oracle.F_EXHAUSTIVE)):
            ref_dense = oracle.unsuitable(inv, w.node_off, w.table, claims, pod_off, dn, do, flags=oflags)
            ref_cand = oracle.unsuitable(inv, w.node_off, w.table, claims, pod_off, cn, co, flags=oflags)
            for r, got in enumerate(_call(W, claims, pod_off, flags=flags)):
                assert got.tobytes() == ref_dense.tobytes(), f"dense, flags {flags}, rank {r}"
            for r, got in enumerate(_call(W, claims, pod_off, cn, co, flags=flags)):
                assert got.tobytes() == ref_cand.tobytes(), f"candidates, flags {flags}, rank {r}"
            assert ref_dense.any() and not np.all(ref_dense == 0xFF)
    finally:
        oracle.set_selectors()
        W.close()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_allocate_then_unsuitable(pkg, oracle, world):
    """The gap the call closes: after a sharded Allocate without F_FRESH_INVENTORY the ranks' copies diverge (each is right
    for its own nodes only).  The sharded call answers on the real state; the single-inventory call on rank 0 does not."""
    R = pkg.records
    w = pkg.synth.cfg2(6000, 40)
    ranges = pkg.shard.plan(w.claims["node"], w.n_node, world)
    bounds = [x[0] for x in ranges] + [ranges[-1][1]]
    n_pod = 600
    pods = w.claims[:n_pod].copy()
    pod_off = np.arange(n_pod + 1, dtype=np.uint32)
    W = _world(pkg, w, world, bounds, n_pod * w.n_node)
    try:
        S.allocate(W, w.claims, None, w.n_out)
        _, real = oracle.allocate(w.gpus, w.node_off, w.table, w.claims)
        dn, do = S.dense(n_pod, w.n_node)
        for flags, oflags in ((0, 0), (pkg.api.F_EXHAUSTIVE, oracle.F_EXHAUSTIVE)):
            ref = oracle.unsuitable(real, w.node_off, w.table, pods, pod_off, dn, do, flags=oflags)
            for r, got in enumerate(_call(W, pods, pod_off, flags=flags)):
                assert got.tobytes() == ref.tobytes(), f"rank {r}, flags {flags}"
        stale = W.ctxs[0].unsuitable(pods, pod_off)
        ref = oracle.unsuitable(real, w.node_off, w.table, pods, pod_off, dn, do)
        assert stale.tobytes() != ref.tobytes(), "the workload does not expose the stale copies"
    finally:
        W.close()


def test_edge_shapes(pkg, oracle):
    """Empty node ranges, n_pair not a multiple of 8 or 32, n_pair == 0, candidates past the inventory, one candidate."""
    w = pkg.synth.mixed(1200, 23, 71, invalid=True)
    rng = np.random.default_rng(5)
    world = 4
    W = _world(pkg, w, world, S.bounds(w.n_node, world, "empty"), 4096)
    try:
        for n_pod in (1, 3, 5, 7):                        # dense n_pair = n_pod * 23: odd, never a multiple of 8
            pod_off = np.linspace(0, 40 * n_pod, n_pod + 1).astype(np.uint32)
            c = w.claims[: pod_off[-1]]
            dn, do = S.dense(n_pod, w.n_node)
            ref = oracle.unsuitable(w.gpus, w.node_off, w.table, c, pod_off, dn, do)
            for got in _call(W, c, pod_off):
                assert got.tobytes() == ref.tobytes()
        for n_pair in (1, 31, 33, 63, 65, 4096):
            pod_off = np.array([0, 2, 2, 5], dtype=np.uint32)
            cand_off = np.array([0, n_pair // 3, n_pair // 2, n_pair], dtype=np.uint32)
            cand_nodes = rng.integers(0, w.n_node + 3, n_pair).astype(np.uint32)
            c = w.claims[:5]
            for flags, oflags in ((0, 0), (pkg.api.F_EXHAUSTIVE, oracle.F_EXHAUSTIVE)):
                ref = oracle.unsuitable(w.gpus, w.node_off, w.table, c, pod_off, cand_nodes, cand_off, flags=oflags)
                for got in _call(W, c, pod_off, cand_nodes, cand_off, flags=flags):
                    assert got.tobytes() == ref.tobytes(), f"n_pair {n_pair}"
        # n_pair == 0 (two pods without candidates): nothing to decide, no output buffer needed, the next call still works
        z = S.dev(np.zeros(3, dtype=np.uint32))
        W.each(lambda r, c: c.unsuitable_global_device(0, 0, z.data_ptr(), 2, z.data_ptr(), z.data_ptr(), 0, 0, 0))
        pod_off = np.array([0, 3], dtype=np.uint32)
        dn, do = S.dense(1, w.n_node)
        ref = oracle.unsuitable(w.gpus, w.node_off, w.table, w.claims[:3], pod_off, dn, do)
        for got in _call(W, w.claims[:3], pod_off):
            assert got.tobytes() == ref.tobytes()
    finally:
        W.close()


def test_world1_equals_single_inventory_call(pkg, oracle):
    w = pkg.synth.mixed(2000, 29, 88)
    rng = np.random.default_rng(1)
    pod_off = S.pod_cuts(rng, w.n_claim, 500, big=True)
    cn, co = S.candidates(rng, len(pod_off) - 1, w.n_node)
    W = _world(pkg, w, 1, [0, w.n_node], 0)
    try:
        c = W.ctxs[0]
        for flags in (0, pkg.api.F_EXHAUSTIVE):
            assert _call(W, w.claims, pod_off, flags=flags)[0].tobytes() == c.unsuitable(w.claims, pod_off, flags=flags).tobytes()
            assert _call(W, w.claims, pod_off, cn, co, flags=flags)[0].tobytes() == \
                c.unsuitable(w.claims, pod_off, cn, co, flags=flags).tobytes()
    finally:
        W.close()


def test_consecutive_calls_interleaved_with_sharded_allocates(pkg, oracle):
    """Calls of changing size, first-fit and exhaustive, between sharded Allocates on the same world: call parity, the
    sequence flags and the peer buffer shared with the allocation gather.  Each answer is checked on the state the
    allocates left."""
    R = pkg.records
    world = 3
    w = pkg.synth.cfg2(4000, 30)
    ranges = pkg.shard.plan(w.claims["node"], w.n_node, world)
    bounds = [x[0] for x in ranges] + [ranges[-1][1]]
    W = _world(pkg, w, world, bounds, 500 * w.n_node)
    rng = np.random.default_rng(3)
    try:
        state = w.gpus
        for step, (n_pod, flags) in enumerate([(500, 0), (37, pkg.api.F_EXHAUSTIVE), (211, 0), (1, 0), (333, pkg.api.F_EXHAUSTIVE), (64, 0)]):
            if step % 2 == 0:                             # a sharded allocate on the live inventory (part of the claims)
                lo = step * 300
                part = w.claims[lo: lo + 600]
                S.allocate(W, part, None, len(part))
                _, state = oracle.allocate(state, w.node_off, w.table, part)
            pods = w.claims[rng.integers(0, w.n_claim, n_pod)]
            pod_off = np.arange(n_pod + 1, dtype=np.uint32)
            oflags = oracle.F_EXHAUSTIVE if flags else 0
            if step % 3 == 1:
                cn, co = S.candidates(rng, n_pod, w.n_node)
                ref = oracle.unsuitable(state, w.node_off, w.table, pods, pod_off, cn, co, flags=oflags)
                got = _call(W, pods, pod_off, cn, co, flags=flags)
            else:
                dn, do = S.dense(n_pod, w.n_node)
                ref = oracle.unsuitable(state, w.node_off, w.table, pods, pod_off, dn, do, flags=oflags)
                got = _call(W, pods, pod_off, flags=flags)
            for r, g in enumerate(got):
                assert g.tobytes() == ref.tobytes(), f"step {step} rank {r}"
    finally:
        W.close()


def test_errors(pkg, oracle):
    """Host-side checks return before anything is enqueued; device-side offset checks fail at sync on EVERY rank (the exchange
    still completes); either way the next valid call works."""
    import torch
    E = pkg.api
    w = pkg.synth.mixed(600, 11, 3)
    world = 2
    bounds = [0, 5, 11]
    n_pod = 20
    pod_off = np.arange(0, 3 * n_pod + 1, 3, dtype=np.uint32)
    claims = w.claims[: pod_off[-1]]
    dn, do = S.dense(n_pod, w.n_node)
    ref = oracle.unsuitable(w.gpus, w.node_off, w.table, claims, pod_off, dn, do)
    d_c, d_p = S.dev(claims), S.dev(pod_off)
    bits = torch.zeros(64, dtype=torch.uint8, device="cuda:0")
    torch.cuda.synchronize()

    def raw(c, **k):
        a = dict(claims=d_c.data_ptr(), n_claim=len(claims), pod_off=d_p.data_ptr(), n_pod=n_pod, cn=None, co=None,
                 n_pair=n_pod * w.n_node, flags=0)
        a.update(k)
        return c._lib.dra_unsuitable_batch_global_device(c._h, a["claims"], a["n_claim"], a["pod_off"], a["n_pod"], a["cn"],
                                                         a["co"], a["n_pair"], bits.data_ptr(), a["flags"])

    # no shard, no export
    with E.Context(device=0) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        assert raw(c) == E.E_STATE
        c.comm_init_local(0, 2); c.set_shard_map(bounds, 0)
        assert raw(c) == E.E_STATE                       # world 2 without export + import
        c.set_shard_pairs(10)
        c.shard_export(16, 0, want_handle=False)
        assert c._lib.dra_set_shard_pairs(c._h, 100) == E.E_STATE   # after the export
    W = _world(pkg, w, world, bounds, n_pod * w.n_node)
    try:
        c0 = W.ctxs[0]
        assert raw(c0, n_pair=n_pod * w.n_node + 1) == E.E_INVAL                 # dense n_pair != n_pod * n_node
        assert raw(c0, flags=0x80) == E.E_INVAL                                  # unknown flag
        assert raw(c0, n_pod=n_pod + 1, n_pair=(n_pod + 1) * w.n_node) == E.E_INVAL   # above max_pairs
        assert raw(c0, cn=d_p.data_ptr()) == E.E_INVAL                           # cand_nodes without cand_off
        for r, got in enumerate(_call(W, claims, pod_off)):
            assert got.tobytes() == ref.tobytes(), f"after host-side errors, rank {r}"
        # device-side: pod_off not monotone / not spanning the claims, cand_off not spanning the pairs
        bad_po = pod_off.copy(); bad_po[5] = bad_po[7] + 1
        short_po = pod_off.copy(); short_po[-1] -= 1
        cn, co = S.candidates(np.random.default_rng(0), n_pod, w.n_node)
        bad_co = co.copy(); bad_co[-1] -= 1
        for po, c_nodes, c_off, n_pair in ((bad_po, None, None, None), (short_po, None, None, None),
                                           (pod_off, cn, bad_co, int(co[-1]))):
            n_pair = n_pod * w.n_node if n_pair is None else n_pair
            outs = S.unsuitable(W, claims, po, None if c_nodes is None else (c_nodes, c_off), n_pair=n_pair,
                                sentinel=SENTINEL, expect=E.E_INVAL)
            for o in outs:                                # nothing was evaluated: every bit zero
                assert not o[0][: (n_pair + 7) // 8].any()
            for r, got in enumerate(_call(W, claims, pod_off)):
                assert got.tobytes() == ref.tobytes(), f"after a device-side error, rank {r}"
    finally:
        W.close()
