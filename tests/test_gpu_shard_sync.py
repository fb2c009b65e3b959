"""GPU suite: the inventory sync of a sharded world (dra_shard_sync_inventory_device).  World contexts of this process on ONE
device, wired with dra_comm_init_local / dra_peer_import_local like test_gpu_shard_pods.py.  The CPU oracle runs every call
on ONE whole inventory; after a sync every rank's live inventory must be byte for byte that inventory, every rank's own
range must be what it held before, and calls under a new shard map must answer as the oracle does on that state."""
import numpy as np
import pytest

import shard_world as S

pytestmark = pytest.mark.gpu
N_POD_UNS = 300


def _world(pkg, w, world, bounds, stray_rank, max_pairs=None):
    return S.World(pkg, w.table, w.node_off, w.gpus, world, bounds, stray_rank, n_out_max=1 << 16, pairs=max_pairs)


def _deallocate(W, claims, out, out_off):
    for c in W.ctxs:                                     # every rank applies every gathered record
        c.deallocate(claims, out, out_off)


def _mixed_sequence(pkg, oracle, W, w, rng, state):
    """Sharded Allocate, sharded pods Allocate first-fit and exhaustive, then every rank deallocates the Allocate's and the
    first-fit pods' gathered records.  Returns the oracle's state of the one whole inventory after the same calls."""
    R, api = pkg.records, pkg.api
    claims = S.shared_mixed(pkg, w, rng)
    out_off, n_out = R.out_offsets(claims, w.n_node)
    ref, state = oracle.allocate(state, w.node_off, w.table, claims, out_off, int(n_out))
    S.same_tables(S.allocate(W, claims, out_off, int(n_out)), ref, "sharded Allocate")
    assert (ref["status"] == 0).any() and (ref["profile"][ref["status"] == 0] == R.PROFILE_SHARED).any()
    done = [(claims, ref, out_off)]
    for flags, oflags in ((0, 0), (api.F_EXHAUSTIVE, oracle.F_EXHAUSTIVE)):
        pc, po, poo, pn = S.malformed_mixed(pkg, w, W.bounds, rng, True)
        ref, state = oracle.allocate_pods(state, w.node_off, w.table, pc, po, poo, pn, oflags)
        S.same_tables(S.pods(W, pc, po, poo, pn, flags), ref, f"sharded pods Allocate flags {flags}")
        done.append((pc, ref, poo))
    for c, out, off in done[:2]:
        state = oracle.deallocate(state, c, out, off, n_node=w.n_node)
        _deallocate(W, c, out, off)
    W.assert_ranges(None, state, "after the mixed sequence")
    return state


def _sync_and_check(W, state, what):
    before = W.inventories()
    W.sync_inventory()
    for r, (b, a) in enumerate(zip(before, W.inventories())):
        g0, g1 = W.gpu_range(r)
        assert a[g0:g1].tobytes() == b[g0:g1].tobytes(), f"{what}: the sync changed rank {r}'s own range"
        assert a.tobytes() == state.tobytes(), f"{what}: rank {r} inventory after the sync differs from the oracle's"


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_sync_after_mixed_sequence(pkg, oracle, world):
    """After one sync every rank holds the world's state, byte for byte; a second sync changes nothing; the pristine copy
    is untouched (DRA_F_FRESH_INVENTORY still starts from the loaded inventory).  World 1: the call enqueues nothing."""
    R, api = pkg.records, pkg.api
    rng = np.random.default_rng(100 + world)
    w = pkg.synth.mixed(2400, 31, 70 + world, invalid=True)
    kind = {1: "even", 2: "uneven", 3: "empty", 4: "uneven"}[world]
    W = _world(pkg, w, world, S.bounds(w.n_node, world, kind), world - 1)
    try:
        state = _mixed_sequence(pkg, oracle, W, w, rng, w.gpus.copy())
        if world > 1:
            assert any(inv.tobytes() != state.tobytes() for inv in W.inventories()), "no rank's copy was stale"
            assert any((inv["share_cnt"] >= 0x8000).any() for inv in W.inventories()) and (state["share_cnt"] < 0x8000).all(), \
                "the per-rank Deallocate wrapped no share count outside a rank's range"
        l0 = [c.launch_count() for c in W.ctxs]
        _sync_and_check(W, state, "first sync")
        if world == 1:
            assert W.ctxs[0].launch_count() == l0[0], "world 1: the sync enqueued a kernel"
        else:
            assert all(c.launch_count() == l + 2 for c, l in zip(W.ctxs, l0))
        _sync_and_check(W, state, "second sync")
        # the pristine copy: a fresh-inventory sharded Allocate answers from the loaded inventory
        claims = S.shared_mixed(pkg, w, rng)
        out_off, n_out = R.out_offsets(claims, w.n_node)
        ref, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, claims, out_off, int(n_out))
        S.same_tables(S.allocate(W, claims, out_off, int(n_out), api.F_FRESH_INVENTORY), ref, "fresh Allocate after a sync")
        W.assert_ranges(None, ref_inv, "fresh Allocate after a sync")
    finally:
        W.close()


def test_sync_across_several_copy_ctas(pkg, oracle):
    """An inventory wide enough for k_isync_copy to run several CTAs (one per 256 GPUs, up to SMs / 4): the elected CTA
    publishes the verdict and the others wait for it before they copy.  Three syncs with the state changing in between, so
    both staging parities are used and the third finds the first one's stale records in its staging."""
    R, api = pkg.records, pkg.api
    rng = np.random.default_rng(17)
    w = pkg.synth.mixed(3000, 300, 17, invalid=True)
    assert w.n_gpu > 4 * 256, "the inventory must span at least five copy CTAs"
    W = _world(pkg, w, 4, [0, 40, 40, 170, 300], 2)
    try:
        state = _mixed_sequence(pkg, oracle, W, w, rng, w.gpus.copy())
        _sync_and_check(W, state, "first sync")
        claims = S.shared_mixed(pkg, w, rng)
        out_off, n_out = R.out_offsets(claims, w.n_node)
        ref, state = oracle.allocate(state, w.node_off, w.table, claims, out_off, int(n_out))
        S.same_tables(S.allocate(W, claims, out_off, int(n_out)), ref, "sharded Allocate between syncs")
        _sync_and_check(W, state, "second sync")
        pc, po, poo, pn = S.malformed_mixed(pkg, w, W.bounds, rng, True)
        ref, state = oracle.allocate_pods(state, w.node_off, w.table, pc, po, poo, pn, oracle.F_EXHAUSTIVE)
        S.same_tables(S.pods(W, pc, po, poo, pn, api.F_EXHAUSTIVE), ref, "pods Allocate between syncs")
        _deallocate(W, pc, ref, poo)
        state = oracle.deallocate(state, pc, ref, poo, n_node=w.n_node)
        _sync_and_check(W, state, "third sync")
    finally:
        W.close()


def _ipc_rank(rank, n_node, q_out, q_in, results, done):
    """One rank of a two-process world on GPU 0: export with an inventory of n_node nodes, import the peer's handle."""
    import importlib
    pkg = importlib.import_module("k8s-dra-driver_b200")
    w = pkg.synth.mixed(600, n_node, 3, invalid=True)
    c = pkg.api.Context(device=0)
    try:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        c.comm_init_local(rank, 2); c.set_shard_map([0, 5, n_node], 0)
        h = c.shard_export(64)
        q_out.put(h)
        other = q_in.get(timeout=120)
        try:
            c.peer_import([h, other] if rank == 0 else [other, h])
            results.put((rank, pkg.api.OK))
        except pkg.api.DraError as e:
            results.put((rank, e.code))
        done.wait(120)                                   # the exports stay alive until both ranks have imported
    finally:
        c.close()


@pytest.mark.parametrize("sizes", [(11, 11), (11, 23)])
def test_ipc_import_requires_alike_exports(pkg, sizes):
    """Over IPC handles (two processes, here on one GPU), dra_peer_import reads each peer's layout from its buffer.  Alike
    exports import; a peer that exported a larger inventory, and so a larger sync staging, is refused with DRA_E_INVAL on
    both sides.  Only host calls run: no kernel of the two processes waits for the other."""
    import multiprocessing as mp
    ctx = mp.get_context("spawn")
    qs, results, done = [ctx.Queue(), ctx.Queue()], ctx.Queue(), ctx.Event()
    procs = [ctx.Process(target=_ipc_rank, args=(r, sizes[r], qs[r], qs[1 - r], results, done)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        got = dict(results.get(timeout=300) for _ in procs)
    finally:
        done.set()
        for p in procs:
            p.join(120)
            if p.is_alive():
                p.kill(); p.join()
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    want = pkg.api.OK if sizes[0] == sizes[1] else pkg.api.E_INVAL
    assert got == {0: want, 1: want}, got


def _pods_for_unsuitable(pkg, w, rng):
    claims = w.claims.copy()
    pod_off = S.pod_cuts(rng, 900, N_POD_UNS - 60)
    return claims[: pod_off[-1]], pod_off


def test_reshard_keeps_allocations(pkg, oracle):
    """Map A, the mixed sequence, sync, map B (boundaries moved, an empty range, another stray rank), then sharded Allocate,
    UnsuitableNodes (dense and candidate lists, first-fit and exhaustive) and pods Allocate: every table and bitmap equals
    the oracle's on the one whole inventory.  After a further sync, dra_unsuitable_batch on one rank alone gives the
    sharded answer."""
    R, api = pkg.records, pkg.api
    rng = np.random.default_rng(7)
    world = 3
    w = pkg.synth.mixed(2400, 31, 91, invalid=True)
    bounds_a, bounds_b = [0, 3, 9, 31], [0, 20, 20, 31]
    W = _world(pkg, w, world, bounds_a, 2, max_pairs=N_POD_UNS * w.n_node)
    try:
        state = _mixed_sequence(pkg, oracle, W, w, rng, w.gpus.copy())
        _sync_and_check(W, state, "sync under map A")
        W.remap(bounds_b, 0)
        W.assert_ranges(None, state, "after the re-map")
        claims = S.shared_mixed(pkg, w, rng)
        out_off, n_out = R.out_offsets(claims, w.n_node)
        ref, state = oracle.allocate(state, w.node_off, w.table, claims, out_off, int(n_out))
        S.same_tables(S.allocate(W, claims, out_off, int(n_out)), ref, "sharded Allocate under map B")
        uc, upo = _pods_for_unsuitable(pkg, w, rng)
        n_pod = len(upo) - 1
        cn, co = S.candidates(rng, n_pod, w.n_node)
        forms = [("dense", None, None) + S.dense(n_pod, w.n_node), ("candidates", cn, co, cn, co)]
        for flags, oflags in ((0, 0), (api.F_EXHAUSTIVE, oracle.F_EXHAUSTIVE)):
            for name, dn, do, on, oo in forms:
                ref_bits = oracle.unsuitable(state, w.node_off, w.table, uc, upo, on, oo, flags=oflags)
                for r, b in enumerate(S.unsuitable(W, uc, upo, None if dn is None else (dn, do), flags)):
                    assert b.tobytes() == ref_bits.tobytes(), f"UnsuitableNodes {name} flags {flags}: rank {r} differs"
        for flags, oflags in ((0, 0), (api.F_EXHAUSTIVE, oracle.F_EXHAUSTIVE)):
            pc, po, poo, pn = S.malformed_mixed(pkg, w, W.bounds, rng, True)
            ref, state = oracle.allocate_pods(state, w.node_off, w.table, pc, po, poo, pn, oflags)
            S.same_tables(S.pods(W, pc, po, poo, pn, flags), ref, f"pods Allocate under map B flags {flags}")
        W.assert_ranges(None, state, "after the calls under map B")
        _sync_and_check(W, state, "sync under map B")
        for flags, oflags in ((0, 0), (api.F_EXHAUSTIVE, oracle.F_EXHAUSTIVE)):
            sharded = S.unsuitable(W, uc, upo, (cn, co), flags)[0]
            assert sharded.tobytes() == oracle.unsuitable(state, w.node_off, w.table, uc, upo, cn, co, flags=oflags).tobytes()
            single = W.ctxs[1].unsuitable(uc, upo, cn, co, flags)
            assert single.tobytes() == sharded.tobytes(), f"flags {flags}: one rank's dra_unsuitable_batch differs"
    finally:
        W.close()


def test_errors_change_nothing(pkg, oracle):
    """DRA_E_STATE with nothing enqueued and no inventory changed: no shard map (none, or a bare dra_set_shard), no export,
    an export without an import, an export made before the inventory was loaded, an inventory that grew after the export.
    A world that refused a call syncs correctly afterwards."""
    api = pkg.api
    w = pkg.synth.mixed(600, 11, 3, invalid=True)
    big = pkg.synth.mixed(600, 23, 4, invalid=True)
    assert big.n_gpu > w.n_gpu

    def refused(c):
        inv, n = c.get_inventory(), c.launch_count()
        assert c._lib.dra_shard_sync_inventory_device(c._h) == api.E_STATE
        assert c.launch_count() == n and c.get_inventory().tobytes() == inv.tobytes()

    with api.Context(device=0) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off); c.comm_init_local(0, 2)
        refused(c)                                                       # no shard at all
        c.set_shard(0, 5, take_stray=True)
        refused(c)                                                       # a bare dra_set_shard
        c.set_shard_map([0, 5, 11], 0)
        refused(c)                                                       # no export
        c.shard_export(64, 0, want_handle=False)
        refused(c)                                                       # export without import
    ctxs = [api.Context(device=0) for _ in range(2)]
    try:
        for r, c in enumerate(ctxs):                                     # export BEFORE the inventory is loaded
            c.comm_init_local(r, 2); c.shard_export(64, 0, want_handle=False)
        for c in ctxs:
            c.peer_import_local(ctxs)
        for c in ctxs:
            c.set_table(w.table); c.set_inventory(w.gpus, w.node_off); c.set_shard_map([0, 5, 11], 1)
        refused(ctxs[0])
    finally:
        for c in ctxs:
            c.close()
    W = _world(pkg, w, 2, [0, 5, 11], 1)
    try:
        for c in W.ctxs:                                                 # the inventory grows after the export
            c.set_inventory(big.gpus, big.node_off); c.set_shard_map([0, 9, 23], 1)
        refused(W.ctxs[0])
        for c in W.ctxs:                                                 # back to the exported size: the sync works
            c.set_inventory(w.gpus, w.node_off); c.set_shard_map([0, 5, 11], 1)
        rng = np.random.default_rng(5)
        state = _mixed_sequence(pkg, oracle, W, w, rng, w.gpus.copy())
        _sync_and_check(W, state, "after refused calls")
    finally:
        W.close()
