"""GPU suite: pods Allocate (spec §12, dra_allocate_pods_batch) at its edges.

Every call goes through the raw ABI on sentinel-filled outputs SLACK records longer than n_out, and is compared byte for
byte with oracle.allocate_pods on the context's live inventory (on the pristine one under DRA_F_FRESH_INVENTORY): the
OutRecs, then the inventory.  Nothing may be written past n_out; slots no claim owns (out_off gaps) read back as 0.

* the pod sort: the pod records are bucketed by node with Allocate's counting sort (records naming no node are dropped),
  and a node's pods must stay in input order.  ROWS puts the pod and node counts on each side of each of the sort's
  thresholds (shapes from the SM count S) and asserts the chain and histogram tile that ran, under four distributions
* the walk: more nodes than the walk has warps, and DRA_F_FRESH_INVENTORY on a live state that differs from the pristine
  one, with pods on a third of the nodes: every other node comes back pristine (with the flag) or untouched (without)
* pod shapes and failure records, every out_off form, nodes of 0 to 32 GPUs (test_pods_edges.py)
* a slot range past n_out: DRA_E_INVAL before anything is enqueued, no output byte and no inventory word written, and
  the next call is right; slot ranges that end exactly at n_out are accepted
* the same shapes and faults on sharded worlds of one to three contexts on one device"""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

import test_pods_edges as E
import shard_world as S

pytestmark = pytest.mark.gpu
SENT, SLACK = 0xA5, 16
NONE = 0xFFFFFFFF
SORTABLE = 102_399                                 # (n_node + 1) u16 counters of the one-warp histogram in 200 KiB


@pytest.fixture(scope="module")
def pctx(pkg):
    c = pkg.api.Context(device=0)
    yield c
    c.close()


def _n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _load(ctx, pb):
    ctx.set_table(pb.table)
    ctx.set_inventory(pb.gpus, pb.node_off)


def raw_pods(pkg, ctx, pb, claims=None, out_off=None, n_out=None, flags=0):
    """dra_allocate_pods_batch on an output of sentinel bytes SLACK records longer than n_out: (rc, out)"""
    R = pkg.records
    claims = pb.claims if claims is None else claims
    out_off = pb.out_off if out_off is None else out_off
    n_out = pb.n_out if n_out is None else n_out
    out = np.full((max(n_out, 1) + SLACK) * 8, SENT, np.uint8).view(R.OUT_DTYPE)
    c = np.ascontiguousarray(claims, dtype=R.CLAIM_DTYPE)
    keep = c.copy()
    po = np.ascontiguousarray(pb.pod_off, dtype=np.uint32)
    oo = None if out_off is None else np.ascontiguousarray(out_off, dtype=np.uint32)
    p = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)      # noqa: E731
    rc = ctx._lib.dra_allocate_pods_batch(ctx._h, p(c), len(c), p(po), len(po) - 1, p(oo), p(out), n_out, flags)
    assert c.tobytes() == keep.tobytes(), "the call wrote the caller's claims"
    return rc, out


def _oflags(pkg, oracle, flags):
    return oracle.F_EXHAUSTIVE if flags & pkg.api.F_EXHAUSTIVE else 0


def check(pkg, oracle, ctx, pb, flags, what, start=None):
    """One call on pb against the oracle on the context's live inventory (start: another starting state, the pristine
    one for DRA_F_FRESH_INVENTORY).  Returns the oracle's OutRecs."""
    A = pkg.api
    before = ctx.get_inventory() if start is None else start
    ref, ref_inv = oracle.allocate_pods(before, pb.node_off, pb.table, pb.claims, pb.pod_off, pb.out_off, pb.n_out,
                                        _oflags(pkg, oracle, flags))
    rc, out = raw_pods(pkg, ctx, pb, flags=flags)
    assert rc == A.OK, f"{what}: rc {rc}"
    got = out[: pb.n_out]
    if got.tobytes() != ref.tobytes():
        bad = np.flatnonzero(got != ref)[:5]
        pytest.fail(f"{what}: OutRecs differ at slots {bad}: device {got[bad]} oracle {ref[bad]}")
    assert (out[pb.n_out:].view(np.uint8) == SENT).all(), f"{what}: written past n_out"
    after = ctx.get_inventory()
    if after.tobytes() != ref_inv.tobytes():
        bad = np.flatnonzero(after != ref_inv)[:5]
        pytest.fail(f"{what}: inventory differs at GPUs {bad}: device {after[bad]} oracle {ref_inv[bad]}")
    return ref


# ---- a. the pod sort at its thresholds ------------------------------------------------------------------------------
SORT8 = {"hist8", "scan8", "scatter"}
WARP = {"hist_warp", "scan", "scatter"}
SMALL = {"bucket_small"}
D4 = ("random", "hot", "nonode", "empty_ends")
# id, shape(S) -> (n_pod, n_node), chain, hist tile (0: no histogram kernel), both flags
ROWS = [
    # the one-CTA counting sort: 8,192 records, and its shared memory at 8,192 records (2,769 nodes)
    ("bucket_small_pods_max", lambda S: (8_192, S), SMALL, 0, True),
    ("hist8_pods_min", lambda S: (8_193, S), SORT8, 2048, True),
    ("bucket_small_smem_max", lambda S: (8_192, 2_769), SMALL, 0, True),
    ("bucket_small_smem_over", lambda S: (8_192, 2_770), SORT8, 2048, True),
    # CTA-wide histogram: 2048-record tiles up to S tiles, then grown tiles
    ("hist8_tile_fixed_max", lambda S: (S * 2048, 1_000), SORT8, 2048, False),
    ("hist8_tile_grown_min", lambda S: (S * 2048 + 1, 1_000), {"hist8_multi", "scan8", "scatter"}, 4096, False),
    # the scan of the tile histograms: one warp per node up to 524,288 counters, coalesced rows beyond
    ("scan8_max", lambda S: (S * 2048, 524_288 // S - 1), SORT8, 2048, False),
    ("scan_rows_min", lambda S: (S * 2048, 524_288 // S), {"hist8", "scan_rows", "scatter"}, 2048, False),
    # CTA-wide histogram while 8 x (n_node + 2) u16 counters fit 200 KiB, one-warp tiles beyond
    ("hist8_nodes_max", lambda S: (50_000, 12_798), SORT8, 2048, True),
    ("hist_warp_nodes_min", lambda S: (50_000, 12_799), WARP, 800, True),
    # the widest node range the sort takes
    ("sortable_max", lambda S: (50_000, SORTABLE), WARP, 800, False),
]
CASES = [pytest.param(r, d, id=f"{r[0]}-{d}") for r in ROWS for d in D4]


def sort_workload(R, n_pod, n_node, dist, seed=3):
    """Nodes of one and two MIG GPUs, pods of one to three 1g-7g claims, so a node's pods compete for it and a node's
    pods out of input order change the answer:
      random      about a quarter of the pods name n_node, n_node + 1000 or 0xFFFFFFFF
      hot         >= 90 % of the pods, and every one of the first 65,536, name node 1
      nonode      about 80 % of the pods name no node
      empty_ends  nodes 0 and n_node - 1 have no GPU, and about a quarter of the pods name one of them"""
    rng = np.random.default_rng(seed)
    widths = 1 + np.arange(n_node) % 2
    if dist == "empty_ends":
        widths[0] = widths[-1] = 0
    g, off = R.make_inventory(list(widths), mig=True)
    node = rng.integers(0, n_node, n_pod).astype(np.uint32)
    st = np.array(E.strays(n_node), np.uint32)
    if dist in ("random", "nonode"):
        m = rng.random(n_pod) < (0.25 if dist == "random" else 0.8)
        node[m] = st[rng.integers(0, 3, int(m.sum()))]
    elif dist == "hot":
        m = rng.random(n_pod) < 0.92
        m[:65_536] = True
        node[m] = 1
    else:
        node[::4] = np.where(rng.random(len(node[::4])) < 0.5, 0, n_node - 1)
    sizes = rng.integers(1, 4, n_pod)
    pod_off = np.zeros(n_pod + 1, np.uint32)
    pod_off[1:] = np.cumsum(sizes)
    c = E._mig(rng.choice(E.MIG_PROFILES, int(pod_off[-1])))
    c["node"] = np.repeat(node, sizes)
    return E.problem(f"{n_pod} pods x {n_node} nodes {dist}", g, off, R.default_table(), c, pod_off)


@pytest.mark.parametrize("row,dist", CASES)
def test_pod_sort_at_boundary(pkg, oracle, pctx, row, dist):
    R = pkg.records
    name, shape, chain, tile, both = row
    S = _n_sm()
    n_pod, n_node = shape(S)
    pb = sort_workload(R, n_pod, n_node, dist)
    for flags in ((0, pkg.api.F_EXHAUSTIVE) if both else (0,)):
        _load(pctx, pb)
        ref = check(pkg, oracle, pctx, pb, flags, f"{name} {dist} f{flags}: {pb.name}, {S} SMs")
        got = pctx.last_chain()
        assert got == chain, f"{name}: {n_pod} pods x {n_node} nodes on {S} SMs took {sorted(got)}"
        assert pctx.last_hist_tile() == tile, f"{name}: hist tile {pctx.last_hist_tile()}"
        st = ref["status"]
        assert (st == R.ST_OK).any() and (st == R.ST_POD).any(), f"{name}: no pod lost its node to the pods before it"
        assert (st == R.ST_INVALID).any() == (dist in ("random", "nonode")), name


# ---- b. the walk ----------------------------------------------------------------------------------------------------
def _spread(R, n, seed, per_node=3, nodes=None):
    """n nodes of one and two MIG GPUs; about per_node pods of 1-3 claims on each node of `nodes` (default: every node),
    a twentieth of them naming no node, in random order"""
    rng = np.random.default_rng(seed)
    g, off = R.make_inventory(list(1 + np.arange(n) % 2), mig=True)
    nodes = np.arange(n) if nodes is None else np.asarray(nodes)
    node = rng.permutation(np.repeat(nodes, per_node)).astype(np.uint32)
    m = rng.random(len(node)) < 0.05
    node[m] = NONE
    sizes = rng.integers(1, 4, len(node))
    pod_off = np.zeros(len(node) + 1, np.uint32)
    pod_off[1:] = np.cumsum(sizes)
    c = E._mig(rng.choice(E.MIG_PROFILES, int(pod_off[-1])))
    c["node"] = np.repeat(node, sizes)
    return E.problem(f"{len(node)} pods on {n} nodes", g, off, R.default_table(), c, pod_off)


def _walk_sizes():
    """the walk launches min((n + 3) / 4, 8 S) CTAs of 4 warps: at 32 S nodes each warp owns one node, past it one warp
    owns two, and at 96 S + 5 every warp owns three or four"""
    S = _n_sm()
    return {"one": 32 * S, "two": 32 * S + 1, "several": 96 * S + 5}


@pytest.mark.parametrize("size", ["one", "two", "several"])
def test_walk_over_more_nodes_than_warps(pkg, oracle, pctx, size):
    R = pkg.records
    n = _walk_sizes()[size]
    pb = _spread(R, n, seed=n)
    for flags in (0, pkg.api.F_EXHAUSTIVE):
        _load(pctx, pb)
        ref = check(pkg, oracle, pctx, pb, flags, f"walk {size} f{flags}: {pb.name}")
        assert (ref["status"] == R.ST_POD).any() and (ref["status"] == R.ST_OK).sum() > n


def test_fresh_inventory_on_a_changed_live_state(pkg, oracle, pctx):
    """A first call puts a 1g on every node, so the live state differs from the pristine one everywhere.  A call with
    DRA_F_FRESH_INVENTORY and pods on a third of the nodes then starts from the pristine state: every node without a pod
    comes back pristine.  Without the flag, those nodes keep the live state."""
    A, R = pkg.api, pkg.records
    n = _walk_sizes()["several"]
    g, off = R.make_inventory(list(1 + np.arange(n) % 2), mig=True)
    one = E._mig([R.GI_1_SLICE] * n)
    one["node"] = np.arange(n)
    first = E.problem("1g everywhere", g, off, R.default_table(), one, np.arange(n + 1))
    third = np.arange(0, n, 3)
    pb = _spread(R, n, seed=11, per_node=2, nodes=third)
    pb.gpus = g                                          # (the same inventory, rebuilt)
    quiet = np.ones(len(g), bool)
    for k in third:
        quiet[off[k]: off[k + 1]] = False
    assert quiet.sum() > len(g) // 2
    _load(pctx, first)
    for flags in (A.F_FRESH_INVENTORY, A.F_FRESH_INVENTORY | A.F_EXHAUSTIVE, 0, A.F_EXHAUSTIVE):
        check(pkg, oracle, pctx, first, 0, "1g everywhere")
        live = pctx.get_inventory()
        assert (live["busy"][off[:-1]] != g["busy"][off[:-1]]).all()
        fresh = bool(flags & A.F_FRESH_INVENTORY)
        check(pkg, oracle, pctx, pb, flags, f"a third of the nodes f{flags}", start=g if fresh else None)
        after = pctx.get_inventory()
        want = g if fresh else live
        assert after[quiet].tobytes() == want[quiet].tobytes(), f"f{flags}: a node without pods changed"
        assert after[~quiet].tobytes() != want[~quiet].tobytes()


# ---- c. pod shapes and failure records ------------------------------------------------------------------------------
@pytest.mark.parametrize("form", E.OUT_FORMS)
def test_pod_shapes_and_failure_records(pkg, oracle, pctx, form):
    A = pkg.api
    for seed in range(3):
        pb = E.shapes(seed, form)
        for flags in (0, A.F_EXHAUSTIVE):
            _load(pctx, pb)
            check(pkg, oracle, pctx, pb, flags, f"{pb.name} f{flags}")
            check(pkg, oracle, pctx, pb, flags, f"{pb.name} f{flags}, again on the state it left")


def test_empty_pods(pkg, oracle, pctx):
    A = pkg.api
    for pb in (E.only_empty(), E.mostly_empty()):
        _load(pctx, pb)
        for flags in (0, A.F_EXHAUSTIVE, A.F_FRESH_INVENTORY):
            check(pkg, oracle, pctx, pb, flags, f"{pb.name} f{flags}", start=pb.gpus if flags & A.F_FRESH_INVENTORY else None)


# ---- d. the slot fault ----------------------------------------------------------------------------------------------
def faults(R, pb, where):
    """Variants of pb in which one claim of the first, a middle or the last well-formed pod has slots past n_out:
    (claims, out_off, what).  The range ends one slot past n_out; it starts past n_out; a GPU claim of count 5 naming
    the pod's node at n_out - 1 (count slots, where naming no node it would have one)."""
    sizes = np.diff(pb.pod_off.astype(np.int64))
    c = pb.claims
    good = [p for p in range(len(sizes)) if 0 < sizes[p] <= R.MAX_POD and c["node"][pb.pod_off[p]] < pb.n_node and
            (c["node"][pb.pod_off[p]: pb.pod_off[p + 1]] == c["node"][pb.pod_off[p]]).all()]
    p = {"first": good[0], "middle": good[len(good) // 2], "last": good[-1]}[where]
    i = int(pb.pod_off[p + 1]) - 1
    sl = int(E.slots(c[i: i + 1], pb.n_node, True)[0])
    one_past = pb.out_off.copy()
    one_past[i] = pb.n_out - sl + 1
    start_past = pb.out_off.copy()
    start_past[i] = pb.n_out + 3
    five = c.copy()
    five["kind"][i], five["profile"][i], five["count"][i] = R.KIND_GPU, 0, 5
    at_end = pb.out_off.copy()
    at_end[i] = pb.n_out - 1
    return [(c, one_past, f"{where} pod {p}: one slot past"), (c, start_past, f"{where} pod {p}: starts past"),
            (five, at_end, f"{where} pod {p}: count 5 at n_out - 1")]


def refused(pkg, ctx, pb, claims, out_off, flags, what):
    A = pkg.api
    before, n0 = ctx.get_inventory(), ctx.launch_count()
    rc, out = raw_pods(pkg, ctx, pb, claims, out_off, flags=flags)
    assert rc == A.E_INVAL, f"{what}: rc {rc}"
    assert (out.view(np.uint8) == SENT).all(), f"{what}: an output byte was written"
    assert ctx.get_inventory().tobytes() == before.tobytes(), f"{what}: the inventory changed"
    assert ctx.launch_count() == n0, f"{what}: the refused call launched kernels"
    msg = (ctx._lib.dra_last_error(ctx._h) or b"").decode()
    assert "outside n_out" in msg and "undefined" not in msg, msg


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_slot_fault_changes_nothing(pkg, oracle, pctx, where):
    """On a live state that differs from the pristine one, so that neither a placed pod nor the FRESH rewrite could go
    unseen; after each refused call the next valid call is right."""
    A, R = pkg.api, pkg.records
    pb = E.shapes(7, "permuted")
    _load(pctx, pb)
    check(pkg, oracle, pctx, pb, 0, "before the faults")
    assert pctx.get_inventory().tobytes() != pb.gpus.tobytes()
    for flags in (0, A.F_FRESH_INVENTORY, A.F_EXHAUSTIVE):
        for claims, oo, what in faults(R, pb, where):
            refused(pkg, pctx, pb, claims, oo, flags, f"{what} f{flags}")
            check(pkg, oracle, pctx, pb, flags, f"after {what} f{flags}",
                  start=pb.gpus if flags & A.F_FRESH_INVENTORY else None)


def test_slots_ending_at_n_out_are_accepted(pkg, oracle, pctx):
    A, R = pkg.api, pkg.records
    for pb in E.boundary():
        for flags in (0, A.F_EXHAUSTIVE):
            _load(pctx, pb)
            ref = check(pkg, oracle, pctx, pb, flags, f"{pb.name} f{flags}")
            assert ref["status"][-1] in ((R.ST_INVALID,) if "count 5" in pb.name else (R.ST_OK,)), pb.name
    pb = E.boundary()[0]                                  # the same call with n_out one short
    _load(pctx, pb)
    rc, out = raw_pods(pkg, pctx, pb, n_out=pb.n_out - 1)
    assert rc == A.E_INVAL and (out.view(np.uint8) == SENT).all()
    assert pctx.get_inventory().tobytes() == pb.gpus.tobytes()


# ---- e. the same problems on sharded worlds -------------------------------------------------------------------------
WORLDS = [(1, "even"), (2, "uneven"), (3, "even"), (3, "empty")]


def _world(pkg, pb, world, kind):
    return S.World(pkg, pb.table, pb.node_off, pb.gpus, world, S.bounds(pb.n_node, world, kind), world - 1,
                   n_out_max=1 << 16)


def _sharded_same(pkg, W, single, pb, flags, what):
    """The call on every rank and on the single context: each rank's table equals the single call's OutRecs on every slot
    a claim owns, and each rank's own GPU range the single call's inventory"""
    A = pkg.api
    rc, ref = raw_pods(pkg, single, pb, flags=flags)
    assert rc == A.OK, f"{what}: single rc {rc}"
    tables = S.pods(W, pb.claims, pb.pod_off, pb.out_off, pb.n_out, flags)
    mine = E.owned(pb)
    inv = single.get_inventory()
    for r, t in enumerate(tables):
        assert t[mine].tobytes() == ref[: pb.n_out][mine].tobytes(), f"{what}: rank {r} table differs"
        g0, g1 = W.gpu_range(r)
        assert W.ctxs[r].get_inventory()[g0:g1].tobytes() == inv[g0:g1].tobytes(), f"{what}: rank {r} inventory differs"


@pytest.mark.parametrize("world,kind", WORLDS)
def test_sharded(pkg, pctx, world, kind):
    A = pkg.api
    for k, form in enumerate(E.OUT_FORMS):
        pb = E.shapes(world + 10 * k, form)
        W = _world(pkg, pb, world, kind)
        try:
            _load(pctx, pb)
            for flags in (A.F_EXHAUSTIVE, 0, A.F_FRESH_INVENTORY, A.F_EXHAUSTIVE | A.F_FRESH_INVENTORY):
                _sharded_same(pkg, W, pctx, pb, flags, f"{pb.name} world {world} {kind} f{flags}")
        finally:
            W.close()
    for pb in E.boundary():
        W = _world(pkg, pb, world, kind)
        try:
            _load(pctx, pb)
            _sharded_same(pkg, W, pctx, pb, A.F_EXHAUSTIVE, f"{pb.name} world {world} {kind}")
        finally:
            W.close()


@pytest.mark.parametrize("world,kind", WORLDS)
def test_sharded_slot_fault(pkg, pctx, world, kind):
    """the faults of test_slot_fault_changes_nothing fail on every rank with no inventory changed, and the next call on
    the world is the single-inventory call's"""
    A, R = pkg.api, pkg.records
    pb = E.shapes(8, "gaps")
    W = _world(pkg, pb, world, kind)
    try:
        _load(pctx, pb)
        _sharded_same(pkg, W, pctx, pb, 0, "before the faults")
        for where in ("first", "middle", "last"):
            for claims, oo, what in faults(R, pb, where):
                for flags in (0, A.F_FRESH_INVENTORY, A.F_EXHAUSTIVE):
                    before = W.inventories()
                    S.pods(W, claims, pb.pod_off, oo, pb.n_out, flags, expect=A.E_INVAL)
                    for r, (b, a) in enumerate(zip(before, W.inventories())):
                        assert a.tobytes() == b.tobytes(), f"{what} f{flags}: rank {r} inventory changed"
                _sharded_same(pkg, W, pctx, pb, A.F_EXHAUSTIVE, f"after {what}")
    finally:
        W.close()
