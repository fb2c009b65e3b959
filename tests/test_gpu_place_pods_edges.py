"""GPU suite: place pods (spec §13, dra_place_pods_batch) at its edges, and the node limit of the sorting pod calls.

Every call goes through the raw ABI on sentinel-filled outputs with slack, and is compared byte for byte with
place_oracle.place_pods on the context's live inventory: the OutRecs, pod_node and the inventory afterwards.  Nothing
may be written past n_out or n_pod, and the caller's claim array is never written.

* the pair sort: the (pod, candidate) records are bucketed by node with Allocate's counting sort, and a node's visit list
  must stay in (pod, position) order.  ROWS puts the pair and node counts on each side of each of the sort's thresholds
  (shapes from the SM count S) and asserts the chain and histogram tile that ran, under four candidate distributions
* long candidate lists, whose scans for the next usable entry run 32 entries at a time (test_place_pods_edges.py)
* exhausted searches across candidates: the sticky search-limit bit (test_place_pods_edges.py)
* pod shapes and both places that write failure records, every out_off form, arbitrary claim node fields
* the walk: a serial hand-off chain across more nodes than the walk has warps, nodes of 1 to 32 GPUs, and
  DRA_F_FRESH_INVENTORY on a live state that differs from the pristine one on every node
* the same problems on sharded worlds of one to three contexts on one device
* the node limit of the counting sort (102,399 nodes): the four single-inventory pod calls that sort refuse a wider
  inventory before anything is enqueued, and the next call on the context is right"""
from types import SimpleNamespace

import numpy as np
import pytest

import place_oracle as P
import preempt_oracle as PR
import preempt_place_oracle as PP
import test_place_pods_edges as E
from test_gpu_pod_call_checks import PLACE, PODS, PRE, PREPL, SENTINEL, _base, _raw
import shard_world as S
from test_gpu_shard_place import _check as _check_sharded
from test_preempt import mig_running, occupied

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


def _filled(n, dtype):
    return np.full((max(n, 1) + SLACK) * np.dtype(dtype).itemsize, SENT, np.uint8).view(dtype)


def raw_place(pkg, ctx, pb, cn, co, flags):
    """dra_place_pods_batch on sentinel-filled outputs SLACK elements longer than the call may write: (rc, out, pod_node)"""
    import ctypes as C
    R = pkg.records
    n_pod = len(pb.pod_off) - 1
    out, node = _filled(pb.n_out, R.OUT_DTYPE), _filled(n_pod, np.uint32)
    c = np.ascontiguousarray(pb.claims, dtype=R.CLAIM_DTYPE)
    keep = c.copy()
    arrs = [np.ascontiguousarray(x, dtype=np.uint32) if x is not None else None for x in (pb.pod_off, cn, co, pb.out_off)]
    po, cn_, co_, oo = arrs
    p = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)      # noqa: E731
    rc = ctx._lib.dra_place_pods_batch(ctx._h, p(c), len(c), p(po), n_pod, p(cn_), p(co_), p(oo), p(out), pb.n_out,
                                       p(node), flags)
    assert c.tobytes() == keep.tobytes(), "the call wrote the caller's claims"
    return rc, out, node


def _same(what, name, got, ref):
    x = got[: ref.size]
    if x.tobytes() != ref.tobytes():
        bad = np.flatnonzero(x.view(np.uint8) != ref.view(np.uint8))[:5]
        pytest.fail(f"{what}: {name} differs at bytes {bad}")
    assert (got[ref.size:].view(np.uint8) == SENT).all(), f"{what}: written past {name}"


def check(pkg, ctx, pb, flags, what, dense=False, cands=None, start=None):
    """One call on pb against the oracle on the context's live inventory (start: another starting state, e.g. the
    pristine one for DRA_F_FRESH_INVENTORY).  cands: (cand_nodes, cand_off) arrays instead of pb's lists."""
    A = pkg.api
    cn, co = (None, None) if dense else cands if cands is not None else E.cand_arrays(pb)
    before = ctx.get_inventory() if start is None else start
    ref, ref_node, ref_inv = P.place_pods(before, pb.node_off, pb.table, pb.claims, pb.pod_off, cn, co, pb.out_off,
                                          pb.n_out, P.F_EXHAUSTIVE if flags & A.F_EXHAUSTIVE else 0)
    rc, out, node = raw_place(pkg, ctx, pb, cn, co, flags)
    assert rc == A.OK, f"{what}: rc {rc}"
    _same(what, "out", out, ref)
    _same(what, "pod_node", node, ref_node)
    after = ctx.get_inventory()
    if after.tobytes() != ref_inv.tobytes():
        bad = np.flatnonzero(after != ref_inv)[:5]
        pytest.fail(f"{what}: inventory differs at GPUs {bad}: device {after[bad]} oracle {ref_inv[bad]}")
    assert "place" in ctx.last_chain(), what
    return ref, ref_node


# ---- a. the pair sort at its thresholds -----------------------------------------------------------------------------
SORT8 = {"hist8", "scan8", "scatter", "place"}
WARP = {"hist_warp", "scan", "scatter", "place"}
D4 = ("random", "hot", "nonode", "empty_ends")
# id, shape(S) -> (n_pair, n_node), chain, hist tile (0: no histogram kernel), both flags
ROWS = [
    # the one-CTA counting sort: 8,192 records, and its shared memory at 8,192 records (2,769 nodes)
    ("bucket_small_pairs_max", lambda S: (8_192, S), {"bucket_small", "place"}, 0, True),
    ("hist8_pairs_min", lambda S: (8_193, S), SORT8, 2048, True),
    ("bucket_small_smem_max", lambda S: (8_192, 2_769), {"bucket_small", "place"}, 0, True),
    ("bucket_small_smem_over", lambda S: (8_192, 2_770), SORT8, 2048, True),
    # CTA-wide histogram: 2048-record tiles up to S tiles, then grown tiles
    ("hist8_tile_fixed_max", lambda S: (S * 2048, 1_000), SORT8, 2048, False),
    ("hist8_tile_grown_min", lambda S: (S * 2048 + 1, 1_000), {"hist8_multi", "scan8", "scatter", "place"}, 4096, False),
    # the scan of the tile histograms: one warp per node up to 524,288 counters, coalesced rows beyond
    ("scan8_max", lambda S: (S * 2048, 524_288 // S - 1), SORT8, 2048, False),
    ("scan_rows_min", lambda S: (S * 2048, 524_288 // S), {"hist8", "scan_rows", "scatter", "place"}, 2048, False),
    # CTA-wide histogram while 8 x (n_node + 2) u16 counters fit 200 KiB, one-warp tiles beyond
    ("hist8_nodes_max", lambda S: (50_000, 12_798), SORT8, 2048, True),
    ("hist_warp_nodes_min", lambda S: (50_000, 12_799), WARP, 800, True),
    # the widest node range the sort takes
    ("sortable_max", lambda S: (50_000, SORTABLE), WARP, 800, False),
]
CASES = [pytest.param(r, d, id=f"{r[0]}-{d}") for r in ROWS for d in D4]


def sort_workload(R, n_pair, n_node, dist, seed=3):
    """Nodes of one and two MIG GPUs, pods of one 1g-7g claim with 8 candidates each (the last pod fewer), so several
    pods compete for each node and a node list out of (pod, position) order changes the answer:
      random      about a quarter of the pairs are strays (n_node, n_node + 1000, 0xFFFFFFFF)
      hot         >= 90 % of the pairs, and every one of the first 65,536, name node 1
      nonode      every pair is a stray but the last of each pod
      empty_ends  nodes 0 and n_node - 1 have no GPU, and every fourth pair names one of them"""
    rng = np.random.default_rng(seed)
    widths = 1 + np.arange(n_node) % 2
    if dist == "empty_ends":
        widths[0] = widths[-1] = 0
    g, off = R.make_inventory(list(widths), mig=True)
    n_pod = (n_pair + 7) // 8
    co = np.minimum(np.arange(n_pod + 1) * 8, n_pair).astype(np.uint32)
    cn = rng.integers(0, n_node, n_pair).astype(np.uint32)
    st = np.array(E.strays(n_node), np.uint32)
    if dist == "random":
        m = rng.random(n_pair) < 0.25
        cn[m] = st[rng.integers(0, 3, int(m.sum()))]
    elif dist == "hot":
        m = rng.random(n_pair) < 0.92
        m[:65_536] = True
        cn[m] = 1
    elif dist == "nonode":
        last = co[1:] - 1
        keep = cn[last].copy()
        cn[:] = st[np.arange(n_pair) % 3]
        cn[last] = keep
    else:
        cn[::4] = np.where(rng.random(len(cn[::4])) < 0.5, 0, n_node - 1)
    c = E._mig(rng.choice([R.GI_1_SLICE, R.GI_2_SLICE, R.GI_3_SLICE, R.GI_4_SLICE, R.GI_7_SLICE], n_pod))
    pb = E.problem(f"{n_pair} pairs x {n_node} nodes {dist}", g, off, R.default_table(), c, np.arange(n_pod + 1), None)
    return pb, cn, co


@pytest.mark.parametrize("row,dist", CASES)
def test_pair_sort_at_boundary(pkg, pctx, row, dist):
    name, shape, chain, tile, both = row
    S = _n_sm()
    n_pair, n_node = shape(S)
    pb, cn, co = sort_workload(pkg.records, n_pair, n_node, dist)
    for flags in ((0, pkg.api.F_EXHAUSTIVE) if both else (0,)):
        _load(pctx, pb)
        ref, node = check(pkg, pctx, pb, flags, f"{name} {dist} f{flags}: {pb.name}, {S} SMs", cands=(cn, co))
        got = pctx.last_chain()
        assert got == chain, f"{name}: {n_pair} pairs x {n_node} nodes on {S} SMs took {sorted(got)}"
        assert pctx.last_hist_tile() == tile, f"{name}: hist tile {pctx.last_hist_tile()}"
        assert (node != NONE).any(), name
    pctx.reset_inventory()
    assert pctx.get_inventory().tobytes() == pb.gpus.tobytes()


# ---- b-d. long lists, exhausted searches, pod shapes ----------------------------------------------------------------
@pytest.mark.parametrize("exhaustive", [False, True])
def test_long_lists(pkg, pctx, exhaustive):
    A = pkg.api
    fl = A.F_EXHAUSTIVE if exhaustive else 0
    pb = E.long_lists(seed=1)
    _load(pctx, pb)
    ref, node = check(pkg, pctx, pb, fl, "long lists")
    assert len(set(node[-10:].tolist())) == 10 and NONE not in node[-10:]
    pctx.reset_inventory()
    check(pkg, pctx, pb, fl, "long lists, dense", dense=True)


def test_exhausted_searches(pkg, pctx):
    A, R = pkg.api, pkg.records
    pb = E.exhausted()
    for flags in (0, A.F_EXHAUSTIVE):
        _load(pctx, pb)
        out, node = check(pkg, pctx, pb, flags, f"exhausted f{flags}")
        for p, (name, (st_ex, node_ex), st_plain) in enumerate(pb.expect):
            st = E.pod_statuses(pb, out, p)
            if flags:
                assert node[p] == node_ex and (st_ex is None or st == {st_ex}), f"{name}: {st}"
            else:
                assert R.ST_SEARCH_LIMIT not in st and (st_plain is None or st == {st_plain}), f"{name}: {st}"


@pytest.mark.parametrize("form", E.OUT_FORMS)
def test_pod_shapes_and_failure_records(pkg, pctx, form):
    """every claim node field gives the bytes of node = 0, and the claim array is never written"""
    A = pkg.api
    for seed in range(3):
        for flags in (0, A.F_EXHAUSTIVE):
            ref = None
            for node_field in E.NODE_FIELDS:
                pb = E.shapes(seed, form, node_field)
                _load(pctx, pb)
                got = check(pkg, pctx, pb, flags, f"{pb.name} f{flags}")
                if ref is not None:
                    assert all(a.tobytes() == b.tobytes() for a, b in zip(got, ref)), pb.name
                ref = got
            pctx.reset_inventory()
            check(pkg, pctx, pb, flags, f"{pb.name} dense f{flags}", dense=True)


# ---- e. the walk ----------------------------------------------------------------------------------------------------
def _n_wide():
    """every warp of the walk owns at least two nodes at any occupancy: at most 16 CTAs of 4 warps per SM"""
    return 128 * _n_sm() + 37


@pytest.mark.parametrize("mirror", [False, True])
def test_serial_hand_off_chain(pkg, pctx, mirror):
    """One-GPU nodes, node at(0) full; pod i (a 7g) lists at(i), at(i+1).  Pod i finds at(i) taken by pod i - 1 and
    takes at(i + 1), so each node evaluates its two pods in order, one hand-off per pod across the whole inventory."""
    R = pkg.records
    n = _n_wide()
    at = (lambda k: n - 1 - k) if mirror else (lambda k: k)
    g, off = R.make_inventory([1] * n, mig=True)
    g["busy"][at(0)] = 0xFF
    cands = [[at(i), at(i + 1)] for i in range(n - 1)]
    pb = E.problem("chain", g, off, R.default_table(), E._mig([R.GI_7_SLICE] * (n - 1)), np.arange(n), cands)
    for flags in (0, pkg.api.F_EXHAUSTIVE):
        _load(pctx, pb)
        out, node = check(pkg, pctx, pb, flags, f"chain mirror {mirror} f{flags}")
        assert (node == np.array([at(i + 1) for i in range(n - 1)], np.uint32)).all()
        assert (out["status"] == R.ST_OK).all()


def _widths_problem(R, seed):
    """nodes of 1, 9, 17, 31 and 32 GPUs, MIG and not, some slices busy; pods of 1g-7g and GPU claims of count 1-3"""
    rng = np.random.default_rng(seed)
    widths = [1, 9, 17, 31, 32] * 6
    parts = [R.make_inventory([w], mig=k % 3 != 2)[0] for k, w in enumerate(widths)]
    g = np.concatenate(parts)
    off = np.zeros(len(widths) + 1, np.uint32)
    off[1:] = np.cumsum(widths)
    g["node"] = np.repeat(np.arange(len(widths)), widths)
    g["busy"][rng.random(len(g)) < 0.5] = 0x0F
    pods = []
    for _ in range(600):
        c = E._mig(rng.choice([R.GI_1_SLICE, R.GI_2_SLICE, R.GI_3_SLICE, R.GI_4_SLICE, R.GI_7_SLICE], int(rng.integers(1, 6))))
        if rng.random() < 0.3:
            c[0]["kind"], c[0]["profile"], c[0]["count"] = R.KIND_GPU, 0, int(rng.integers(1, 4))
        pods.append(c)
    claims = np.concatenate(pods)
    pod_off = np.concatenate([[0], np.cumsum([len(c) for c in pods])])
    cands = [[int(x) for x in rng.integers(0, len(widths) + 2, 8)] for _ in pods]
    out_off, n_out = E.out_form(claims, "packed", rng)
    return E.problem(f"widths {seed}", g, off, R.default_table(), claims, pod_off, cands, out_off, n_out)


def test_node_widths(pkg, pctx):
    for seed in range(2):
        pb = _widths_problem(pkg.records, seed)
        for flags in (0, pkg.api.F_EXHAUSTIVE):
            _load(pctx, pb)
            out, node = check(pkg, pctx, pb, flags, f"{pb.name} f{flags}")
            assert (node != NONE).sum() > 50
            pctx.reset_inventory()
            check(pkg, pctx, pb, flags, f"{pb.name} dense f{flags}", dense=True)


def test_fresh_inventory_on_a_changed_live_state(pkg, pctx):
    """A first call puts a 1g on every node, so the live state differs from the pristine one everywhere; calls with
    DRA_F_FRESH_INVENTORY then start from the pristine state, in both forms, and their result becomes the live one."""
    A, R = pkg.api, pkg.records
    n = _n_wide()
    rng = np.random.default_rng(9)
    g, off = R.make_inventory([2] * n, mig=True)
    t = R.default_table()
    first = E.problem("1g everywhere", g, off, t, E._mig([R.GI_1_SLICE] * n), np.arange(n + 1), [[i] for i in range(n)])
    _load(pctx, first)
    check(pkg, pctx, first, 0, first.name)
    live = pctx.get_inventory()
    assert (live["busy"][off[:-1]] != g["busy"][off[:-1]]).all()
    n_pod = 3000
    c = E._mig(rng.choice([R.GI_3_SLICE, R.GI_4_SLICE, R.GI_7_SLICE], n_pod))
    cands = [[int(x) for x in rng.integers(0, n + 2, 8)] for _ in range(n_pod)]
    pb = E.problem("fresh", g, off, t, c, np.arange(n_pod + 1), cands)
    for flags in (A.F_FRESH_INVENTORY, A.F_FRESH_INVENTORY | A.F_EXHAUSTIVE):
        check(pkg, pctx, first, 0, "1g everywhere again", start=pctx.get_inventory())
        check(pkg, pctx, pb, flags, f"fresh f{flags}", start=g)
        few = E.problem("fresh dense", g, off, t, c[:40], np.arange(41), None)
        check(pkg, pctx, first, 0, "1g everywhere, then dense")
        check(pkg, pctx, few, flags, f"fresh dense f{flags}", dense=True, start=g)


def test_no_candidates_after_a_sorted_allocate(pkg, oracle):
    """The candidate form with no candidate at all sorts no pair, so the walk must find every visit list empty, not the
    node offsets the previous call's counting sort left (here an Allocate on the sorting chain): every pod is placed
    nowhere and the inventory keeps what the Allocate took."""
    A, R = pkg.api, pkg.records
    w = pkg.synth.mixed(600, 8, 5)
    with A.Context(device=0, flags=A.CFG_NO_FUSED) as ctx:
        ctx.set_table(w.table)
        ctx.set_inventory(w.gpus, w.node_off)
        out = ctx.allocate(w.claims, w.out_off, w.n_out)
        assert not {"fused_staged", "fused_stream", "fused_direct"} & ctx.last_chain()
        ref, live = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
        assert out.tobytes() == ref.tobytes() and ctx.get_inventory().tobytes() == live.tobytes()
        c, po = w.claims[:6].copy(), np.array([0, 2, 4, 6], np.uint32)
        placed = c.copy()
        placed["node"] = 0
        oo, n_out = R.out_offsets(placed, 1)
        cn, co = np.zeros(0, np.uint32), np.zeros(4, np.uint32)
        for flags in (0, A.F_EXHAUSTIVE):
            got, node = ctx.place_pods(c, po, cn, co, oo, n_out, flags)
            want, want_node, after = P.place_pods(live, w.node_off, w.table, c, po, cn, co, oo, n_out, flags)
            assert got.tobytes() == want.tobytes() and node.tobytes() == want_node.tobytes(), flags
            assert (node == NONE).all() and ctx.get_inventory().tobytes() == live.tobytes(), flags


# ---- f. the same problems on a sharded world ------------------------------------------------------------------------
def _sharded(pkg, pb, world, kind, flags, what):
    w = SimpleNamespace(gpus=pb.gpus, node_off=pb.node_off, table=pb.table, n_node=pb.n_node)
    W = S.World(pkg, pb.table, pb.node_off, pb.gpus, world, S.bounds(pb.n_node, world, kind), world - 1, n_out_max=1 << 16,
                place=max(len(pb.pod_off) - 1, 1))
    try:
        for cn, co in (E.cand_arrays(pb), (None, None)):
            _check_sharded(W, w, pb.claims, pb.pod_off, cn, co, pb.out_off, pb.n_out, flags,
                           f"{what} world {world} {kind} {'dense' if cn is None else 'cands'}")
    finally:
        W.close()


@pytest.mark.parametrize("world,kind", [(1, "even"), (2, "uneven"), (3, "even"), (3, "empty")])
def test_sharded(pkg, world, kind):
    A = pkg.api
    _sharded(pkg, E.long_lists(seed=2), world, kind, A.F_EXHAUSTIVE, "long lists")
    _sharded(pkg, E.exhausted(), world, kind, A.F_EXHAUSTIVE | A.F_FRESH_INVENTORY, "exhausted")
    _sharded(pkg, E.exhausted(), world, kind, 0, "exhausted first-fit")
    for form, node_field in zip(E.OUT_FORMS, E.NODE_FIELDS):
        _sharded(pkg, E.shapes(world, form, node_field), world, kind, A.F_EXHAUSTIVE, f"shapes {form} {node_field}")


# ---- the node limit of the sorting pod calls ------------------------------------------------------------------------
def _big(R, n, running=True, bad=False):
    """n one-GPU MIG nodes; two pending pods of one 1g claim; running 1g pods on nodes 0 and n - 1 (bad: the second's
    OutRec names a GPU past the inventory, a fault found on the device)"""
    g, off = R.make_inventory([1] * n, mig=True)
    c = E._mig([R.GI_1_SLICE] * 2)
    rc, rpo, rpr, ro = mig_running([(0, 0, 1, R.GI_1_SLICE, 0), (n - 1, 0, 1, R.GI_1_SLICE, 0)], off)
    g = occupied(g, rc, ro)
    if bad:
        ro = ro.copy()
        ro["gpu"][1] = n + 5
    if not running:
        rc, rpo, rpr, ro = rc[:0], np.zeros(1, np.uint32), rpr[:0], ro[:0]
    return SimpleNamespace(g=g, off=off, t=R.default_table(), c=c, po=np.array([0, 1, 2], np.uint32),
                           prio=np.array([1, 1], np.int32), rc=rc, rpo=rpo, rpr=rpr, ro=ro)


def _cands(n):
    return dict(cn=[0, n - 1, 5], co=[0, 2, 3])


def _answer(pkg, oracle, ctx, w, fn, a):
    """the call of a on w through the raw ABI, bit-exact with its oracle on the live inventory"""
    A = pkg.api
    live = ctx.get_inventory()
    cn, co = (None, None) if a.get("cn") is None else (np.array(a["cn"], np.uint32), np.array(a["co"], np.uint32))
    if fn == PLACE:
        out, node, inv = P.place_pods(live, w.off, w.t, a["c"], w.po, cn, co, None, len(a["c"]))
        ref = [out, node]
    elif fn == PODS:
        out, inv = oracle.allocate_pods(live, w.off, w.t, a["c"], w.po)
        ref = [out]
    elif fn == PRE:
        ref = [x.ravel() for x in PR.preempt(live, w.off, w.t, a["c"], w.po, w.prio, w.rc, w.rpo, w.rpr, w.ro, None, cn,
                                             co, max_victims=a["mv"])]
        inv = live
    else:
        *ref, inv = PP.preempt_place(live, w.off, w.t, a["c"], w.po, w.prio, w.rc, w.rpo, w.rpr, w.ro, None, cn, co,
                                     None, len(a["c"]))
    rc, outs = _raw(pkg, ctx, w, fn, a)
    assert rc == A.OK, (fn, rc)
    for o, y in zip(outs, ref):
        y = np.ascontiguousarray(y)
        assert o.view(np.uint8)[: y.nbytes].tobytes() == y.view(np.uint8).tobytes(), fn
        assert (o.view(np.uint8)[y.nbytes:] == SENTINEL).all(), f"{fn}: written past an output"
    assert ctx.get_inventory().tobytes() == inv.tobytes(), fn


def _refused(pkg, ctx, w, fn, a):
    A = pkg.api
    before, n0 = ctx.get_inventory(), ctx.launch_count()
    rc, outs = _raw(pkg, ctx, w, fn, a)
    assert rc == A.E_INVAL, (fn, rc)
    assert ctx.launch_count() == n0, f"{fn}: the refused call launched kernels"
    assert all((o.view(np.uint8) == SENTINEL).all() for o in outs), f"{fn}: an output was written"
    assert ctx.get_inventory().tobytes() == before.tobytes(), f"{fn}: the inventory changed"


def _calls(w, n):
    """fn -> the call that sorts a non-empty record list"""
    pc = w.c.copy()
    pc["node"] = [0, n - 1]
    return {PLACE: dict(_base(w), **_cands(n)), PODS: dict(_base(w), c=pc),
            PRE: dict(_base(w), **_cands(n)), PREPL: dict(_base(w), **_cands(n))}


@pytest.mark.parametrize("fn", [PLACE, PODS, PRE, PREPL])
def test_widest_sortable_inventory_answers(pkg, oracle, fn):
    R = pkg.records
    w = _big(R, SORTABLE)
    with pkg.api.Context(device=0) as c:
        c.set_table(w.t); c.set_inventory(w.g, w.off)
        _answer(pkg, oracle, c, w, fn, _calls(w, SORTABLE)[fn])
        if fn == PREPL:                                   # running pods and the dense form
            c.reset_inventory()
            _answer(pkg, oracle, c, w, fn, _base(w))


@pytest.mark.parametrize("fn", [PLACE, PODS, PRE, PREPL])
def test_one_node_past_the_sort_is_refused_up_front(pkg, oracle, fn):
    """E_INVAL with no kernel launched, no output byte and no inventory word written; the next calls on the context,
    the ones that sort nothing, are right; reset_inventory() gives back the inventory as loaded."""
    R = pkg.records
    n = SORTABLE + 1
    w = _big(R, n)
    bad = _big(R, n, bad=True)
    idle = _big(R, n, running=False)
    with pkg.api.Context(device=0) as c:
        c.set_table(w.t); c.set_inventory(w.g, w.off)
        refused = [(w, _calls(w, n)[fn])]
        if fn in (PRE, PREPL):
            refused.append((bad, _calls(bad, n)[fn]))     # running pods a device check would also have failed
        if fn == PREPL:
            refused += [(w, _base(w)), (idle, _calls(idle, n)[fn])]
        for v, a in refused:
            _refused(pkg, c, v, fn, a)
            _answer(pkg, oracle, c, idle, PLACE, _base(idle))                     # the dense form sorts nothing
            _answer(pkg, oracle, c, idle, PRE, dict(_base(idle), **_cands(n)))    # no running pods: nothing to sort
            _answer(pkg, oracle, c, idle, PREPL, _base(idle))
            c.reset_inventory()
            assert c.get_inventory().tobytes() == w.g.tobytes()
