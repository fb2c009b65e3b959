"""GPU suite: pod capacity (spec §16) through the C ABI — every output byte for byte the CPU oracle's, the inventory
untouched."""
import ctypes as C

import numpy as np
import pytest

from test_pod_capacity import _flat, problem

import capacity_oracle as K

pytestmark = pytest.mark.gpu
WIDTHS = {8: (0, 1, 2, 3, 8, 8), 16: (0, 1, 3, 8, 9, 16), 32: (0, 2, 8, 16, 17, 32)}


@pytest.fixture(scope="module")
def cctx(pkg):
    c = pkg.api.Context(device=0)
    yield c
    c.close()


def _check(ctx, g, off, t, claims, pod_off, cn=None, co=None, max_copies=64, exhaustive=False, stop=True, totals=True, what=""):
    """One call on the device against the oracle on the context's inventory; returns the device's outputs."""
    before = ctx.get_inventory()
    got = ctx.pod_capacity(claims, pod_off, cn, co, max_copies, exhaustive, stop, totals)
    ref = K.capacity(before, off, t, claims, pod_off, cn, co, max_copies, K.F_EXHAUSTIVE if exhaustive else 0)
    for name, x, y in zip(("pair_copies", "pair_stop", "pod_total", "pod_nodes"), got, ref):
        if x is None:
            assert not (stop if name == "pair_stop" else totals), name
        elif x.tobytes() != y.tobytes():
            bad = np.flatnonzero(x != y)[:5]
            pytest.fail(f"{what}: {name} differs at {bad}: device {x[bad]} oracle {y[bad]}")
    assert ctx.get_inventory().tobytes() == before.tobytes(), what
    assert "pod_capacity" in ctx.last_chain()
    return got


@pytest.mark.parametrize("width", [8, 16, 32])
def test_random_problems_at_each_lane_width(pkg, cctx, width):
    """The CPU suite's generator on inventories whose widest node has <= 8, 9..16 and 17..32 GPUs: dense and candidate
    forms, first-fit and exhaustive, with and without each optional output."""
    forms, stops = set(), set()
    for seed in range(10):
        g, off, t, c, pod_off, cands = problem(1000 * width + seed, WIDTHS[width], n_node=8, n_run=60)
        widest = int(np.diff(off.astype(np.int64)).max())
        if not width // 2 < widest <= width:
            g, off, t, c, pod_off, cands = problem(1000 * width + seed, WIDTHS[width] + (width,) * 6, n_node=8, n_run=60)
        cctx.set_table(t); cctx.set_inventory(g, off)
        cn, co = (None, None) if cands is None else _flat(cands)
        forms.add(cands is None)
        for k, (exh, stop, totals) in enumerate(((False, True, True), (True, True, True), (True, False, True),
                                                 (False, True, False), (True, False, False))):
            got = _check(cctx, g, off, t, c, pod_off, cn, co, (64, 1, 5)[(seed + k) % 3], exh, stop, totals,
                         f"w{width} seed {seed} exh {exh}")
            if got[1] is not None:
                stops |= set(got[1].tolist())
    assert forms == {True, False} and {K.ST_OK, K.ST_POD, K.ST_INVALID} <= stops


def test_selectors_search_limit_and_the_share_count(pkg, cctx):
    R = pkg.records
    t = R.default_table()
    g, off = R.make_inventory([8, 8, 1, 1], mig=True)
    g["busy"][[8, 15]] = 0xFF
    g["flags"][17] = 0                                        # node 3: one plain GPU, 65,500 shares taken
    g["share_cnt"][17] = 65500
    attrs = np.zeros(len(g), R.ATTR_DTYPE)
    attrs["index"] = np.arange(len(g)) % 8
    sels = np.stack([R.selector(("cmp", R.ATTR_INDEX, R.CMP_LT, 4)), R.selector(("cmp", R.ATTR_INDEX, R.CMP_GE, 6))])
    c = np.zeros(14, R.CLAIM_DTYPE)
    c["kind"], c["count"] = R.KIND_MIG, 1
    c["profile"][:5] = [R.GI_1_SLICE, R.GI_1_SLICE, R.GI_1_SLICE, R.GI_3_SLICE, R.GI_3_SLICE]
    c["mem_limit_mib"][:5] = [1, 2, 3, 1, 2]
    c["profile"][5:13] = [R.GI_1_SLICE] * 7 + [R.GI_7_SLICE]  # 7 x 1g + 7g: the search runs out of budget on an empty GPU
    c[13]["kind"] = R.KIND_SHARED
    pod_off = np.array([0, 1, 2, 3, 5, 13, 14], np.uint32)
    cctx.set_table(t); cctx.set_inventory(g, off)
    cctx.set_gpu_attrs(attrs); cctx.set_selectors(sels)
    K.set_selectors(attrs, sels)
    try:
        for exh in (False, True):
            copies, stop, total, nodes = _check(cctx, g, off, t, c, pod_off, max_copies=65535, exhaustive=exh, what=f"exh {exh}")
            copies, stop = copies.reshape(6, 4), stop.reshape(6, 4)
            assert copies[:4, :2].tolist() == [[28, 21], [14, 7], [0, 0], [4, 2]] and stop[2, 0] == K.ST_INVALID
            assert stop[4, 2] == (K.ST_SEARCH_LIMIT if exh else K.ST_POD) and copies[4, 2:].tolist() == [0, 0]
            assert copies[5].tolist() == [0, 0, 0, 35] and total[5] == 35 and nodes[5] == 1
        g["share_cnt"][17] = 0
        cctx.set_inventory(g, off)
        copies, stop, _, _ = _check(cctx, g, off, t, c[13:], np.array([0, 1], np.uint32), max_copies=65535, what="cap")
        assert copies[3] == 65535 and stop[3] == K.ST_OK
    finally:
        cctx.set_gpu_attrs(None); cctx.set_selectors(None)
        K.set_selectors()


def test_copies_against_pods_allocate_and_unsuitable(pkg, cctx):
    """Without the oracle, on synth.pods over cfg5's fragmented inventory: pair_copies is the number of pods
    dra_allocate_pods_batch places out of max_copies identical copies, and copies >= 1 is the exhaustive UnsuitableNodes
    bit."""
    R, A = pkg.records, pkg.api
    w, pod_off = pkg.synth.pods(n_pod=40, n_node=12, seed=3)
    n_node, max_copies = w.n_node, 6
    cctx.set_table(w.table); cctx.set_inventory(w.gpus, w.node_off)
    for exh in (False, True):
        flags = A.F_EXHAUSTIVE if exh else 0
        copies, _, total, _ = cctx.pod_capacity(w.claims, pod_off, max_copies=max_copies, exhaustive=exh)
        copies = copies.reshape(40, n_node)
        assert total.tolist() == copies.sum(axis=1).tolist()
        if exh:
            bits = cctx.unsuitable(w.claims, pod_off, flags=flags)
            assert (np.unpackbits(bits, bitorder="little")[: 40 * n_node].reshape(40, n_node).astype(bool) == (copies >= 1)).all()
        # one Allocate call per pod: max_copies copies of it for every node, each node's copies in a row
        for p in range(0, 40, 3):
            pod = w.claims[pod_off[p]: pod_off[p + 1]]
            c = np.tile(pod, n_node * max_copies)
            c["node"] = np.repeat(np.arange(n_node, dtype=np.uint32), max_copies * len(pod))
            po = (np.arange(n_node * max_copies + 1) * len(pod)).astype(np.uint32)
            out = cctx.allocate_pods(c, po, flags=flags | A.F_FRESH_INVENTORY)
            placed = (out["status"].reshape(n_node, max_copies, len(pod)) == R.ST_OK).all(axis=2)
            assert placed.sum(axis=1).tolist() == copies[p].tolist(), (exh, p)
            assert (placed[:, :-1] >= placed[:, 1:]).all()                  # the placed copies are a prefix
        cctx.reset_inventory()
    assert copies.max() >= 2 and (copies == 0).any()


def _raw(pkg, ctx, a, sentinel=0xAB):
    """dra_pod_capacity_batch on sentinel-filled outputs; returns (rc, outputs)"""
    A = pkg.api
    n_pod = len(a["po"]) - 1
    n_pair = max(n_pod * ctx.n_node if a["co"] is None else len(a["cn"]), 1)
    outs = [np.full(n * np.dtype(d).itemsize, sentinel, np.uint8).view(d)
            for n, d in ((n_pair, np.uint16), (n_pair, np.uint8), (max(n_pod, 1), np.uint64), (max(n_pod, 1), np.uint32))]
    keep = [None if a[k] is None else np.ascontiguousarray(a[k], dtype=d)
            for k, d in (("c", A.R.CLAIM_DTYPE), ("po", np.uint32), ("cn", np.uint32), ("co", np.uint32))]
    p = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)      # noqa: E731
    c, po, cn, co = keep
    rc = ctx._lib.dra_pod_capacity_batch(ctx._h, p(c), len(c), p(po), n_pod, p(cn), p(co), a["mc"],
                                         p(outs[0]) if a.get("copies", True) else None, *[p(o) for o in outs[1:]], a["fl"])
    return rc, outs


def test_call_errors_purity_and_reset(pkg, cctx, oracle):
    A, R = pkg.api, pkg.records
    w, pod_off = pkg.synth.pods(n_pod=30, n_node=8, seed=5)
    cctx.set_table(w.table); cctx.set_inventory(w.gpus, w.node_off)
    out = cctx.allocate_pods(w.claims, pod_off)                # the live inventory now differs from the pristine one
    live = cctx.get_inventory()
    assert live.tobytes() != w.gpus.tobytes()
    ok = dict(c=w.claims[:3], po=[0, 1, 3], cn=[0, 9, 1, 1], co=[0, 2, 4], mc=4, fl=0)
    rc, outs = _raw(pkg, cctx, ok)
    ref = K.capacity(live, w.node_off, w.table, w.claims[:3], [0, 1, 3], [0, 9, 1, 1], [0, 2, 4], 4)
    assert rc == A.OK and all(o.tobytes() == r.tobytes() for o, r in zip(outs, ref))
    for name, kw in [("flags", dict(fl=1)), ("flags", dict(fl=A.F_FRESH_INVENTORY)), ("max_copies 0", dict(mc=0)),
                     ("max_copies 65536", dict(mc=65536)), ("pod_off span", dict(po=[0, 1, 2])),
                     ("pod_off start", dict(po=[1, 1, 3])), ("pod_off order", dict(po=[0, 3, 2, 3], co=[0, 1, 2, 4])),
                     ("cand_off start", dict(co=[1, 2, 4])), ("cand_off order", dict(co=[0, 3, 2])),
                     ("cand_nodes without cand_off", dict(co=None)), ("no pair_copies", dict(copies=False))]:
        rc, outs = _raw(pkg, cctx, dict(ok, **kw))
        assert rc == A.E_INVAL, name
        assert all((o.view(np.uint8) == 0xAB).all() for o in outs), name
        assert cctx.get_inventory().tobytes() == live.tobytes(), name
    rc, outs = _raw(pkg, cctx, dict(ok, c=w.claims[:0], po=[0], cn=None, co=None))   # no pods: OK, nothing written
    assert rc == A.OK and all((o.view(np.uint8) == 0xAB).all() for o in outs)
    rc, _ = _raw(pkg, cctx, dict(ok, c=w.claims[:0], po=[0], cn=None, co=None, mc=0))
    assert rc == A.E_INVAL
    # the next call is correct, the live inventory is as it was, and the pristine copy is still the loaded one
    _check(cctx, live, w.node_off, w.table, w.claims, pod_off, exhaustive=True, what="after the errors")
    cctx.reset_inventory()
    assert cctx.get_inventory().tobytes() == w.gpus.tobytes()
    assert cctx.allocate_pods(w.claims, pod_off).tobytes() == out.tobytes()


def test_dense_over_two_to_the_32_pairs(pkg, cctx):
    R = pkg.records
    n = 1 << 16
    g, off = R.make_inventory([1] * n, mig=True)
    cctx.set_table(R.default_table()); cctx.set_inventory(g, off)
    with pytest.raises(pkg.api.DraError):
        cctx._check(cctx._lib.dra_pod_capacity_batch(cctx._h, None, 0, np.zeros(n + 1, np.uint32).ctypes.data_as(C.c_void_p), n,
                                                     None, None, 1, np.zeros(8, np.uint16).ctypes.data_as(C.c_void_p),
                                                     None, None, None, 0))


def test_resident_context_around_a_capacity_call(pkg, oracle):
    """A DRA_CFG_RESIDENT context answers Allocate batches through the resident kernel before and after a capacity call,
    which stops that kernel and sees the state it left."""
    R, A = pkg.records, pkg.api
    w = pkg.synth.cfg2(2000, 60)
    r1, inv1 = oracle.allocate(w.gpus, w.node_off, w.table, w.claims)
    r2, inv2 = oracle.allocate(inv1, w.node_off, w.table, w.claims)
    c1 = np.zeros(4, R.CLAIM_DTYPE)
    c1["kind"], c1["count"], c1["profile"] = R.KIND_MIG, 1, [R.GI_1_SLICE, R.GI_2_SLICE, R.GI_3_SLICE, R.GI_7_SLICE]
    with A.Context(device=0, flags=A.CFG_RESIDENT) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        pc = A.PinnedBuffer(w.n_claim, R.CLAIM_DTYPE); pc.array[:] = w.claims
        po = A.PinnedBuffer(w.n_out, R.OUT_DTYPE)
        assert c.allocate(pc.array, None, w.n_out, out=po.array).tobytes() == r1.tobytes() and c.serve_batches() == 1
        got = c.pod_capacity(c1, np.arange(5, dtype=np.uint32), exhaustive=True)
        ref = K.capacity(inv1, w.node_off, w.table, c1, np.arange(5, dtype=np.uint32), flags=K.F_EXHAUSTIVE)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(got, ref)) and ref[2][0] > 0
        assert c.allocate(pc.array, None, w.n_out, out=po.array).tobytes() == r2.tobytes() and c.serve_batches() == 2
        assert c.get_inventory().tobytes() == inv2.tobytes()
        pc.free(); po.free()


def test_sharded_world_sync_then_capacity_on_any_rank(pkg, oracle):
    """Two ranks on one device: after sharded pods Allocate calls each rank's copy is right for its own range only;
    dra_shard_sync_inventory_device makes every copy the world's state, and the capacity call on either rank then answers
    as the oracle does on that state."""
    import shard_world as S
    w = pkg.synth.mixed(2400, 31, 72, invalid=True)
    bounds = [0, 11, w.n_node]
    rng = np.random.default_rng(2)
    W = S.World(pkg, w.table, w.node_off, w.gpus, 2, bounds, n_out_max=1 << 16)
    try:
        state = w.gpus
        for flags, oflags in ((0, 0), (pkg.api.F_EXHAUSTIVE, oracle.F_EXHAUSTIVE)):
            pc, po, poo, pn = S.malformed_mixed(pkg, w, bounds, rng, True)
            _, state = oracle.allocate_pods(state, w.node_off, w.table, pc, po, poo, pn, oflags)
            S.pods(W, pc, po, poo, pn, flags)
        assert any(inv.tobytes() != state.tobytes() for inv in W.inventories())
        W.sync_inventory()
        pods_w, pod_off = pkg.synth.pods(n_pod=50, n_node=w.n_node, seed=1)
        cn, co = _flat([list(rng.integers(0, w.n_node + 2, 5)) for _ in range(50)])
        for r, ctx in enumerate(W.ctxs):
            for exh in (False, True):
                ref = K.capacity(state, w.node_off, w.table, pods_w.claims, pod_off, flags=K.F_EXHAUSTIVE if exh else 0)
                got = _check(ctx, state, w.node_off, w.table, pods_w.claims, pod_off, exhaustive=exh, what=f"rank {r} dense")
                assert all(x.tobytes() == y.tobytes() for x, y in zip(got, ref)) and ref[2].max() > 0
                _check(ctx, state, w.node_off, w.table, pods_w.claims, pod_off, cn, co, 9, exh, what=f"rank {r} candidates")
    finally:
        W.close()


def test_cpp_driver_pod_capacity_batch(pkg):
    """Driver::PodCapacityBatch of the C++ host layer (tests/cpp/capacity_test.cpp)."""
    import subprocess
    exe = pkg.build.build_cpp_capacity_test()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "capacity_test ok" in r.stdout
