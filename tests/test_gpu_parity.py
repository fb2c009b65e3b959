"""GPU suite: the CUDA path through the C ABI must be BIT-EXACT with the CPU oracle (integer work)."""
import numpy as np
import pytest

from conftest import GOLDEN_CASES, load_golden

pytestmark = pytest.mark.gpu


def _run(ctx, w, flags=0, sort=False):
    ctx.set_table(w.table)
    ctx.set_inventory(w.gpus, w.node_off)
    out = ctx.allocate(w.claims, w.out_off, w.n_out, flags=flags)
    return out, ctx.get_inventory()


def _assert_same(out, inv, ref_out, ref_inv, what=""):
    if out.tobytes() != ref_out.tobytes():
        bad = np.nonzero(out.view(np.uint64) != ref_out.view(np.uint64))[0]
        raise AssertionError(f"{what}: {len(bad)} OutRecs differ, first at {bad[0]}: cuda={out[bad[0]]} oracle={ref_out[bad[0]]}")
    if inv.tobytes() != ref_inv.tobytes():
        bad = np.nonzero(inv.view("V16") != ref_inv.view("V16"))[0]
        raise AssertionError(f"{what}: inventory differs at gpu {bad[0]}: cuda={inv[bad[0]]} oracle={ref_inv[bad[0]]}")


# ---- frozen golden fixtures: no oracle needed on the box -------------------------------------------
@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_cuda_matches_golden(pkg, ctx, name):
    g = load_golden(name)
    ctx.set_table(g["table"])
    ctx.set_inventory(g["gpus"], g["node_off"])
    out = ctx.allocate(g["claims"], g["out_off"], len(g["out"]))
    _assert_same(out, ctx.get_inventory(), g["out"], g["gpus_after"], name)


# ---- every BASELINE config at full size, against the oracle ----------------------------------------
@pytest.mark.parametrize("cfg", ["cfg1", "cfg2", "cfg3", "cfg4", "cfg5"])
def test_cuda_matches_oracle_on_baseline_configs(pkg, ctx, oracle, cfg):
    w = pkg.synth.CONFIGS[cfg]()
    out, inv = _run(ctx, w)
    ref_out, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
    _assert_same(out, inv, ref_out, ref_inv, cfg)


@pytest.mark.parametrize("cfg", ["cfg2", "cfg5"])
def test_node_sorted_fast_path(pkg, ctx, oracle, cfg):
    w = pkg.synth.CONFIGS[cfg]().node_sorted()
    out, inv = _run(ctx, w, flags=pkg.api.F_NODE_SORTED)
    ref_out, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
    _assert_same(out, inv, ref_out, ref_inv, cfg + " sorted")


def test_node_sorted_flag_is_verified(pkg, ctx):
    w = pkg.synth.cfg2(2000, 20)           # generation order: not sorted
    ctx.set_table(w.table)
    ctx.set_inventory(w.gpus, w.node_off)
    with pytest.raises(pkg.api.DraError) as e:
        ctx.allocate(w.claims, flags=pkg.api.F_NODE_SORTED)
    assert e.value.code == pkg.api.E_INVAL
    assert ctx.get_inventory().tobytes() == w.gpus.tobytes()      # nothing changed
    # and the context is still usable
    out = ctx.allocate(w.claims)
    assert (out["status"] == 0).any()


# ---- fuzz: ragged heterogeneous nodes, all kinds, counts, groups, malformed claims ------------------
@pytest.mark.parametrize("seed", range(12))
def test_cuda_matches_oracle_fuzz(pkg, ctx, oracle, seed):
    n_claim = [50, 333, 1000, 4000, 9000, 20000][seed % 6]
    n_node = [1, 3, 17, 64, 200, 501][(seed * 5) % 6]
    w = pkg.synth.mixed(n_claim, n_node, 100 + seed, invalid=seed % 3 != 0)
    out, inv = _run(ctx, w)
    ref_out, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
    _assert_same(out, inv, ref_out, ref_inv, f"mixed seed {seed}")


# ---- large batches: hist tiles grown to multiples of 2048 (one wave of tiles); only 1M x 10k has enough counters
# (n_tiles x (n_node + 1) > 524,288) for the row-wise scan — 350k x 6,000 gives 86 x 6,001 = 516,086 ----
# The sort path is what every context takes at these sizes; the chain each shape takes holds from 86 to 170 SMs.
@pytest.mark.parametrize("n_claim,n_node,kind", [(350_000, 6000, "mixed"), (700_000, 1200, "mixed"), (1_000_000, 10_000, "cfg2")])
def test_large_batches_match_oracle(pkg, ctx, oracle, n_claim, n_node, kind):
    w = pkg.synth.mixed(n_claim, n_node, 77, invalid=True) if kind == "mixed" else pkg.synth.cfg2(n_claim, n_node)
    out, inv = _run(ctx, w)
    ref_out, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
    _assert_same(out, inv, ref_out, ref_inv, f"{kind} {n_claim} x {n_node}")
    scan = "scan_rows" if n_node == 10_000 else "scan8"
    pack = "pack1" if n_node == 1200 else "pack4"
    assert ctx.last_chain() == {"hist8_multi", scan, "scatter", pack}, ctx.last_chain()


def test_large_batch_through_a_replayed_graph(pkg, oracle):
    """The row-wise scan finds its predecessors' sums by an epoch that the kernel itself advances on the device: a captured
    graph replays with the same arguments and must still see a fresh epoch every time (eager, capture, replay, replay)."""
    R = pkg.records
    w = pkg.synth.cfg2(600_000, 6000)
    ref, _ = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, threads=8)
    with pkg.api.Context(device=0, flags=pkg.api.CFG_USE_GRAPH | pkg.api.CFG_NO_DIRECT) as g:
        g.set_table(w.table); g.set_inventory(w.gpus, w.node_off)
        pc = pkg.api.PinnedBuffer(w.n_claim, R.CLAIM_DTYPE); pc.array[:] = w.claims
        po = pkg.api.PinnedBuffer(w.n_out, R.OUT_DTYPE)
        for it in range(5):
            po.array[:] = 0
            g.allocate(pc.array, None, w.n_out, flags=pkg.api.F_FRESH_INVENTORY, out=po.array)
            assert po.array.tobytes() == ref.tobytes(), it
            assert g.last_chain() == {"hist8_multi", "scan_rows", "scatter", "pack4"}, it   # (a replay reports the captured chain)
        pc.free(); po.free()


# ---- the packers' lean plain-MIG loop: one lane per GPU and a ballot; 3 shift steps for rows of <= 8 slices, 4 wider ----
@pytest.mark.parametrize("seed,model,wide16,max_width", [
    (0, 0, False, 8), (1, 0, False, 32), (2, 1, False, 8), (3, 0, True, 8), (4, 0, True, 32), (5, 1, False, 32),
    (6, 0, False, 1), (7, 0, False, 9)])
def test_fast_loops_match_oracle(pkg, ctx, oracle, seed, model, wide16, max_width):
    for n_claim, n_node in ((700, 5), (6000, 40), (30000, 300)):
        w = pkg.synth.homog(n_claim, n_node, seed, model=model, wide16=wide16, max_width=max_width)
        out, inv = _run(ctx, w)
        ref_out, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims)
        _assert_same(out, inv, ref_out, ref_inv, f"homog seed {seed} {n_claim}x{n_node}")
        assert (out["status"] == 0).any() and (out["status"] != 0).any()


def test_edge_cases(pkg, ctx, oracle):
    R = pkg.records
    t = R.default_table()
    # empty batch
    g, off = R.make_inventory([8, 8], mig=True)
    ctx.set_table(t); ctx.set_inventory(g, off)
    assert len(ctx.allocate(np.zeros(0, dtype=R.CLAIM_DTYPE))) == 0
    assert ctx.get_inventory().tobytes() == g.tobytes()
    # empty inventory (nodes without GPUs), every claim fails the way the oracle says
    g0, off0 = R.make_inventory([0, 0, 0], mig=True)
    w = pkg.synth.mixed(300, 3, 5)
    w.gpus, w.node_off = g0, off0
    out, inv = _run(ctx, w)
    ref_out, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
    _assert_same(out, inv, ref_out, ref_inv, "empty inventory")
    # one node, one claim; maximum node width (32 GPUs); a run of exactly 32 and of 33 members
    g, off = R.make_inventory([32], mig=True)
    c = np.zeros(1 + 32 + 33, dtype=R.CLAIM_DTYPE)
    c["kind"] = R.KIND_MIG; c["count"] = 1; c["profile"] = R.GI_1_SLICE
    c["group"][1:33] = 5; c["group"][33:] = 6
    ctx.set_inventory(g, off)
    out = ctx.allocate(c)
    ref_out, ref_inv = oracle.allocate(g, off, t, c)
    _assert_same(out, ctx.get_inventory(), ref_out, ref_inv, "wide node + long runs")
    # all claims on a single node out of many (one long sequential chain, > one TMA ring)
    w = pkg.synth.cfg2(5000, 40)
    w.claims["node"] = 7
    out, inv = _run(ctx, w)
    ref_out, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims)
    _assert_same(out, inv, ref_out, ref_inv, "single hot node")


def test_deallocate_counts_slots_like_allocate(pkg, ctx, oracle):
    """A multi-count GPU claim that names no node has ONE (INVALID) slot in Allocate and in Deallocate (spec §9)."""
    R = pkg.records
    g, off = R.make_inventory([2], mig=False)
    c = np.zeros(2, dtype=R.CLAIM_DTYPE)
    c["kind"] = R.KIND_GPU
    c["count"] = [1, 2]
    c["node"] = [0, 1]
    out_off, n_out = R.out_offsets(c, 1)
    ctx.set_table(R.default_table()); ctx.set_inventory(g, off)
    out = ctx.allocate(c, out_off, n_out)
    ref_out, ref_inv = oracle.allocate(g, off, R.default_table(), c, out_off, n_out)
    _assert_same(out, ctx.get_inventory(), ref_out, ref_inv, "invalid multi-count claim")
    ctx.deallocate(c, out, out_off)                        # used to fail: slot count ran past n_out
    assert ctx.get_inventory().tobytes() == g.tobytes()


def test_out_off_out_of_range_is_an_error(pkg, ctx):
    R = pkg.records
    g, off = R.make_inventory([4], mig=False)
    c = np.zeros(2, dtype=R.CLAIM_DTYPE); c["kind"] = R.KIND_GPU; c["count"] = 2
    ctx.set_table(R.default_table()); ctx.set_inventory(g, off)
    with pytest.raises(pkg.api.DraError):
        ctx.allocate(c, out_off=np.array([0, 3], np.uint32), n_out=4)


# ---- state across batches, deallocate round trip ----------------------------------------------------
def test_batches_accumulate_and_deallocate_round_trips(pkg, ctx, oracle):
    w = pkg.synth.mixed(6000, 50, 42, invalid=False)
    ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
    half = len(w.claims) // 2
    c1, c2 = w.claims[:half], w.claims[half:]
    o1, n1 = pkg.records.out_offsets(c1, w.n_node)
    o2, n2 = pkg.records.out_offsets(c2, w.n_node)
    out1 = ctx.allocate(c1, o1, n1)
    out2 = ctx.allocate(c2, o2, n2)
    r1, gi = oracle.allocate(w.gpus, w.node_off, w.table, c1, o1, n1)
    r2, gj = oracle.allocate(gi, w.node_off, w.table, c2, o2, n2)
    _assert_same(out1, ctx.get_inventory(), r1, gj, "batch 1")
    assert out2.tobytes() == r2.tobytes()
    ctx.deallocate(c2, out2, o2)
    assert ctx.get_inventory().tobytes() == gi.tobytes()
    ctx.deallocate(c1, out1, o1)
    assert ctx.get_inventory().tobytes() == w.gpus.tobytes()
    # FRESH_INVENTORY evaluates against the loaded inventory regardless of what happened since
    out1b = ctx.allocate(c1, o1, n1)
    out1c = ctx.allocate(c1, o1, n1, flags=pkg.api.F_FRESH_INVENTORY)
    assert out1c.tobytes() == r1.tobytes() and out1b.tobytes() == r1.tobytes()
    assert ctx.get_inventory().tobytes() == gi.tobytes()


# ---- size-independent properties at full BASELINE sizes ----------------------------------------------
@pytest.mark.parametrize("cfg", ["cfg2", "cfg3", "cfg5"])
def test_properties_at_full_size(pkg, ctx, cfg):
    R = pkg.records
    w = pkg.synth.CONFIGS[cfg]()
    out, inv = _run(ctx, w)
    ok = out["status"] == 0
    # 1. conservation: slices newly occupied == sum of sizes of successful MIG claims
    newly = (inv["busy"] & ~w.gpus["busy"])
    pop = np.array([bin(int(x)).count("1") for x in newly]).sum()
    assert pop == int(out["size"][ok].sum())
    # 2. no overlap: per GPU, the placements handed out are pairwise disjoint and avoid the initial busy mask
    masks = ((1 << out["size"][ok].astype(np.int64)) - 1) << out["start"][ok].astype(np.int64)
    acc = w.gpus["busy"].astype(np.int64).copy()
    for gidx, m in zip(out["gpu"][ok], masks):
        assert acc[gidx] & m == 0
        acc[gidx] |= m
    assert np.array_equal(acc, inv["busy"].astype(np.int64))
    # 3. every placement is one the table offers, on a GPU of the claim's node
    node_of = w.gpus["node"][out["gpu"][ok]]
    assert np.array_equal(node_of, w.claims["node"][ok])
    ent = w.table[0][out["profile"][ok]]
    assert np.all((ent["start_mask"] >> out["start"][ok]) & 1) and np.array_equal(ent["size"], out["size"][ok])
    # 4. first-fit fixed point: replaying the failed claims against the final inventory still fails them all
    failed = w.claims[~ok]
    ctx.set_inventory(inv, w.node_off)
    again = ctx.allocate(failed)
    assert not (again["status"] == 0).any()
    # 5. deallocate everything -> initial inventory
    ctx.deallocate(w.claims, out)
    assert ctx.get_inventory().tobytes() == w.gpus.tobytes()


# ---- UnsuitableNodes ------------------------------------------------------------------------------------
def test_unsuitable_matches_oracle(pkg, ctx, oracle):
    R = pkg.records
    rng = np.random.default_rng(7)
    w = pkg.synth.mixed(3000, 40, 77, invalid=False)
    # pods of 1..4 claims; each with 1..12 candidate nodes (a few unknown)
    sizes = rng.integers(1, 5, size=3000)
    pod_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    pod_off = pod_off[pod_off <= len(w.claims)]
    if pod_off[-1] != len(w.claims):
        pod_off = np.append(pod_off, len(w.claims)).astype(np.uint32)
    n_pod = len(pod_off) - 1
    ncand = rng.integers(1, 13, size=n_pod)
    cand_off = np.concatenate([[0], np.cumsum(ncand)]).astype(np.uint32)
    cand_nodes = rng.integers(0, w.n_node + 2, size=int(cand_off[-1])).astype(np.uint32)
    # partially filled inventory makes the answer interesting
    _, inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims[:800], w.out_off[:800], int(w.out_off[800]))
    ctx.set_table(w.table); ctx.set_inventory(inv, w.node_off)
    got = ctx.unsuitable(w.claims, pod_off, cand_nodes, cand_off)
    ref = oracle.unsuitable(inv, w.node_off, w.table, w.claims, pod_off, cand_nodes, cand_off)
    assert got.tobytes() == ref.tobytes()
    assert 0 < np.unpackbits(got).sum() < int(cand_off[-1])
    assert ctx.get_inventory().tobytes() == inv.tobytes()      # pure


def test_launch_counter_counts_our_kernels(pkg, ctx):
    """Each path's chain as the library reports it, and one counted launch per kernel of it."""
    w = pkg.synth.cfg2(1000, 10)
    ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
    before = ctx.launch_count()
    ctx.allocate(w.claims)
    want = {"auto": {"fused_direct"}, "copy-engine": {"fused_staged"}, "bucket+pack": {"bucket_small", "pack1"}}[ctx.path]
    assert ctx.last_chain() == want and ctx.last_hist_tile() == 0
    assert ctx.launch_count() - before == len(want)
    ctx.set_inventory(w.gpus, w.node_off)
    before = ctx.launch_count()
    ctx.allocate(w.node_sorted().claims, flags=pkg.api.F_NODE_SORTED)
    assert ctx.last_chain() == {"sorted_prep", "pack1"}
    assert ctx.launch_count() - before == 2
    w = pkg.synth.cfg2(40_000, 300)
    ctx.set_inventory(w.gpus, w.node_off)
    before = ctx.launch_count()
    ctx.allocate(w.claims)
    assert ctx.last_chain() == {"hist8", "scan8", "scatter", "pack1"} and ctx.last_hist_tile() == 2048
    assert ctx.launch_count() - before == 4


# ---- selectors on the device (spec §10) -----------------------------------------------------------------
@pytest.mark.parametrize("seed", range(4))
def test_selectors_match_oracle(pkg, ctx, oracle, seed):
    w = pkg.synth.mixed([300, 2500, 6000, 12000][seed], [5, 40, 90, 160][seed], 200 + seed, invalid=seed % 2 == 0)
    attrs, sels = pkg.synth.with_selectors(w, seed)
    ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
    ctx.set_gpu_attrs(attrs); ctx.set_selectors(sels)
    oracle.set_selectors(attrs, sels)
    try:
        out = ctx.allocate(w.claims, w.out_off, w.n_out)
        inv = ctx.get_inventory()
        ref_out, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
        _assert_same(out, inv, ref_out, ref_inv, f"selectors seed {seed}")
        # UnsuitableNodes sees the same selectors
        pod_off = np.arange(0, len(w.claims) + 1, 3, dtype=np.uint32)
        if pod_off[-1] != len(w.claims):
            pod_off = np.append(pod_off, len(w.claims)).astype(np.uint32)
        n_pod = len(pod_off) - 1
        cand_off = (np.arange(n_pod + 1, dtype=np.uint32) * 2)
        cand_nodes = (np.arange(2 * n_pod, dtype=np.uint32) * 13) % np.uint32(w.n_node)
        ctx.set_inventory(w.gpus, w.node_off)
        got = ctx.unsuitable(w.claims, pod_off, cand_nodes, cand_off)
        ref = oracle.unsuitable(w.gpus, w.node_off, w.table, w.claims, pod_off, cand_nodes, cand_off)
        assert got.tobytes() == ref.tobytes()
    finally:
        oracle.set_selectors()
        ctx.set_selectors(None); ctx.set_gpu_attrs(None)


def test_unsuitable_dense_form_and_wide_nodes(pkg, ctx, oracle):
    """Dense form (every pod x every node, no candidate arrays) == explicit lists; 8-, 16- and 32-lane groups."""
    R = pkg.records
    for width in (8, 13, 32):
        g, off = R.make_inventory([width, 3, width, 0, 5], mig=True)
        g["flags"][::3] = 0
        w = pkg.synth.mixed(900, 5, 31 + width, invalid=False)
        w.gpus, w.node_off = g, off
        _, inv = oracle.allocate(g, off, w.table, w.claims[:200], w.out_off[:200], int(w.out_off[200]))
        pod_off = np.arange(0, 901, 3, dtype=np.uint32)
        n_pod = len(pod_off) - 1
        ctx.set_table(w.table); ctx.set_inventory(inv, off)
        dense = ctx.unsuitable(w.claims, pod_off)
        cand_nodes = np.tile(np.arange(5, dtype=np.uint32), n_pod)
        cand_off = (np.arange(n_pod + 1, dtype=np.uint32) * 5)
        sparse = ctx.unsuitable(w.claims, pod_off, cand_nodes, cand_off)
        ref = oracle.unsuitable(inv, off, w.table, w.claims, pod_off, cand_nodes, cand_off)
        assert dense.tobytes() == ref.tobytes() and sparse.tobytes() == ref.tobytes(), width


def test_cuda_graph_replay_of_the_host_call(pkg, oracle):
    """DRA_CFG_USE_GRAPH: the 2nd call of a shape is captured, later calls replay one graph; results must not
    depend on whether a call ran eagerly, was captured, or was replayed — including after the buffers' CONTENT
    changes and after the shape changes."""
    R = pkg.records
    w = pkg.synth.cfg2(3000, 40)
    ref, _ = oracle.allocate(w.gpus, w.node_off, w.table, w.claims)
    with pkg.api.Context(device=0, flags=pkg.api.CFG_USE_GRAPH) as g:
        g.set_table(w.table); g.set_inventory(w.gpus, w.node_off)
        pc = pkg.api.PinnedBuffer(w.n_claim, R.CLAIM_DTYPE); pc.array[:] = w.claims
        po = pkg.api.PinnedBuffer(w.n_out, R.OUT_DTYPE)
        F = pkg.api.F_FRESH_INVENTORY
        for it in range(5):                                   # eager, capture, replay, replay, replay
            po.array[:] = 0
            l0 = g.launch_count()
            g.allocate(pc.array, None, w.n_out, flags=F, out=po.array)
            assert po.array.tobytes() == ref.tobytes(), it
            assert g.launch_count() - l0 == 1
        # same buffers, new content: the graph reads what is there now
        w2 = pkg.synth.cfg2(3000, 40, seed_off=77)
        pc.array[:] = w2.claims
        ref2, _ = oracle.allocate(w.gpus, w.node_off, w.table, w2.claims)
        g.allocate(pc.array, None, w.n_out, flags=F, out=po.array)
        assert po.array.tobytes() == ref2.tobytes()
        # without FRESH the live inventory carries over between replays too
        g.reset_inventory()
        a = g.allocate(pc.array, None, w.n_out, flags=0, out=po.array).copy()
        b = g.allocate(pc.array, None, w.n_out, flags=0, out=po.array).copy()
        r1, inv1 = oracle.allocate(w.gpus, w.node_off, w.table, w2.claims)
        r2, _ = oracle.allocate(inv1, w.node_off, w.table, w2.claims)
        assert a.tobytes() == r1.tobytes() and b.tobytes() == r2.tobytes()
        # a different shape falls back to eager, then gets its own graph
        g.set_inventory(w.gpus, w.node_off)
        out = g.allocate(w.claims[:1000].copy())
        r3, _ = oracle.allocate(w.gpus, w.node_off, w.table, w.claims[:1000])
        assert out.tobytes() == r3.tobytes()
        pc.free(); po.free()


def test_adjacent_integer_searches(pkg, ctx, oracle):
    """limit.Megabyte (sharing.go:234-237, vectors of sharing_test.go) and the IMEX offset search
    (imex.go:336-349) as batch kernels, against the oracle's restatements."""
    q = pkg.sharing.quantity_value
    vals = [q(x) for x in ("2Gi", "1Gi", "10Mi", "10M", "1G", "1M", "0", "1048575", "1048576")] + [-5 * 2 ** 20, 2 ** 50 + 123]
    mib, valid = ctx.mps_limits(vals)
    for v, m, ok in zip(vals, mib, valid):
        assert (int(m), bool(ok)) == oracle.megabyte(v)
    assert list(mib[:6]) == [2048, 1024, 10, 9, 953, 0] and list(valid[:6]) == [True] * 5 + [False]
    rng = np.random.default_rng(3)
    doms = [[], [0], [0, 128, 384], list(range(0, 2048, 128)), [128, 256], list(range(0, 2048, 128))[:-1]]
    doms += [sorted(rng.choice(np.arange(0, 2048, 128), size=int(rng.integers(0, 16)), replace=False).tolist()) for _ in range(50)]
    got = ctx.imex_offsets(doms)
    assert list(got) == [oracle.imex_offset(d) for d in doms]
    wide = ctx.imex_offsets([list(range(0, 64 * 10, 10))], step=10, limit=1000)      # more than 32 windows
    assert wide[0] == oracle.imex_offset(list(range(0, 640, 10)), step=10, limit=1000) == 640


# ---- property-based: arbitrary small problems (random placement tables with odd sizes and arbitrary start masks,
# ragged blocked / pre-occupied inventories, every claim kind incl. malformed ones and co-location runs) -----------
def test_cuda_matches_oracle_on_arbitrary_problems(pkg, ctx, oracle):
    from hypothesis import HealthCheck, given, settings
    from test_oracle_properties import problems

    import os
    n_ex = int(os.environ.get("DRA_PROP_EXAMPLES", "0"))      # > 0: that many RANDOM examples instead of the fixed 120
    @settings(max_examples=n_ex or 120, deadline=None, suppress_health_check=list(HealthCheck), derandomize=n_ex == 0, database=None)
    @given(problems())
    def run(prob):
        g, off, t, c, out_off, n_out = prob
        ctx.set_table(t)
        ctx.set_inventory(g, off)
        if len(c):                                         # UnsuitableNodes first (pure): every pod x every node
            cut = [i for i in range(1, len(c)) if c["group"][i] == 0 or c["group"][i] != c["group"][i - 1]]
            pod_off = np.array([0] + cut[::2] + [len(c)], dtype=np.uint32)     # pods never split a co-location run
            n_pod, n_node = len(pod_off) - 1, len(off) - 1
            bits = ctx.unsuitable(c, pod_off)
            cand_nodes = np.tile(np.arange(n_node, dtype=np.uint32), n_pod)
            cand_off = (np.arange(n_pod + 1, dtype=np.uint32) * n_node).astype(np.uint32)
            ref_bits = oracle.unsuitable(g, off, t, c, pod_off, cand_nodes, cand_off)
            assert bits[: len(ref_bits)].tobytes() == ref_bits.tobytes(), "UnsuitableNodes differs"
            assert ctx.get_inventory().tobytes() == g.tobytes()
        out = ctx.allocate(c, out_off, n_out)
        inv = ctx.get_inventory()
        ref_out, ref_inv = oracle.allocate(g, off, t, c, out_off, n_out)
        _assert_same(out, inv, ref_out, ref_inv, "arbitrary problem")
        if len(c):                                         # Deallocate (spec §9) on the device: back to the start
            ctx.deallocate(c, out, out_off)
            assert ctx.get_inventory().tobytes() == g.tobytes()

    run()


def test_cuda_selectors_match_oracle_on_arbitrary_problems(pkg, ctx, oracle):
    """Random selector programs (well-formed trees and garbage), random attributes, every claim kind: the device's
    predicate evaluation and its interplay with runs / the failure memo against the oracle (spec §10)."""
    import os
    from hypothesis import HealthCheck, given, settings
    from test_oracle_selector_properties import selector_problems
    R = pkg.records
    n_ex = int(os.environ.get("DRA_PROP_EXAMPLES", "0"))

    @settings(max_examples=n_ex or 100, deadline=None, suppress_health_check=list(HealthCheck), derandomize=n_ex == 0, database=None)
    @given(selector_problems(), __import__("hypothesis").strategies.integers(0, 3))
    def run(prob, every):
        g, off, t, c, out_off, n_out, attrs, sels, sid = prob
        cs = c.copy()                                      # every claim, or every 2nd / 3rd / 4th, carries the selector
        pick = (np.arange(len(cs)) % (every + 1)) == 0
        gm = pick & ((cs["kind"] == R.KIND_GPU) | (cs["kind"] == R.KIND_MIG))
        cs["mem_limit_mib"] = np.where(gm, sid, cs["mem_limit_mib"])
        cs["group"] = np.where(pick & (cs["kind"] == R.KIND_SHARED), sid, cs["group"])
        ctx.set_table(t); ctx.set_inventory(g, off)
        ctx.set_gpu_attrs(attrs); ctx.set_selectors(sels.reshape(-1, R.SEL_MAX_INS))
        oracle.set_selectors(attrs, sels)
        try:
            out = ctx.allocate(cs, out_off, n_out)
            inv = ctx.get_inventory()
            ref_out, ref_inv = oracle.allocate(g, off, t, cs, out_off, n_out)
            _assert_same(out, inv, ref_out, ref_inv, "selectors on an arbitrary problem")
        finally:
            oracle.set_selectors()
            ctx.set_selectors(None); ctx.set_gpu_attrs(None)

    run()
