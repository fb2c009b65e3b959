"""GPU suite: the exhaustive pod search (spec §12, pod_eval in dra_device.cuh) at its structural limits — pods of 31-33
claims, starts of 8 and above at positions 16 and above (the st_hi half of the start stack), resumes from start 15 and
from the last lane of a group, searches of exactly 4095 / 4096 / 4097 descents, every lane width of the exhaustive
UnsuitableNodes kernel, co-location and selectors inside the search, and long pod sequences on one node.

Every case compares OutRecs and inventory byte for byte with the C oracle, with and without F_EXHAUSTIVE, and the
exhaustive UnsuitableNodes bitmap with the oracle's in the dense form and with candidate lists; then it asserts the
property it exists for.  The literal fixtures and their descent counts are checked without a GPU in
tests/test_pod_search_fixtures.py."""

import numpy as np
import pytest

import test_pod_search_fixtures as F
from test_gpu_parity import _assert_same

pytestmark = pytest.mark.gpu

R = F.R


class Inv:
    """Fixtures side by side: one node per fixture, the fixtures' pods retargeted to their node, in fixture order."""

    def __init__(self, fixtures, table=None):
        self.fx = fixtures
        self.table = F.fixture_table() if table is None else table
        self.gpus = np.concatenate([f["gpus"] for f in fixtures])
        self.node_off = np.zeros(len(fixtures) + 1, np.uint32)
        self.node_off[1:] = np.cumsum([len(f["gpus"]) for f in fixtures])
        self.gpus["node"] = np.repeat(np.arange(len(fixtures), dtype=np.uint32), np.diff(self.node_off))
        cs, self.pods = [], []                           # pods[k] = (fixture index, pod index, c0, c1)
        n = 0
        for k, f in enumerate(fixtures):
            for q, p in enumerate(f["pods"]):
                p = p.copy()
                p["node"] = k
                cs.append(p)
                self.pods.append((k, q, n, n + len(p)))
                n += len(p)
        self.claims = np.concatenate(cs)
        self.pod_off = np.array([0] + [c1 for _, _, _, c1 in self.pods], np.uint32)
        self.n_node = len(fixtures)

    def slices(self, out, name):
        """The OutRecs of fixture `name`'s pods, one array per pod (every claim has one slot here)."""
        k = next(i for i, f in enumerate(self.fx) if f["name"] == name)
        return [out[c0:c1] for kk, _, c0, c1 in self.pods if kk == k], int(self.node_off[k])


def _flags(api, oracle):
    return ((0, 0), (api.F_EXHAUSTIVE, oracle.F_EXHAUSTIVE))


def _allocate(pkg, ctx, oracle, inv, what):
    """allocate_pods without and with F_EXHAUSTIVE on a fresh copy of the inventory, against the oracle."""
    res = {}
    for flags, oflags in _flags(pkg.api, oracle):
        ctx.set_table(inv.table); ctx.set_inventory(inv.gpus, inv.node_off)
        out = ctx.allocate_pods(inv.claims, inv.pod_off, flags=flags)
        ref, ref_inv = oracle.allocate_pods(inv.gpus, inv.node_off, inv.table, inv.claims, inv.pod_off, flags=oflags)
        _assert_same(out, ctx.get_inventory(), ref, ref_inv, f"{what} flags {flags}")
        res[bool(flags)] = out
    return res[False], res[True]


def _candidates(n_pod, n_node, rng):
    """Candidate lists: every node, one node twice, and nodes beyond the inventory."""
    lists = []
    for _ in range(n_pod):
        c = list(rng.permutation(n_node)) + [int(rng.integers(0, n_node)), n_node, n_node + 7, 0xFFFFFFFF]
        lists.append(np.array(c, np.uint32))
    off = np.zeros(n_pod + 1, np.uint32)
    off[1:] = np.cumsum([len(x) for x in lists])
    return np.concatenate(lists), off


def _unsuitable(pkg, ctx, oracle, gpus, node_off, table, claims, pod_off, what, seed=0):
    """Exhaustive (and first-fit) UnsuitableNodes against the oracle, dense and with candidate lists.  Returns the
    exhaustive dense verdict as a [pod, node] bool array."""
    api = pkg.api
    n_pod, n_node = len(pod_off) - 1, len(node_off) - 1
    ctx.set_table(table); ctx.set_inventory(gpus, node_off)
    dn = np.tile(np.arange(n_node, dtype=np.uint32), n_pod)
    do = (np.arange(n_pod + 1, dtype=np.uint64) * n_node).astype(np.uint32)
    cn, co = _candidates(n_pod, n_node, np.random.default_rng(seed))
    dense = None
    for flags, oflags in _flags(api, oracle):
        bits = ctx.unsuitable(claims, pod_off, flags=flags)
        ref = oracle.unsuitable(gpus, node_off, table, claims, pod_off, dn, do, flags=oflags)
        assert bits.tobytes() == ref.tobytes(), f"{what}: dense UnsuitableNodes flags {flags} differs"
        cbits = ctx.unsuitable(claims, pod_off, cn, co, flags=flags)
        cref = oracle.unsuitable(gpus, node_off, table, claims, pod_off, cn, co, flags=oflags)
        assert cbits.tobytes() == cref.tobytes(), f"{what}: candidate-list UnsuitableNodes flags {flags} differs"
        if flags:
            dense = np.unpackbits(bits, bitorder="little")[: n_pod * n_node].reshape(n_pod, n_node).astype(bool)
            c = np.unpackbits(cbits, bitorder="little")[: int(co[-1])].astype(bool)
            for p in range(n_pod):                       # the candidate form answers each pair as the dense one does
                nodes = cn[co[p]: co[p + 1]]
                known = nodes < n_node
                assert (c[co[p]: co[p + 1]][known] == dense[p, nodes[known]]).all()
                assert not c[co[p]: co[p + 1]][~known].any()
    return dense


def _reach(recs, base, fx):
    for p, g, s in fx.get("reach", []):
        assert (int(recs[p]["gpu"]), int(recs[p]["start"])) == (base + g, s), \
            f"{fx['name']}: position {p} at {(int(recs[p]['gpu']) - base, int(recs[p]['start']))}, not {(g, s)}"


def _own_node_verdict(inv, dense):
    """Exhaustive verdict of each pod on its own fixture's node."""
    return [bool(dense[i, k]) for i, (k, _, _, _) in enumerate(inv.pods)]


# ---- 1. deep pods ------------------------------------------------------------------------------------------------------
def test_deep_pods(pkg, ctx, oracle):
    inv = Inv(F.deep_fixtures())
    ff, ex = _allocate(pkg, ctx, oracle, inv, "deep pods")
    for fx in inv.fx:
        (first, *later), base = inv.slices(ex, fx["name"])
        (ff_first, *ff_later), _ = inv.slices(ff, fx["name"])
        if fx["name"] == "deep_33":
            assert set(first["status"]) == set(ff_first["status"]) == {R.ST_INVALID}
            continue
        if fx["name"] == "deep_31_then_fail":
            assert set(ff_first["status"]) == {R.ST_POD}
            assert len(set(first["status"])) == 1 and first["status"][0] in (R.ST_POD, R.ST_SEARCH_LIMIT)
            for recs in (later, ff_later):                  # the node as it was before the failed pod
                assert [int(r["status"][0]) for r in recs] == [0, 0]
                assert [int(r["gpu"][0]) - base for r in recs] == [0, 1] and [int(r["start"][0]) for r in recs] == [0, 0]
            continue
        assert (first["status"] == 0).all(), fx["name"]
        _reach(first, base, fx)
        if fx.get("resume"):                             # placed only by backtracking
            assert set(ff_first["status"]) == {R.ST_POD}, fx["name"]
        else:
            assert first.tobytes() == ff_first.tobytes()
    recs, _ = inv.slices(ex, "deep_32_high_starts")
    assert len(recs[0]) == 32 and (recs[0]["start"][16:] >= 8).all()
    dense = _unsuitable(pkg, ctx, oracle, inv.gpus, inv.node_off, inv.table, inv.claims, inv.pod_off, "deep pods")
    for i, (k, q, c0, c1) in enumerate(inv.pods):
        if c1 - c0 > R.MAX_POD:
            assert not dense[i].any()                    # 33 claims: unsuitable everywhere
    own = dict(zip([(inv.fx[k]["name"], q) for k, q, _, _ in inv.pods], _own_node_verdict(inv, dense)))
    assert own[("deep_32_high_starts", 0)] and own[("deep_32_mixed", 0)] and own[("deep_mig_at_31", 0)]
    assert own[("deep_backtrack_at_16", 0)] and own[("deep_backtrack_across_16", 0)]
    assert not own[("deep_31_then_fail", 0)]


# ---- 2. resume edges ---------------------------------------------------------------------------------------------------
def test_resume_edges(pkg, ctx, oracle):
    inv = Inv(F.resume_fixtures())
    ff, ex = _allocate(pkg, ctx, oracle, inv, "resume")
    for fx in inv.fx:
        (recs,), base = inv.slices(ex, fx["name"])
        (ff_recs,), _ = inv.slices(ff, fx["name"])
        assert (recs["status"] == 0).all() and set(ff_recs["status"]) == {R.ST_POD}, fx["name"]
        _reach(recs, base, fx)


@pytest.mark.parametrize("name,width", [("resume_lane_7", 8), ("resume_lane_15", 16)])
def test_resume_on_last_lane_in_unsuitable(pkg, ctx, oracle, name, width):
    """Inventories whose widest node is 8 / 16 GPUs (W = 8 / 16, four / two searches per warp): the fixture's node five
    times, so that every group of a warp resumes on its lane W - 1, next to an empty node of the same width."""
    fx = next(f for f in F.resume_fixtures() if f["name"] == name)
    empty = dict(name="empty", gpus=F.node([0] * width), pods=[])
    inv = Inv([fx] * 5 + [empty])
    dense = _unsuitable(pkg, ctx, oracle, inv.gpus, inv.node_off, inv.table, inv.claims, inv.pod_off, name)
    assert dense.all()


# ---- 3. budget boundary ------------------------------------------------------------------------------------------------
def test_budget_boundary(pkg, ctx, oracle):
    inv = Inv(F.budget_fixtures())
    want = {"fail_4095": R.ST_POD, "fail_4096": R.ST_POD, "fail_4097": R.ST_SEARCH_LIMIT,
            "ok_4095": R.ST_OK, "ok_4096": R.ST_OK, "ok_4097": R.ST_SEARCH_LIMIT}
    ff, ex = _allocate(pkg, ctx, oracle, inv, "budget")
    for fx in inv.fx:
        (recs,), _ = inv.slices(ex, fx["name"])
        (ff_recs,), _ = inv.slices(ff, fx["name"])
        assert set(recs["status"]) == {want[fx["name"]]}, f"{fx['name']}: {set(recs['status'])}"
        assert set(ff_recs["status"]) == {R.ST_POD}
    dense = _unsuitable(pkg, ctx, oracle, inv.gpus, inv.node_off, inv.table, inv.claims, inv.pod_off, "budget")
    own = _own_node_verdict(inv, dense)
    assert own == [want[f["name"]] == R.ST_OK for f in inv.fx]


# ---- 4. lane widths of the exhaustive UnsuitableNodes ------------------------------------------------------------------
@pytest.mark.parametrize("widest", [8, 9, 16, 17, 32])
def test_unsuitable_lane_widths(pkg, ctx, oracle, widest):
    """Nodes: the widest one with only its last GPU free (the 7 x 1g + 7g pod exhausts the budget there, a 1g fits in one
    descent), widths 0, 1 and widest - 1, a widest node whose last GPU resumes, and two more.  Pods interleave
    searches that fail at the pre-check, fit in one descent and exhaust the budget, so a warp's groups run searches of
    very different length; 7 nodes put the pods' pairs at every offset within a warp."""
    t = R.default_table()
    W = widest
    full = 0xFF
    widths, busy = [], []

    def add(b):
        widths.append(len(b)); busy.extend(b)

    add([full] * (W - 1) + [0])                          # n0: the last GPU free
    add([])                                              # n1: no GPU
    add([0])                                             # n2: one empty GPU
    add([0] * (W - 1))                                   # n3: widest - 1, empty
    add([full] * (W - 1) + [0x10])                       # n4: last GPU with slice 4 busy
    add([full] * (W - 1) + [0])                          # n5 = n0
    add([0x10])                                          # n6: one GPU, slice 4 busy
    g, off = R.make_inventory(widths, mig=True)
    g["busy"] = busy
    P = {"limit": [R.GI_1_SLICE] * 7 + [R.GI_7_SLICE],
         "pre": [R.GI_1_SLICE, R.GI_8_SLICE],            # a profile the table does not offer: fails at the pre-check
         "fit": [R.GI_1_SLICE],
         "resume": [R.GI_1_SLICE, R.GI_3_SLICE],         # one group: the 1g leaves slices 0-3 for the 3g
         "p32": [R.GI_1_SLICE] * 32,
         "p33": [R.GI_1_SLICE] * 33}
    order = ["limit", "pre", "fit", "limit", "resume", "p32", "pre", "limit", "p33", "fit", "resume", "limit", "pre", "fit"]
    cs = []
    for name in order:
        c = F.mig(*P[name], group=1 if name == "resume" else 0)
        cs.append(c)
    claims = np.concatenate(cs)
    pod_off = np.zeros(len(cs) + 1, np.uint32)
    pod_off[1:] = np.cumsum([len(c) for c in cs])
    dense = _unsuitable(pkg, ctx, oracle, g, off, t, claims, pod_off, f"widest {W}", seed=W)
    rows = {name: dense[order.index(name)] for name in P}
    assert not rows["limit"][0] and not rows["limit"][2] and rows["limit"][3]      # budget on n0 / n2, a fit on n3
    assert rows["fit"][[0, 2, 3, 5]].all() and not rows["fit"][1]
    assert not rows["pre"].any() and not rows["p33"].any()
    assert rows["p32"][3] and not rows["p32"][0]
    assert rows["resume"][4] and rows["resume"][6]
    # the statuses behind the first row: SEARCH_LIMIT on n0 and n2 (the budget, not a plain failure)
    for n in (0, 2):
        c = F.mig(*P["limit"]); c["node"] = n
        out, _ = oracle.allocate_pods(g, off, t, c, np.array([0, len(c)], np.uint32), flags=oracle.F_EXHAUSTIVE)
        assert set(out["status"]) == {R.ST_SEARCH_LIMIT}


# ---- 5. co-location and selectors in the search ------------------------------------------------------------------------
def _selector_fixtures():
    mig_only = R.GPU_MIG_ENABLED
    return [
        # a SHARED claim whose selector id (its group field) is 3, next to MIG group 3: it co-locates nothing
        dict(name="shared_selector_equals_group", gpus=F.node([0, 0, 0], flags=[0, mig_only, mig_only]),
             pods=[F.claims(("shared", 0, 3), ("mig", F.G1, 3), ("mig", F.G4, 3))], reach=[(1, 1, 0), (2, 1, 8)]),
        # MIG claims of one pod with different selectors: selector 1 = GPU 1 only, selector 2 = GPU 2 only; the 4g on
        # GPU 1 (slice 8 busy) sends the first 1g back to start 9
        dict(name="mig_per_claim_selectors", gpus=F.node([0, 0x0100, 0]),
             pods=[F.claims(("mig", F.G1, 0, 1), ("mig", F.G2, 0, 2), ("mig", F.G4, 0, 1))],
             reach=[(0, 1, 9), (1, 2, 0), (2, 1, 0)]),
        # a selector id beyond the table: that claim INVALID, the others POD
        dict(name="selector_beyond_table", gpus=F.node([0, 0]),
             pods=[F.claims(("mig", F.G1), ("mig", F.G1, 0, 4), ("mig", F.G2))]),
    ]


def _selectors(inv):
    attrs = np.zeros(len(inv.gpus), dtype=R.ATTR_DTYPE)
    attrs["index"] = np.arange(len(inv.gpus)) - np.repeat(inv.node_off[:-1], np.diff(inv.node_off))
    sels = np.stack([R.selector(("cmp", R.ATTR_INDEX, R.CMP_EQ, 1)), R.selector(("cmp", R.ATTR_INDEX, R.CMP_EQ, 2)),
                     R.selector(("cmp", R.ATTR_INDEX, R.CMP_GE, 0))])
    return attrs, sels


def test_colocation_and_selectors(pkg, ctx, oracle):
    inv = Inv(F.colocation_fixtures() + _selector_fixtures())
    attrs, sels = _selectors(inv)
    ctx.set_gpu_attrs(attrs); ctx.set_selectors(sels)
    oracle.set_selectors(attrs, sels)
    try:
        ff, ex = _allocate(pkg, ctx, oracle, inv, "co-location")
        for fx in inv.fx:
            (recs,), base = inv.slices(ex, fx["name"])
            if fx["name"] == "selector_beyond_table":
                assert list(recs["status"]) == [R.ST_POD, R.ST_INVALID, R.ST_POD]
                continue
            assert (recs["status"] == 0).all(), fx["name"]
            _reach(recs, base, fx)
            c = fx["pods"][0]
            for grp in set(int(x) for x in c["group"][c["kind"] == R.KIND_MIG]) - {0}:
                members = (c["kind"] == R.KIND_MIG) & (c["group"] == grp)
                assert len(set(recs["gpu"][members])) == 1, f"{fx['name']}: group {grp} split"
        (recs,), base = inv.slices(ex, "group_moves_member")
        (ff_recs,), _ = inv.slices(ff, "group_moves_member")
        assert set(ff_recs["status"]) == {R.ST_POD} and int(recs["gpu"][0]) == base + 1
        (recs,), base = inv.slices(ex, "shared_selector_equals_group")
        assert int(recs["gpu"][0]) == base and int(recs["profile"][0]) == R.PROFILE_SHARED
        dense = _unsuitable(pkg, ctx, oracle, inv.gpus, inv.node_off, inv.table, inv.claims, inv.pod_off, "co-location")
        assert _own_node_verdict(inv, dense) == [f["name"] != "selector_beyond_table" for f in inv.fx]
    finally:
        oracle.set_selectors()
        ctx.set_selectors(None); ctx.set_gpu_attrs(None)


# ---- 6. pod sequences on one node --------------------------------------------------------------------------------------
def _sequences(seed=5):
    """60 pods on each of four nodes (32, 17, 9 and 1 GPUs of the 16-slice part, partly busy), interleaved across the
    nodes: successes and failures alternate on every node."""
    rng = np.random.default_rng(seed)
    widths = [32, 17, 9, 1]
    fx = []
    for w in widths:
        busy = np.where(rng.integers(0, 3, w) == 0, rng.integers(0, 1 << 16, w), 0).astype(np.uint16)
        fx.append(dict(name=f"seq{w}", gpus=F.node(busy), pods=[]))
    profs = np.array([F.G1, F.G1, F.G1, F.G2, F.G2, F.G3, F.G4, F.G7])
    for q in range(60):
        for k, w in enumerate(widths):
            n = int(rng.integers(1, 7 if w > 1 else 4))
            c = F.mig(*profs[rng.integers(0, len(profs), n)])
            if n > 1 and rng.integers(0, 3) == 0:
                c["group"][rng.integers(0, n, 2)] = 1 + q
            fx[k]["pods"].append(c)
    return fx


def test_pod_sequences_and_fresh_inventory(pkg, ctx, oracle):
    api = pkg.api
    inv = Inv(_sequences())
    ff, ex = _allocate(pkg, ctx, oracle, inv, "sequences")
    for out in (ff, ex):
        for fx in inv.fx:
            pods, _ = inv.slices(out, fx["name"])
            ok = [bool((p["status"] == 0).all()) for p in pods]
            assert any(not a and b for a, b in zip(ok, ok[1:])), f"{fx['name']}: no success after a failure"
    # F_FRESH_INVENTORY: the second call starts from the pristine inventory, not from the first call's state
    ctx.set_table(inv.table); ctx.set_inventory(inv.gpus, inv.node_off)
    first = ctx.allocate_pods(inv.claims, inv.pod_off, flags=api.F_EXHAUSTIVE)
    assert ctx.get_inventory().tobytes() != inv.gpus.tobytes()
    assert first.tobytes() == ex.tobytes()
    again = ctx.allocate_pods(inv.claims, inv.pod_off, flags=api.F_EXHAUSTIVE | api.F_FRESH_INVENTORY)
    ref, ref_inv = oracle.allocate_pods(inv.gpus, inv.node_off, inv.table, inv.claims, inv.pod_off, flags=oracle.F_EXHAUSTIVE)
    _assert_same(again, ctx.get_inventory(), ref, ref_inv, "F_FRESH_INVENTORY")
    stale, _ = oracle.allocate_pods(ctx.get_inventory(), inv.node_off, inv.table, inv.claims, inv.pod_off,
                                    flags=oracle.F_EXHAUSTIVE)
    assert stale.tobytes() != ref.tobytes(), "the second call would not tell fresh from stale state"


# ---- 7. the same fixtures through the sharded call ---------------------------------------------------------------------
@pytest.mark.parametrize("world", [1, 2])
def test_sharded_call_matches_single_context(pkg, oracle, world):
    import shard_world as S
    api = pkg.api
    inv = Inv(F.deep_fixtures() + F.budget_fixtures() + F.colocation_fixtures() + _selector_fixtures())
    attrs, sels = _selectors(inv)
    bounds = [0, inv.n_node] if world == 1 else [0, inv.n_node // 2, inv.n_node]
    W = S.World(pkg, inv.table, inv.node_off, inv.gpus, world, bounds, attrs=attrs, sels=sels, n_out_max=1 << 16)
    oracle.set_selectors(attrs, sels)
    try:
        with api.Context(device=0) as single:
            single.set_table(inv.table); single.set_gpu_attrs(attrs); single.set_selectors(sels)
            # the first call starts from the pristine inventory; the later ones from it again, by F_FRESH_INVENTORY
            for flags in (api.F_EXHAUSTIVE, api.F_FRESH_INVENTORY, api.F_EXHAUSTIVE | api.F_FRESH_INVENTORY):
                single.set_inventory(inv.gpus, inv.node_off)
                want = single.allocate_pods(inv.claims, inv.pod_off, flags=flags & ~api.F_FRESH_INVENTORY)
                tables = S.pods(W, inv.claims, inv.pod_off, None, len(inv.claims), flags)
                for r, t in enumerate(tables):
                    assert t.tobytes() == want.tobytes(), f"world {world} rank {r} flags {flags}: table differs"
                for r in range(world):
                    g0, g1 = W.gpu_range(r)
                    assert W.ctxs[r].get_inventory()[g0:g1].tobytes() == single.get_inventory()[g0:g1].tobytes()
    finally:
        oracle.set_selectors()
        W.close()
