"""GPU suite: preemption with disruption budgets (spec §14, "Disruption budgets") at its edges, on one inventory
(dra_preempt_pdb_batch) and on a sharded world of one device (dra_preempt_pdb_batch_global_device).  Every call's eight
outputs are compared byte for byte with preempt_oracle.preempt_pdb on the same inventory, nothing may be written past an
output or into one the call was not given, and no inventory word may change, live or pristine.  A call the oracle
rejects fails with DRA_E_INVAL and writes nothing.

1. the hand-written fixtures of test_preempt_pdb.py, also with an unused 9- and 17-GPU node appended (lane widths 16, 32),
   and on sharded worlds
2. crowded nodes: thousands of running pods in one to three budgets, budget chains walked hundreds of links, members above
   the pending pod's priority, more than 1,023 violations on a pair
3. every bucketing path of the running pods, with budgets
4. random problems (test_preempt_pdb.pdb_problems), single and sharded
5. sharded packing and ownership: the crowded node on each rank, a partial holding the SEARCH_LIMIT bit and a violation
   count, the violation key across ranks, the chosen node's victim row behind an empty window
6. every combination of the optional outputs
7. one context reused by budgeted calls that grow and shrink every size, interleaved with the calls sharing its buffers
8. the documented limits, and the wrapper's check of run_pdb's length"""
import ctypes as C
import dataclasses
import functools
import inspect

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

import capacity_oracle as CO
import preempt_oracle as P
import preempt_place_oracle as PP
import shard_world as S
import test_preempt_pdb as TB
from preempt_problems import I32_MAX, NONE, Problem
from shard_world import Running
from test_gpu_preempt_edges import CONFIGS, N_EX, _n_sm, _pick, _shared_world, _widen

pytestmark = pytest.mark.gpu
SENT, SLACK, SHARD_SENT = 0xA5, 16, 0x5C
NAMES = S.PREEMPT_NAMES
OPTIONAL = (0, 1, 6, 7)                 # pair_status, pair_victims, pair_violations, pod_violations: each may be NULL
ALL = (True,) * 4
PDB_MAX_RUNNING = 1 << 29               # DRA_PDB_MAX_RUNNING
ALLOWED_EDGES = (0, 1, 7, 255, 256, 1023, I32_MAX)


@pytest.fixture(scope="module")
def bctx(pkg):
    c = pkg.api.Context(device=0)
    yield c
    c.close()


@dataclasses.dataclass
class Case(Problem):
    """A §14 problem with budgets: run_pdb (None: no array), allowed (None: no array) and n_pdb (None: len(allowed))"""
    run_pdb: np.ndarray | None = None
    allowed: np.ndarray | None = None
    n_pdb: int | None = None

    @property
    def npdb(self):
        return (0 if self.allowed is None else len(self.allowed)) if self.n_pdb is None else self.n_pdb

    def ref(self, gpus=None, flags=None, mv=None):
        cn, co = self.cand_arrays()
        return P.preempt_pdb(self.gpus if gpus is None else gpus, self.node_off, self.table, self.claims, self.pod_off,
                             self.prio, self.run_claims, self.run_pod_off, self.run_prio, self.run_out, self.run_pdb,
                             self.allowed, self.run_out_off, cn, co, self.max_victims if mv is None else mv,
                             self.flags if flags is None else flags, n_pdb=self.n_pdb)


def case(pb, run_pdb, allowed, n_pdb=None, **kw):
    d = {f.name: getattr(pb, f.name) for f in dataclasses.fields(Problem)}
    d.update(kw)
    return Case(**d, run_pdb=None if run_pdb is None else np.asarray(run_pdb, np.uint32),
                allowed=None if allowed is None else np.asarray(allowed, np.int32), n_pdb=n_pdb)


def _arr(x, dtype):
    return None if x is None else np.ascontiguousarray(x, dtype=dtype)


def _p(x):
    return None if x is None else x.ctypes.data


def _raw(pkg, ctx, cs, flags, mv, asked=ALL, run=None):
    """dra_preempt_pdb_batch on sentinel-filled outputs SLACK elements longer than the call needs, the optional ones
    passed only where `asked` (OPTIONAL order) says; `run`: a RunningPods to pass instead of cs's.  Returns (rc, outputs
    in NAMES order)."""
    A, R = pkg.api, pkg.records
    n_pod = len(cs.pod_off) - 1
    cn, co = cs.cand_arrays()
    n_pair = n_pod * ctx.n_node if co is None else int(co[-1])

    def filled(n, dtype):
        return np.full((max(n, 1) + SLACK) * np.dtype(dtype).itemsize, SENT, np.uint8).view(dtype)
    outs = [filled(n_pair, np.uint8), filled(n_pair, np.uint32), filled(n_pod, np.uint32), filled(n_pod, np.uint8),
            filled(n_pod, np.uint32), filled(n_pod * mv, np.uint32), filled(n_pair, np.uint32), filled(n_pod, np.uint32)]
    c, po, pr = _arr(cs.claims, R.CLAIM_DTYPE), _arr(cs.pod_off, np.uint32), _arr(cs.prio, np.int32)
    cn, co = _arr(cn, np.uint32), _arr(co, np.uint32)
    keep = [_arr(cs.run_claims, R.CLAIM_DTYPE), _arr(cs.run_pod_off, np.uint32), _arr(cs.run_prio, np.int32),
            _arr(cs.run_out, R.OUT_DTYPE), _arr(cs.run_out_off, np.uint32), _arr(cs.run_pdb, np.uint32),
            _arr(cs.allowed, np.int32)]
    rc, rpo, rpr, ro, roo, rp, al = keep
    if run is None:
        run = A.RunningPods(_p(rc), len(rc), _p(rpo), len(rpo) - 1, _p(rpr), _p(roo), _p(ro), len(ro))
    bud = A.DisruptionBudgets(_p(rp), _p(al), cs.npdb)
    p = [_p(o) if k not in OPTIONAL or asked[OPTIONAL.index(k)] else None for k, o in enumerate(outs)]
    rc_ = ctx._lib.dra_preempt_pdb_batch(ctx._h, _p(c), len(c), _p(po), _p(pr), n_pod, _p(cn), _p(co), C.byref(run),
                                         C.byref(bud), p[0], p[1], p[6], p[2], p[3], p[4], p[7], p[5], mv, flags)
    return rc_, outs


def _call(pkg, ctx, cs, pristine, flags=None, mv=None, chain=("preempt",), asked=ALL, what=""):
    """dra_preempt_pdb_batch on cs against the oracle on the context's live inventory.  Afterwards the live inventory is
    unchanged and, reset, equals `pristine`.  Returns the outputs (None for one not asked for), or None when the call
    must fail (E_INVAL, nothing written)."""
    A = pkg.api
    flags = cs.flags if flags is None else flags
    mv = cs.max_victims if mv is None else mv
    before = ctx.get_inventory()
    rc_, outs = _raw(pkg, ctx, cs, A.F_EXHAUSTIVE if flags else 0, mv, asked)
    try:
        ref = cs.ref(before, flags, mv)
    except ValueError:
        ref = None
    got = None
    if ref is None:
        assert rc_ == A.E_INVAL, what
        assert all((o.view(np.uint8) == SENT).all() for o in outs), f"{what}: an output was written"
    else:
        assert rc_ == A.OK, what
        chain_now = ctx.last_chain()
        for c in chain:
            assert c in chain_now, (what, c, chain_now)
        got = []
        for k, (name, o, y) in enumerate(zip(NAMES, outs, ref)):
            if k in OPTIONAL and not asked[OPTIONAL.index(k)]:
                assert (o.view(np.uint8) == SENT).all(), f"{what}: {name} written without being asked"
                got.append(None)
                continue
            x = o[: y.size]
            if x.tobytes() != y.tobytes():
                bad = np.flatnonzero(x != y.reshape(-1))[:5]
                pytest.fail(f"{what}: {name} differs at {bad}: device {x[bad]} oracle {y.reshape(-1)[bad]}")
            assert (o[y.size:].view(np.uint8) == SENT).all(), f"{what}: written past {name}"
            got.append(x.reshape(y.shape))
    assert ctx.get_inventory().tobytes() == before.tobytes(), f"{what}: live inventory changed"
    ctx.reset_inventory()
    assert ctx.get_inventory().tobytes() == pristine.tobytes(), f"{what}: pristine inventory changed"
    return got


def _load(ctx, pb):
    ctx.set_table(pb.table)
    ctx.set_inventory(pb.gpus, pb.node_off)


def _run(pkg, ctx, cs, **kw):
    _load(ctx, cs)
    return _call(pkg, ctx, cs, cs.gpus, **kw)


class DevBudgets:
    """cs's run_pdb and allowed on the device (None stays NULL), and the dra_disruption_budgets struct pointing at them"""

    def __init__(self, pkg, cs):
        self.keep = [None if x is None else S.dev(np.asarray(x, d)) for x, d in ((cs.run_pdb, np.uint32),
                                                                                  (cs.allowed, np.int32))]
        self.struct = pkg.api.DisruptionBudgets(S.ptr(self.keep[0]), S.ptr(self.keep[1]), cs.npdb)


def _world(pkg, cs, world, kind=None, bounds=None):
    return S.World(pkg, cs.table, cs.node_off, cs.gpus, world, bounds or S.bounds(cs.n_node, world, kind),
                   n_out_max=max(1, len(cs.run_out)), preempt=(64, 4096, 4096), pairs=4096)


def _sharded_on(pkg, W, cs, asked=None, mv=None, what=""):
    """cs on the world W, every rank against the oracle on the world's state; returns every rank's outputs (None: a
    call-level error, which must fail every rank with nothing written).  The inventories stay as they were."""
    A = pkg.api
    mv = cs.max_victims if mv is None else mv
    run = Running(pkg, cs.run_claims, cs.run_pod_off, cs.run_prio, cs.run_out, out_off=cs.run_out_off)
    bud = DevBudgets(pkg, cs)
    fl = A.F_EXHAUSTIVE if cs.flags else 0
    cands = cs.cand_arrays() if cs.cands is not None else None
    try:
        ref = cs.ref(W.state(), mv=mv)
    except ValueError:
        ref = None
    res = None
    if ref is None:
        try:
            outs = S.preempt(W, cs.claims, cs.pod_off, cs.prio, run, cands, mv, fl, pdb=True, bud=bud,
                             sentinel=SHARD_SENT, expect=A.E_INVAL)
        except A.DraError as e:                          # refused on the host, before anything was enqueued
            assert e.code == A.E_INVAL, what
        else:
            for r, o in enumerate(outs):
                assert all((h == SHARD_SENT).all() for h in o), f"{what}: rank {r} wrote an output"
    else:
        res = S.preempt(W, cs.claims, cs.pod_off, cs.prio, run, cands, mv, fl, pdb=True, bud=bud, sentinel=SHARD_SENT,
                        asked=asked)
        for r, x in enumerate(res):
            S.same(x, ref, NAMES, f"{what} rank {r}")
            assert "preempt_shard" in W.ctxs[r].last_chain(), (what, r)
    for r, c in enumerate(W.ctxs):
        assert c.get_inventory().tobytes() == cs.gpus.tobytes(), f"{what}: rank {r}'s live inventory changed"
    return res


def _sharded(pkg, cs, world, kind, bounds=None, what=""):
    """cs on a fresh world of `world` contexts; returns rank 0's outputs (None: a call-level error).  Afterwards every
    rank's pristine inventory is unchanged too."""
    W = _world(pkg, cs, world, kind, bounds)
    what = f"{what} world {world} {kind if bounds is None else bounds}"
    try:
        res = _sharded_on(pkg, W, cs, what=what)
        for r, c in enumerate(W.ctxs):
            c.reset_inventory()
            assert c.get_inventory().tobytes() == cs.gpus.tobytes(), f"{what}: rank {r}'s pristine inventory changed"
        return None if res is None else res[0]
    finally:
        W.close()


# ---- 1. the hand-written fixtures of test_preempt_pdb.py ------------------------------------------------------------
def _expand(f):
    """f, or one call per parameter set of its parametrize mark"""
    marks = [m for m in getattr(f, "pytestmark", []) if m.name == "parametrize"]
    if not marks:
        return [f]
    names, values = marks[0].args[:2]
    return [functools.partial(f, *(v if "," in names else (v,))) for v in values]


FIXTURES = [TB.test_a_pair_with_violations_loses_to_one_without, TB.test_a_violating_member_is_tried_first_and_stays,
            TB.test_allowed_counts_the_members_in_v_order, TB.test_budget_counts_members_before_the_reprieve,
            TB.test_a_budget_spanning_two_nodes_starts_full_on_each_pair,
            TB.test_members_at_or_above_the_pending_priority_do_not_count,
            TB.test_a_budget_chain_through_none_and_other_budgets,
            TB.test_the_highest_victim_index_is_the_lowest_when_the_violating_phase_goes_first,
            TB.test_the_sum_decides_on_tied_violations_and_violations_beat_the_sum,
            TB.test_violations_beat_a_lower_highest_priority_and_ties_keep_the_later_keys,
            TB.test_the_fewest_violations_past_one_warp, TB.test_call_level_errors]


def _fixture_cases(monkeypatch):
    """every preempt_oracle.preempt_pdb call the fixtures make (each still checks its own answer), rejected ones
    included, as Cases"""
    calls, orig = [], P.preempt_pdb
    sig = inspect.signature(orig)

    def record(*args, **kw):
        b = sig.bind(*args, **kw)
        b.apply_defaults()
        calls.append(dict(b.arguments))
        return orig(*args, **kw)
    monkeypatch.setattr(P, "preempt_pdb", record)
    try:
        for f in FIXTURES:
            for g in _expand(f):
                g()
    finally:
        monkeypatch.undo()
    out = []
    for a in calls:
        co, cn = a["cand_off"], a["cand_nodes"]
        cands = None if co is None else [[int(x) for x in cn[co[p]: co[p + 1]]] for p in range(len(co) - 1)]
        pb = Problem(a["gpus"], np.asarray(a["node_off"], np.uint32), a["table"], a["claims"],
                     np.asarray(a["pod_off"], np.uint32), np.asarray(a["prio"], np.int32), cands, a["run_claims"],
                     np.asarray(a["run_pod_off"], np.uint32), np.asarray(a["run_prio"], np.int32), a["run_out"],
                     a["run_out_off"], a["max_victims"], a["flags"], True, False)
        out.append(case(pb, a["run_pdb"], a["pdb_allowed"], a["n_pdb"]))
    return out


def test_hand_written_fixtures_at_every_lane_width(pkg, bctx, monkeypatch):
    R = pkg.records
    cases = _fixture_cases(monkeypatch)
    assert len(cases) >= 40
    for i, cs in enumerate(cases):
        n_pod, n = len(cs.prio), cs.n_node
        for flags in (0, P.F_EXHAUSTIVE):
            base = _run(pkg, bctx, cs, flags=flags, what=f"fixture {i} f{flags}")
            for width in (9, 17):                          # W = 16, then 32
                got = _run(pkg, bctx, _widen(R, cs, width), flags=flags, what=f"fixture {i} f{flags} +{width}")
                if base is None:
                    assert got is None, (i, flags, width)
                    continue
                for k in (0, 1, 6):
                    x = got[k].reshape(n_pod, n + 1)[:, :n] if cs.cands is None else got[k]
                    assert x.tobytes() == base[k].tobytes(), (i, flags, width, NAMES[k])
                for k in (2, 3, 4, 5, 7):
                    assert got[k].tobytes() == base[k].tobytes(), (i, flags, width, NAMES[k])


def test_sharded_fixtures(pkg, monkeypatch):
    for i, cs in enumerate(_fixture_cases(monkeypatch)):
        for world, kind in ((1, "even"), (2, "even"), (3, "uneven")):
            _sharded(pkg, cs, world, kind, what=f"fixture {i}")


# ---- 2. crowded nodes, long chains, large counts --------------------------------------------------------------------
def _crowded(R, seed, shares, n_crowd=2400, n_node=4, crowd=0, flags=0, mv=64):
    """n_node non-MIG 8-GPU nodes; node `crowd` holds n_crowd time-slicing pods (an equal share on each GPU), the others
    1-3 a GPU, one of them of INT32_MAX.  The crowded node's pods on GPUs 0-6 have priorities -5..2, those on GPU 7
    priorities 3..9: at or above the first and third pending pods' priority 3, and in the same budgets.  Pending: a
    one-GPU pod (frees one of GPUs 0-6), an eight-GPU pod of INT32_MAX (evicts the whole node, and only the crowded node
    lets it) and a two-GPU pod.  shares: [(allowed, share of the pods)] per budget; the rest of the pods have none."""
    rng = np.random.default_rng(seed)
    per = rng.integers(1, 4, 8 * n_node)
    per[8 * crowd: 8 * crowd + 8] = n_crowd // 8
    pb = _shared_world(R, [8] * n_node, per, seed)
    node = np.repeat(np.arange(8 * n_node) // 8, per)
    first = int(per[: 8 * crowd].sum())
    gpu = np.repeat(np.arange(8), n_crowd // 8)
    pb.run_prio[first: first + n_crowd] = np.where(gpu < 7, rng.integers(-5, 3, n_crowd), rng.integers(3, 10, n_crowd))
    pb.run_prio[[int(np.argmax(node == n)) for n in range(n_node) if n != crowd]] = I32_MAX   # only `crowd` for pod 1
    c = np.zeros(3, R.CLAIM_DTYPE)
    c["kind"], c["count"] = R.KIND_GPU, [1, 8, 2]
    n_run = len(pb.run_prio)
    w = np.array([s for _, s in shares] + [max(0.0, 1 - sum(s for _, s in shares))])
    b = rng.choice(len(shares) + 1, n_run, p=w / w.sum())
    run_pdb = np.where(b == len(shares), NONE, b).astype(np.uint32)
    return case(pb, run_pdb, [a for a, _ in shares], claims=c, prio=np.array([3, I32_MAX, 3], np.int32), flags=flags,
                max_victims=mv)


def _node_of_running(cs):
    node = np.full(len(cs.run_prio), NONE, np.int64)
    for r in range(len(cs.run_prio)):
        i = int(cs.run_pod_off[r])
        node[r] = cs.gpus["node"][cs.run_out["gpu"][i]]
    return node


def _walk_bound(cs):
    """the most budget-chain steps one pass over a node's V can take: per node and budget, members × min(allowed,
    members)"""
    node = _node_of_running(cs)
    worst = 0
    for n in np.unique(node):
        tot = 0
        for b, a in enumerate(cs.allowed):
            m = int(((node == n) & (cs.run_pdb == b)).sum())
            tot += m * min(max(int(a), 0), m)
        worst = max(worst, tot)
    return worst


CROWDS = [[(0, 0.9)], [(1023, 0.6), (7, 0.3)], [(255, 0.3), (256, 0.3), (I32_MAX, 0.3)],
          [(1, 0.5), (I32_MAX, 0.2), (255, 0.2)], [(256, 0.45), (0, 0.45)]]


def test_crowded_nodes_long_chains_and_large_counts(pkg, bctx):
    R = pkg.records
    longest, most = 0, 0
    for i, shares in enumerate(CROWDS):
        cs = _crowded(R, i, shares, flags=P.F_EXHAUSTIVE if i % 2 else 0, mv=(64, 3000)[i % 2])
        assert all(a in ALLOWED_EDGES for a, _ in shares)
        assert _walk_bound(cs) <= 10_000_000
        longest = max(longest, int(np.bincount(_node_of_running(cs)).max()))
        got = _run(pkg, bctx, cs, what=f"crowded {shares}")
        assert (got[0].reshape(3, -1)[:, 0] == P.EVICT).all() and got[2][1] == 0, shares
        most = max(most, int(got[6].max()))
        cands = [[0, 1, 0], [2, 0, 3, NONE], [0]]
        _run(pkg, bctx, dataclasses.replace(cs, cands=cands), what=f"crowded {shares} cands")
    assert longest > 256 and most > 1023, (longest, most)


# ---- 3. every bucketing path of the running pods --------------------------------------------------------------------
def _with_budgets(pb, seed, n_pdb, pool):
    rng = np.random.default_rng(seed)
    run_pdb = rng.integers(0, n_pdb + 1, len(pb.run_prio))
    run_pdb[run_pdb == n_pdb] = NONE
    allowed = rng.choice(np.array(pool, np.int64), n_pdb)
    allowed[0] = 0                                       # one budget that allows nothing, so that the budgets bite
    return case(pb, run_pdb, allowed)


def test_bucket_small(pkg, bctx):
    cs = _with_budgets(_shared_world(pkg.records, [8] * 20, np.full(160, 10), 1), 1, 3, ALLOWED_EDGES)
    assert len(cs.run_prio) <= 8192
    got = _run(pkg, bctx, cs, chain=("preempt", "bucket_small"), what="bucket_small")
    assert (got[3] == P.EVICT).any() and got[6].any()


def test_hist8_scan8_with_a_node_of_8800_pods(pkg, bctx):
    per = np.full(8 * 500, 4)
    per[:8] = 1100
    pb = _shared_world(pkg.records, [8] * 500, per, 2)
    pb.run_prio[:8800] = np.arange(8800) % 8 - 5
    assert 8192 < len(pb.run_prio) <= _n_sm() * 2048
    cs = _with_budgets(pb, 2, 3, (0, 1, 7))                # small allowed: at most 7 chain steps per member
    for flags in (0, P.F_EXHAUSTIVE):
        got = _run(pkg, bctx, cs, flags=flags, chain=("preempt", "hist8", "scan8", "scatter"), what=f"hist8 f{flags}")
        assert got[1][0] > 1000 and got[6][0] > 0


def test_hist8_multi(pkg, bctx):
    n_gpu = 2000 * 8
    per = np.full(n_gpu, (_n_sm() * 2048 + 8000) // n_gpu + 1)
    pb = _shared_world(pkg.records, [8] * 2000, per, 3, n_cand=24)
    assert len(pb.run_prio) > _n_sm() * 2048
    cs = _with_budgets(pb, 3, 4096, ALLOWED_EDGES)
    got = _run(pkg, bctx, cs, chain=("preempt", "hist8_multi", "scatter"), what="hist8_multi")
    assert (got[0] == P.EVICT).any() and got[6].any()


def test_scan_rows_and_the_grid_stride_of_the_victim_sort(pkg, bctx):
    n_node = 12000
    assert n_node > _n_sm() * 8
    cs = _with_budgets(_shared_world(pkg.records, [1] * n_node, np.full(n_node, 8), 4), 4, 64, ALLOWED_EDGES)
    got = _run(pkg, bctx, cs, chain=("preempt", "hist8", "scan_rows", "scatter"), what="scan_rows")
    assert (got[0] == P.EVICT).sum() > 100 and got[6].any()


def test_hist_warp_and_scan(pkg, bctx):
    n_node = 20000
    per = np.random.default_rng(5).integers(0, 2, n_node)
    cs = _with_budgets(_shared_world(pkg.records, [1] * n_node, per, 5), 5, 2, (0, 0, 1))
    assert len(cs.run_prio) > 8192
    got = _run(pkg, bctx, cs, chain=("preempt", "hist_warp", "scan", "scatter"), what="hist_warp")
    assert (got[0] == P.EVICT).any() and got[6].any()


# ---- 4. random problems ---------------------------------------------------------------------------------------------
def _random_case(x):
    pb, run_pdb, allowed = x
    return case(pb, run_pdb, allowed)


def test_random_problems(pkg, bctx):
    @settings(max_examples=N_EX or 120, deadline=None, suppress_health_check=list(HealthCheck), derandomize=N_EX == 0,
              database=None)
    @given(TB.pdb_problems())
    def run(x):
        cs = _random_case(x)
        _run(pkg, bctx, cs, what=cs.what)
    run()


def test_sharded_random_problems(pkg):
    @settings(max_examples=N_EX or 40, deadline=None, suppress_health_check=list(HealthCheck), derandomize=N_EX == 0,
              database=None)
    @given(TB.pdb_problems(), st.sampled_from(CONFIGS))
    def run(x, cfg):
        cs = _random_case(x)
        _sharded(pkg, cs, *cfg, what=cs.what)
    run()


# ---- 5. sharded packing and ownership -------------------------------------------------------------------------------
SHARD_CONFIGS = CONFIGS + [(4, "even"), (4, "uneven"), (4, "empty")]


def test_sharded_crowded_node_on_each_rank(pkg):
    for crowd in range(4):
        cs = _crowded(pkg.records, 10 + crowd, [(0, 0.45), (7, 0.45)], crowd=crowd, mv=3000)
        got = _sharded(pkg, cs, 4, "even", what=f"crowded on rank {crowd}")
        assert got[7][1] > 1023 and got[2][1] == crowd and got[4][1] == 2400


def _limit_and_count(R, k):
    """Node 0, one GPU: test_preempt.test_search_limit's shape — a 1g pod of priority 0 at slice 0 keeps 7 x 1g + 7g out,
    and with it removed the exhaustive search runs out of budget.  Node 1, two GPUs: seven 1g pods and one 7g pod of
    priority 1; the pending pod fits only with all eight gone, k of them under a budget that allows nothing.  Node 2: a
    7g pod of priority 20 (NO)."""
    g, off = R.make_inventory([1, 2, 1], mig=True)
    pods = [(0, 0, 1, R.GI_1_SLICE, 0)] + [(1, s, 1, R.GI_1_SLICE, 1) for s in range(7)] + \
        [(2, 0, 8, R.GI_7_SLICE, 1), (3, 0, 8, R.GI_7_SLICE, 20)]
    rc, rpo, rpr, ro = TB.mig_running(pods, off)
    g = TB.occupied(g, rc, ro)
    c = TB._mig(R, [R.GI_1_SLICE] * 7 + [R.GI_7_SLICE])
    pb = Problem(g, off, R.default_table(), c, np.array([0, 8], np.uint32), np.array([5], np.int32), None, rc, rpo, rpr,
                 ro, None, 16, P.F_EXHAUSTIVE, True, False)
    return case(pb, [NONE] + [0] * k + [NONE] * (8 - k) + [NONE], [0])


def test_a_partial_with_the_limit_bit_and_a_violation_count(pkg):
    """rank 0 holds nodes 0 and 1: its partial carries SEARCH_LIMIT in bit 0 and the EVICT pair's violations above it,
    odd and even"""
    for k in (3, 4):
        cs = _limit_and_count(pkg.records, k)
        ref = cs.ref()
        assert list(ref[0]) == [P.SEARCH_LIMIT, P.EVICT, P.NO] and list(ref[6]) == [0, k, 0]
        assert list(ref[3]) == [P.EVICT] and list(ref[7]) == [k] and list(ref[4]) == [8]
        for world, bounds in ((1, None), (2, [0, 2, 3]), (3, [0, 2, 2, 3]), (3, [0, 2, 3, 3])):
            _sharded(pkg, cs, world, "even", bounds=bounds, what=f"limit and {k} violations")
        for world, kind in SHARD_CONFIGS:
            _sharded(pkg, cs, world, kind, what=f"limit and {k} violations")


def test_the_violation_key_across_ranks(pkg):
    """The fewest-violation pair on one rank, a lower-priority one on the other, in both orders; the 64-bit-sum shape
    with tied and deciding violations on two ranks; the two-warp candidate lists on every world"""
    R = pkg.records
    g, off, t, rc, rpo, rpr, ro = TB.warp_world()
    c = TB._mig(R, [R.GI_7_SLICE])

    def warp(cands, budgets, mv=2):
        pb = Problem(g, off, t, c if len(cands) == 1 else TB._mig(R, [R.GI_7_SLICE] * 2),
                     np.arange(len(cands) + 1, dtype=np.uint32), np.full(len(cands), 100, np.int32), cands, rc, rpo, rpr,
                     ro, None, mv, 0, True, False)
        return case(pb, *budgets)
    for cands, bounds in (([[0, 1]], [0, 1, 3]), ([[1, 0]], [0, 1, 3]), ([[2, 1]], [0, 2, 3]), ([[1, 2]], [0, 2, 3])):
        got = _sharded(pkg, warp(cands, TB.WARP_OVER), 2, "even", bounds=bounds, what=f"violations {cands}")
        assert list(got[2]) == [1] and list(got[7]) == [0]
    for world, kind in SHARD_CONFIGS:
        for budgets in (TB.WARP_OVER, TB.WARP_TIE):
            _sharded(pkg, warp(TB.warp_cands(), budgets), world, kind, what=f"two warps {budgets}")
    for a_first in (True, False):
        g2, off2, t2, rc2, rpo2, rpr2, ro2, nb = TB.sum_world(a_first)
        for cands in (None, [[0, 1]], [[1, 0]]):
            pb = Problem(g2, off2, t2, c, np.array([0, 1], np.uint32), np.array([11], np.int32), cands, rc2, rpo2, rpr2,
                         ro2, None, 4, 0, True, False)
            for budgets, node in ((([0, NONE, 0, NONE], [0]), nb), (([NONE, NONE, 0, 0], [1]), 1 - nb)):
                got = _sharded(pkg, case(pb, *budgets), 2, "even", bounds=[0, 1, 2], what=f"sum {a_first} {cands}")
                assert list(got[2]) == [node]


def test_the_chosen_node_on_the_last_rank_behind_an_empty_window(pkg):
    """Node 0 (rank 0): one 7g pod of priority 1 under a budget that allows nothing; node 1 (the last rank): two 3g pods
    of priority 5.  The clean pair on node 1 wins; its victim row is its owner's, past a rank that owns no node."""
    R = pkg.records
    g, off = R.make_inventory([1, 1], mig=True)
    rc, rpo, rpr, ro = TB.mig_running([(0, 0, 8, R.GI_7_SLICE, 1), (1, 0, 4, R.GI_3_SLICE, 5),
                                       (1, 4, 4, R.GI_3_SLICE, 5)], off)
    g = TB.occupied(g, rc, ro)
    for mv in (1, 2, 5):
        pb = Problem(g, off, R.default_table(), TB._mig(R, [R.GI_7_SLICE]), np.array([0, 1], np.uint32),
                     np.array([10], np.int32), None, rc, rpo, rpr, ro, None, mv, 0, True, False)
        cs = case(pb, [0, NONE, NONE], [0])
        for bounds in ([0, 1, 1, 2], [0, 1, 1, 1, 2], [0, 0, 1, 1, 2]):
            got = _sharded(pkg, cs, len(bounds) - 1, "even", bounds=bounds, what=f"empty window mv{mv}")
            assert list(got[2]) == [1] and list(got[5][0][:2]) == [1, 2][:mv]


# ---- 6. optional outputs --------------------------------------------------------------------------------------------
def _masks():
    return [tuple(bool(m >> i & 1) for i in range(4)) for m in range(16)]


def _synth_case(pkg, seed, cands_k=None, mv=8):
    from test_gpu_preempt_pdb import budgets
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=30, seed=seed)
    rng = np.random.default_rng(seed)
    run_pdb, allowed = budgets(rng, len(w.run_prio), 3)
    cands = None
    if cands_k:
        nodes = rng.integers(0, 14, (len(w.prio), cands_k))
        cands = [[int(x) for x in row] for row in nodes]
    pb = Problem(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, cands, w.run_claims, w.run_pod_off, w.run_prio,
                 w.run_out, None, mv, 0, True, False)
    return case(pb, run_pdb, allowed)


def test_every_combination_of_the_optional_outputs(pkg, bctx):
    for seed, k in ((21, None), (22, 6)):
        cs = _synth_case(pkg, seed, k)
        _load(bctx, cs)
        full = _call(pkg, bctx, cs, cs.gpus, what=f"masks {seed} full")
        assert full[6].any()
        for asked in _masks():
            _call(pkg, bctx, cs, cs.gpus, asked=asked, what=f"masks {seed} {asked}")


def test_sharded_optional_outputs(pkg):
    for seed, k, world, kind in ((23, None, 3, "uneven"), (24, 5, 2, "even")):
        cs = _synth_case(pkg, seed, k)
        W = _world(pkg, cs, world, kind)
        try:
            for asked in _masks():
                full = [asked[0], asked[1], True, True, True, True, asked[2], asked[3]]
                res = _sharded_on(pkg, W, cs, asked=full, what=f"sharded masks {seed} {asked}")
                if asked == (False, False, True, False):          # only pair_violations
                    assert res[0][6].any() and res[0][0] is None and res[0][7] is None
        finally:
            W.close()


# ---- 7. one context, sizes growing and shrinking, shared buffers in between -----------------------------------------
def test_context_reuse(pkg):
    A, R = pkg.api, pkg.records
    ctx = A.Context(device=0)
    try:
        steps = ((1, 0, 8), (4, 4096, 64), (16, 1, 3), (2, 4096, 0), (16, 0, 64), (1, 1, 1), (8, 4096, 64), (1, 0, 3))
        for it, (scale, n_pdb, mv) in enumerate(steps):
            pb = dataclasses.replace(_pick(scale, it % 2 == 0, 2000 * it), max_victims=mv)
            rng = np.random.default_rng(it)
            n_run = len(pb.run_prio)
            if n_pdb:
                run_pdb = rng.integers(0, n_pdb + 1, n_run)
                run_pdb[run_pdb == n_pdb] = NONE
                cs = case(pb, run_pdb, rng.choice(np.array(TB.ALLOWED + ALLOWED_EDGES, np.int64), n_pdb))
            else:
                cs = case(pb, np.full(n_run, NONE, np.uint32), [])      # n_pdb = 0 with a run_pdb of all NONE
            what = f"reuse {it} scale {scale} n_pdb {n_pdb}"
            _load(ctx, cs)
            _call(pkg, ctx, cs, cs.gpus, what=what)
            live = ctx.get_inventory()
            cn, co = cs.cand_arrays()
            fl = A.F_EXHAUSTIVE if cs.flags else 0
            # budget-free preemption on the same buffers
            got = ctx.preempt(cs.claims, cs.pod_off, cs.prio, cs.run_claims, cs.run_pod_off, cs.run_prio, cs.run_out,
                              cs.run_out_off, cn, co, 4, fl)
            ref = P.preempt(live, cs.node_off, cs.table, cs.claims, cs.pod_off, cs.prio, cs.run_claims, cs.run_pod_off,
                            cs.run_prio, cs.run_out, cs.run_out_off, cn, co, 4, cs.flags)
            assert all(x.tobytes() == y.tobytes() for x, y in zip(got, ref)), what + " preempt"
            # pod capacity
            ref = CO.capacity(live, cs.node_off, cs.table, cs.claims, cs.pod_off, cn, co, 5, cs.flags)
            got = ctx.pod_capacity(cs.claims, cs.pod_off, cn, co, 5, bool(cs.flags))
            assert all(x.tobytes() == y.tobytes() for x, y in zip(got, ref)), what + " capacity"
            _call(pkg, ctx, cs, cs.gpus, mv=(3, 64)[it % 2], what=what + " after capacity")
            # preempt and place, which grows the same running-pod buffers and takes the live inventory on
            placed = cs.claims.copy()
            placed["node"] = 0
            sl = R.claim_slots(placed, 1).astype(np.int64)
            oo = np.concatenate([[0], np.cumsum(sl)[:-1]]).astype(np.uint32) if len(sl) else np.zeros(0, np.uint32)
            out, node, pst, ev = ctx.preempt_place(cs.claims, cs.pod_off, cs.prio, cs.run_claims, cs.run_pod_off,
                                                   cs.run_prio, cs.run_out, cs.run_out_off, cn, co, oo, int(sl.sum()), fl)
            ref = PP.preempt_place(live, cs.node_off, cs.table, cs.claims, cs.pod_off, cs.prio, cs.run_claims,
                                   cs.run_pod_off, cs.run_prio, cs.run_out, cs.run_out_off, cn, co, oo, int(sl.sum()),
                                   cs.flags)
            for x, y in zip((out, node, pst, ev), ref):
                assert x.tobytes() == y.tobytes(), what + " preempt_place"
            assert ctx.get_inventory().tobytes() == ref[4].tobytes(), what + " preempt_place inventory"
            # budgets again, on the inventory preempt and place left
            _call(pkg, ctx, cs, cs.gpus, mv=(64, 3)[it % 2], what=what + " after preempt_place")
    finally:
        ctx.close()


# ---- 8. limits and argument edges -----------------------------------------------------------------------------------
def _one_pod(R):
    g, off = R.make_inventory([1, 1], mig=True)
    rc, rpo, rpr, ro = TB.mig_running([(0, 0, 8, R.GI_7_SLICE, 1), (1, 0, 8, R.GI_7_SLICE, 1)], off)
    g = TB.occupied(g, rc, ro)
    return Problem(g, off, R.default_table(), TB._mig(R, [R.GI_7_SLICE]), np.array([0, 1], np.uint32),
                   np.array([10], np.int32), None, rc, rpo, rpr, ro, None, 4, 0, True, False)


def test_budgets_with_the_most_running_pods_fail(pkg, bctx):
    """n_pdb > 0 with DRA_PDB_MAX_RUNNING running pods: E_INVAL before anything is read or written.  The running arrays
    are zero pages the kernel hands out lazily; only a call that failed to refuse would touch them."""
    A = pkg.api
    pb = _one_pod(pkg.records)
    _load(bctx, pb)
    rpo = np.zeros(PDB_MAX_RUNNING + 1, np.uint32)
    rpr = np.zeros(PDB_MAX_RUNNING, np.int32)
    rp = np.zeros(PDB_MAX_RUNNING, np.uint32)
    cs = case(pb, None, [0])
    cs.run_pdb = rp
    run = A.RunningPods(None, 0, rpo.ctypes.data, PDB_MAX_RUNNING, rpr.ctypes.data, None, None, 0)
    n0 = bctx.launch_count()
    rc_, outs = _raw(pkg, bctx, cs, 0, 4, run=run)
    assert rc_ == A.E_INVAL
    assert all((o.view(np.uint8) == SENT).all() for o in outs)
    assert bctx.launch_count() == n0 and bctx.get_inventory().tobytes() == pb.gpus.tobytes()
    # the next call works
    _call(pkg, bctx, case(pb, [0, NONE], [0]), pb.gpus, what="after the limit")


def test_no_pending_pods_leave_run_pdb_unexamined(pkg, bctx):
    R = pkg.records
    pb = _one_pod(R)
    empty = dataclasses.replace(pb, claims=pb.claims[:0], pod_off=np.array([0], np.uint32), prio=np.zeros(0, np.int32))
    for run_pdb in ([7, 7], [1, NONE], [NONE, 0xFFFFFFFE]):
        cs = case(empty, run_pdb, [0])
        got = _run(pkg, bctx, cs, what=f"no pods {run_pdb}")
        assert all(x.size == 0 for x in got)
        for world, kind in ((1, "even"), (2, "even")):
            _sharded(pkg, cs, world, kind, what=f"no pods {run_pdb}")


def test_no_running_pods_need_no_run_pdb(pkg, bctx):
    R = pkg.records
    pb = _one_pod(R)
    free = dataclasses.replace(pb, run_claims=pb.run_claims[:0], run_pod_off=np.zeros(1, np.uint32),
                               run_prio=np.zeros(0, np.int32), run_out=pb.run_out[:0], gpus=R.make_inventory([1, 1])[0])
    for allowed in ([0], [0, -1, 5]):
        cs = case(free, None, allowed)
        got = _run(pkg, bctx, cs, what=f"no running pods {allowed}")
        assert list(got[3]) == [P.FITS]
        for world, kind in ((1, "even"), (2, "even")):
            _sharded(pkg, cs, world, kind, what=f"no running pods {allowed}")


def test_the_wrapper_checks_the_length_of_run_pdb(pkg, bctx):
    """Context.preempt_pdb raises ValueError, before anything is enqueued, for a run_pdb that does not hold one entry
    per running pod (the library would read one per running pod past its end)"""
    w = pkg.synth.preempt(n_node=8, gpus_per_node=8, n_pending=20, seed=31)
    _load(bctx, w)
    n_run = len(w.run_prio)
    args = (w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out)
    n0 = bctx.launch_count()
    for n in (0, 1, n_run - 1, n_run + 1):
        with pytest.raises(ValueError):
            bctx.preempt_pdb(*args, np.zeros(n, np.uint32), np.array([1], np.int32))
    assert bctx.launch_count() == n0
    got = bctx.preempt_pdb(*args, np.zeros(n_run, np.uint32), np.array([1], np.int32))
    ref = P.preempt_pdb(bctx.get_inventory(), w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims,
                        w.run_pod_off, w.run_prio, w.run_out, np.zeros(n_run, np.uint32), [1])
    assert all(x.tobytes() == y.tobytes() for x, y in zip(got, ref))
