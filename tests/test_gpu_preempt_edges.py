"""GPU suite: preemption (spec §14) at its edges, on one inventory (dra_preempt_batch) and on a sharded world of one device
(dra_preempt_batch_global_device).  Every call's six outputs are compared byte for byte with preempt_oracle.preempt on the
same inventory, nothing may be written past an output, and no inventory word may change, live or pristine.

* the hand-written §14 fixtures of test_preempt.py, also with an unused 9- and 17-GPU node appended (lane widths 16, 32)
* the 64-bit priority sum, and choices whose best pair sits past the first warp of a pod's candidates
* random problems (tests/preempt_problems.py): mismatched records, run_out_off, priorities at the int32 ends
* every bucketing path the running pods can take, asserted by the kernel chain
* one context reused by calls that grow and shrink every size, interleaved with the calls sharing its buffers"""
import dataclasses
import functools
import inspect
import os
from types import SimpleNamespace

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

import preempt_oracle as P
import test_preempt as T
from preempt_problems import I32_MAX, I32_MIN, NONE, Problem, problems, random_problem
from test_gpu_preempt import _raw
from test_gpu_shard_preempt import Running, World, _same
from test_gpu_shard_unsuitable import _bounds
from test_pod_mode import _mig
from test_preempt import mig_running, occupied

pytestmark = pytest.mark.gpu
SENT, SLACK = 0xA5, 16
NAMES = ("pair_status", "pair_victims", "pod_node", "pod_status", "n_victims", "victims")
N_EX = int(os.environ.get("DRA_PROP_EXAMPLES", "0"))      # > 0: that many RANDOM examples instead of the fixed ones


@pytest.fixture(scope="module")
def ectx(pkg):
    c = pkg.api.Context(device=0)
    yield c
    c.close()


def _load(ctx, pb):
    ctx.set_table(pb.table)
    ctx.set_inventory(pb.gpus, pb.node_off)


def _call(pkg, ctx, pb, pristine, flags=None, mv=None, chain=("preempt",), what=""):
    """dra_preempt_batch on pb against the oracle on the context's live inventory.  Afterwards the live inventory is
    unchanged and, reset, equals `pristine`.  Returns the outputs, or None when the call must fail (E_INVAL, nothing
    written)."""
    A = pkg.api
    flags = pb.flags if flags is None else flags
    mv = pb.max_victims if mv is None else mv
    before = ctx.get_inventory()
    cn, co = pb.cand_arrays()
    a = dict(c=pb.claims, po=pb.pod_off, prio=pb.prio, rc=pb.run_claims, rpo=pb.run_pod_off, rpr=pb.run_prio,
             ro=pb.run_out, roo=pb.run_out_off, cn=cn, co=co, mv=mv, fl=A.F_EXHAUSTIVE if flags else 0)
    rc_, outs = _raw(pkg, ctx, before, a, SENT, SLACK)
    try:
        ref = pb.oracle(before, flags, mv)
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
        for name, o, y in zip(NAMES, outs, ref):
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


def _run(pkg, ctx, pb, **kw):
    _load(ctx, pb)
    return _call(pkg, ctx, pb, pb.gpus, **kw)


# ---- 1. the hand-written fixtures of test_preempt.py ----------------------------------------------------------------
FIXTURES = [T.test_seven_slivers_four_victims, T.test_equal_priority_never_evicts,
            *[functools.partial(T.test_tie_breaks, w) for w in ("highest", "sum", "count", "latest")],
            T.test_tie_break_position, T.test_int32_extremes, T.test_exhaustive_only, T.test_search_limit,
            T.test_max_victims_shorter_than_the_count, T.test_invalid_and_empty_pods]


def _fixture_problems(monkeypatch):
    """every preempt_oracle.preempt call the fixtures make (each still checks its own answer), as Problems"""
    calls, orig = [], P.preempt
    sig = inspect.signature(orig)

    def record(*args, **kw):
        res = orig(*args, **kw)
        b = sig.bind(*args, **kw)
        b.apply_defaults()
        calls.append(dict(b.arguments))
        return res
    monkeypatch.setattr(P, "preempt", record)
    try:
        for f in FIXTURES:
            f()
    finally:
        monkeypatch.undo()
    out = []
    for a in calls:
        co, cn = a["cand_off"], a["cand_nodes"]
        cands = None if co is None else [[int(x) for x in cn[co[p]: co[p + 1]]] for p in range(len(co) - 1)]
        out.append(Problem(a["gpus"], np.asarray(a["node_off"], np.uint32), a["table"], a["claims"],
                           np.asarray(a["pod_off"], np.uint32), np.asarray(a["prio"], np.int32), cands, a["run_claims"],
                           np.asarray(a["run_pod_off"], np.uint32), np.asarray(a["run_prio"], np.int32), a["run_out"],
                           a["run_out_off"], a["max_victims"], a["flags"], True, False))
    return out


def _widen(R, pb, width):
    """pb with one more node of `width` UNAVAILABLE GPUs: no pod fits there and no running pod is on it"""
    extra = np.zeros(width, R.GPU_DTYPE)
    extra["flags"], extra["node"], extra["mem_free_mib"] = R.GPU_MIG_ENABLED | R.GPU_UNAVAILABLE, pb.n_node, 40960
    return dataclasses.replace(pb, gpus=np.concatenate([pb.gpus, extra]),
                               node_off=np.append(pb.node_off, pb.node_off[-1] + width).astype(np.uint32))


def test_hand_written_fixtures_at_every_lane_width(pkg, ectx, monkeypatch):
    R = pkg.records
    pbs = _fixture_problems(monkeypatch)
    assert len(pbs) >= 20
    for i, pb in enumerate(pbs):
        n_pod, n = len(pb.prio), pb.n_node
        for flags in (0, P.F_EXHAUSTIVE):
            base = _run(pkg, ectx, pb, flags=flags, what=f"fixture {i} f{flags}")
            for width in (9, 17):                          # W = 16, then 32
                got = _run(pkg, ectx, _widen(R, pb, width), flags=flags, what=f"fixture {i} f{flags} +{width}")
                for k in (0, 1):
                    x = got[k].reshape(n_pod, n + 1)[:, :n] if pb.cands is None else got[k]
                    assert x.tobytes() == base[k].tobytes(), (i, flags, width, NAMES[k])
                for k in range(2, 6):
                    assert got[k].tobytes() == base[k].tobytes(), (i, flags, width, NAMES[k])


# ---- 2. the 64-bit priority sum -------------------------------------------------------------------------------------
def _sum_world(R, a_first):
    """Two one-GPU nodes, each held by two 3g pods; A's priorities {10, -9}, B's {10, -11}.  A 7g pod of priority 11
    must evict both pods of either node: the same highest priority and count, Σ(prio + 2^31) = 2^32 + 1 on A and
    2^32 - 1 on B, so B wins (on 32 bits A would).  Returns (problem, B's node, B's running pods in V order)."""
    g, off = R.make_inventory([1, 1], mig=True)
    na, nb = (0, 1) if a_first else (1, 0)
    pods = [(na, 0, 4, R.GI_3_SLICE, 10), (na, 4, 4, R.GI_3_SLICE, -9), (nb, 0, 4, R.GI_3_SLICE, 10),
            (nb, 4, 4, R.GI_3_SLICE, -11)]
    rc, rpo, rpr, ro = mig_running(pods, off)
    g = occupied(g, rc, ro)
    pb = Problem(g, off, R.default_table(), _mig(R, [R.GI_7_SLICE]), np.array([0, 1], np.uint32),
                 np.array([11], np.int32), None, rc, rpo, rpr, ro, None, 4, 0, True, False)
    return pb, nb, [2, 3]


def test_priority_sum_is_64_bit(pkg, ectx):
    for a_first in (True, False):
        for cands in (None, [[0, 1]], [[1, 0]]):
            pb, nb, vic = _sum_world(pkg.records, a_first)
            pb = dataclasses.replace(pb, cands=cands)
            for flags in (0, P.F_EXHAUSTIVE):
                st_, pv, node, pst, nv, row = _run(pkg, ectx, pb, flags=flags, what=f"sum {a_first} {cands}")
                assert list(st_) == [P.EVICT, P.EVICT] and list(pv) == [2, 2]
                assert list(node) == [nb] and list(pst) == [P.EVICT] and list(nv) == [2]
                assert list(row[0]) == vic + [NONE, NONE]


# ---- 3. choices past one warp ---------------------------------------------------------------------------------------
def _warp_world(R):
    """Three one-GPU nodes, each held by one 7g pod: running pod 0 on node 2 (priority 5), 1 on node 1 (priority 6), 2 on
    node 0 (priority 5).  For a 7g pod every pair is EVICT with one victim; node 0 beats node 2 on the latest index of
    the highest-priority victim, and both beat node 1 on the highest priority."""
    g, off = R.make_inventory([1, 1, 1], mig=True)
    rc, rpo, rpr, ro = mig_running([(2, 0, 8, R.GI_7_SLICE, 5), (1, 0, 8, R.GI_7_SLICE, 6), (0, 0, 8, R.GI_7_SLICE, 5)],
                                   off)
    return occupied(g, rc, ro), off, rc, rpo, rpr, ro


def test_choice_past_one_warp(pkg, ectx):
    R = pkg.records
    g, off, rc, rpo, rpr, ro = _warp_world(R)
    stray = [3, 4, NONE]
    # pod 0: node 0 at positions 5, 6, 37 and 69 (all tie), node 2 before it and on other lanes, node 1 and strays around
    a = [stray[k % 3] if k % 4 else 1 for k in range(70)]
    for k in (0, 2, 33, 36, 64):
        a[k] = 2
    for k in (5, 6, 37, 69):
        a[k] = 0
    # pod 1: its best pair at position 63 (lane 31's second), a tying one at 64 (lane 0's third); node 2 on every lane
    b = [2 if k % 3 == 0 else 1 if k % 3 == 1 else stray[k % 2] for k in range(70)]
    b[63], b[64] = 0, 0
    c = _mig(R, [R.GI_7_SLICE, R.GI_7_SLICE])
    pb = Problem(g, off, R.default_table(), c, np.array([0, 1, 2], np.uint32), np.array([100, 100], np.int32), [a, b],
                 rc, rpo, rpr, ro, None, 2, 0, True, False)
    for flags in (0, P.F_EXHAUSTIVE):
        st_, pv, node, pst, nv, row = _run(pkg, ectx, pb, flags=flags, what="past one warp")
        assert list(node) == [0, 0] and list(pst) == [P.EVICT, P.EVICT] and list(nv) == [1, 1]
        assert [list(r) for r in row] == [[2, NONE], [2, NONE]]


# ---- 4. random problems ---------------------------------------------------------------------------------------------
def test_random_problems(pkg, ectx):
    @settings(max_examples=N_EX or 120, deadline=None, suppress_health_check=list(HealthCheck), derandomize=N_EX == 0,
              database=None)
    @given(problems())
    def run(pb):
        _run(pkg, ectx, pb, what=pb.what)
    run()


# ---- 5. every bucketing path of the running pods --------------------------------------------------------------------
def _shared_world(R, widths, per_gpu, seed, n_cand=None):
    """Non-MIG nodes; per_gpu[i] time-slicing pods on GPU i (one claim each, in GPU order), priorities -5..5 and now and
    then INT32_MAX.  Pending: a one-GPU pod of priority 3, a two-GPU pod of INT32_MAX, a time-slicing pod of INT32_MIN.
    n_cand: that many random candidates per pod (strays included) instead of the dense form."""
    rng = np.random.default_rng(seed)
    g, off = R.make_inventory(widths, mig=False)
    per_gpu = np.asarray(per_gpu, np.int64)
    gpu = np.repeat(np.arange(len(g)), per_gpu)
    n = len(gpu)
    rc = np.zeros(n, R.CLAIM_DTYPE)
    rc["kind"], rc["count"], rc["node"] = R.KIND_SHARED, 1, g["node"][gpu]
    ro = np.zeros(n, R.OUT_DTYPE)
    ro["gpu"], ro["profile"], ro["status"] = gpu, R.PROFILE_SHARED, R.ST_OK
    assert per_gpu.max(initial=0) < 0xFFFF
    g["share_cnt"] = per_gpu
    rpr = rng.integers(-5, 6, n).astype(np.int32)
    rpr[rng.integers(0, 50, n) == 0] = I32_MAX
    c = np.zeros(3, R.CLAIM_DTYPE)
    c["kind"], c["count"] = [R.KIND_GPU, R.KIND_GPU, R.KIND_SHARED], [1, 2, 1]
    n_node = len(widths)
    cands = None
    if n_cand:
        cands = [[int(x) for x in rng.integers(0, n_node + 2, n_cand)] for _ in range(3)]
    return Problem(g, off, R.default_table(), c, np.array([0, 1, 2, 3], np.uint32),
                   np.array([3, I32_MAX, I32_MIN], np.int32), cands, rc, np.arange(n + 1, dtype=np.uint32), rpr, ro,
                   None, 64, 0, True, False)


def _n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_bucket_small(pkg, ectx):
    pb = _shared_world(pkg.records, [8] * 20, np.full(160, 10), 1)
    assert len(pb.run_prio) <= 8192
    got = _run(pkg, ectx, pb, chain=("preempt", "bucket_small"), what="bucket_small")
    assert (got[3] == P.EVICT).any()


def test_hist8_scan8_with_a_node_of_8800_pods(pkg, ectx):
    per = np.full(8 * 500, 4)
    per[:8] = 1100                                        # node 0: 8,800 pods, so the histogram rows run full on it
    pb = _shared_world(pkg.records, [8] * 500, per, 2)
    pb.run_prio[:8800] = np.arange(8800) % 8 - 5           # all below the first pending pod's priority
    assert 8192 < len(pb.run_prio) <= _n_sm() * 2048
    for flags in (0, P.F_EXHAUSTIVE):
        got = _run(pkg, ectx, pb, flags=flags, chain=("preempt", "hist8", "scan8", "scatter"), what=f"hist8 f{flags}")
        assert got[1][0] > 1000                            # the first pod's pair on node 0: a long reprieve


def test_hist8_multi(pkg, ectx):
    n_gpu = 2000 * 8
    per = np.full(n_gpu, (_n_sm() * 2048 + 8000) // n_gpu + 1)
    pb = _shared_world(pkg.records, [8] * 2000, per, 3, n_cand=24)
    assert len(pb.run_prio) > _n_sm() * 2048
    got = _run(pkg, ectx, pb, chain=("preempt", "hist8_multi", "scatter"), what="hist8_multi")
    assert (got[0] == P.EVICT).any()


def test_scan_rows_and_the_grid_stride_of_the_victim_sort(pkg, ectx):
    n_node = 12000
    assert n_node > _n_sm() * 8
    pb = _shared_world(pkg.records, [1] * n_node, np.full(n_node, 8), 4)
    got = _run(pkg, ectx, pb, chain=("preempt", "hist8", "scan_rows", "scatter"), what="scan_rows")
    assert (got[0] == P.EVICT).sum() > 100


def test_hist_warp_and_scan(pkg, ectx):
    n_node = 20000
    per = np.random.default_rng(5).integers(0, 2, n_node)
    pb = _shared_world(pkg.records, [1] * n_node, per, 5)
    assert len(pb.run_prio) > 8192
    got = _run(pkg, ectx, pb, chain=("preempt", "hist_warp", "scan", "scatter"), what="hist_warp")
    assert (got[0] == P.EVICT).any()


def test_no_running_pods(pkg, ectx):
    pb = _shared_world(pkg.records, [8, 3, 0, 8], np.zeros(19, np.int64), 6)
    assert len(pb.run_prio) == 0
    for cands in (None, [[0, 1, 5], [], [2, 3]]):
        got = _run(pkg, ectx, dataclasses.replace(pb, cands=cands), what="no running pods")
        assert not (got[3] == P.EVICT).any()


# ---- 6. one context, sizes growing and shrinking, shared buffers in between -----------------------------------------
def _pick(scale, want_off, start):
    """the first valid random problem from seed `start` on with (or without) run_out_off"""
    s = start
    while True:
        pb = random_problem(s, scale)
        if (pb.run_out_off is not None) == want_off and not pb.error and len(pb.prio):
            return pb
        s += 1


def test_context_reuse(pkg, oracle):
    import place_oracle
    R, A = pkg.records, pkg.api
    ctx = A.Context(device=0)
    try:
        for it, scale in enumerate((1, 4, 16, 2, 16, 1, 8, 1)):
            pb = _pick(scale, it % 2 == 0, 1000 * it)
            pb = dataclasses.replace(pb, max_victims=(64, 0, 3, 64, 1, 64, 0, 3)[it])
            what = f"reuse {it} scale {scale}"
            _load(ctx, pb)
            _call(pkg, ctx, pb, pb.gpus, what=what)
            # the running claims through Allocate, which takes the live inventory on
            oo, n_out = R.out_offsets(pb.run_claims, pb.n_node)
            out = ctx.allocate(pb.run_claims, oo, n_out)
            ref, live = oracle.allocate(pb.gpus, pb.node_off, pb.table, pb.run_claims, oo, n_out)
            assert out.tobytes() == ref.tobytes() and ctx.get_inventory().tobytes() == live.tobytes(), what
            _call(pkg, ctx, dataclasses.replace(pb, flags=P.F_EXHAUSTIVE - pb.flags), pb.gpus, what=what + " after")
            # UnsuitableNodes and place pods on the pending pods
            cn, co = pb.cand_arrays()
            if cn is None:
                n_pod = len(pb.prio)
                cn = np.tile(np.arange(pb.n_node, dtype=np.uint32), n_pod)
                co = (np.arange(n_pod + 1) * pb.n_node).astype(np.uint32)
            bits = ctx.unsuitable(pb.claims, pb.pod_off, cn, co, flags=pb.flags)
            assert bits.tobytes() == oracle.unsuitable(pb.gpus, pb.node_off, pb.table, pb.claims, pb.pod_off, cn, co,
                                                       flags=pb.flags).tobytes(), what
            placed = pb.claims.copy()                    # slots as if every claim named a node
            placed["node"] = 0
            po, n_po = R.out_offsets(placed, 1)
            out, node = ctx.place_pods(pb.claims, pb.pod_off, cn, co, po, n_po, flags=pb.flags)
            ref, rnode, after = place_oracle.place_pods(pb.gpus, pb.node_off, pb.table, pb.claims, pb.pod_off, cn, co,
                                                        po, n_po, flags=pb.flags)
            assert out.tobytes() == ref.tobytes() and node.tobytes() == rnode.tobytes(), what
            assert ctx.get_inventory().tobytes() == after.tobytes(), what
            _call(pkg, ctx, pb, pb.gpus, mv=(3, 64)[it % 2], what=what + " after place")
    finally:
        ctx.close()


# ---- 7. the sharded call on one device ------------------------------------------------------------------------------
CONFIGS = [(1, "even"), (2, "even"), (2, "uneven"), (3, "empty"), (3, "uneven"), (3, "even")]


def _sharded(pkg, pb, world, kind, bounds=None, what=""):
    """pb on a world of `world` contexts, every rank against the oracle; returns rank 0's outputs (None: a call-level
    error, which must fail every rank with nothing written)"""
    A = pkg.api
    w = SimpleNamespace(gpus=pb.gpus, node_off=pb.node_off, table=pb.table, run_claims=pb.run_claims)
    W = World(pkg, w, world, bounds or _bounds(pb.n_node, world, kind), sizes=(64, 4096, 64), n_out=len(pb.run_out))
    what = f"{what} world {world} {kind}"
    try:
        run = Running(pkg, pb.run_claims, pb.run_pod_off, pb.run_prio, pb.run_out, out_off=pb.run_out_off)
        fl = A.F_EXHAUSTIVE if pb.flags else 0
        try:
            ref = pb.oracle(W.state())
        except ValueError:
            ref = None
        if ref is None:
            outs, _ = W.enqueue(pb.claims, pb.pod_off, pb.prio, run, pb.cand_arrays() if pb.cands is not None else None,
                                pb.max_victims, fl)
            for r, c in enumerate(W.ctxs):
                with pytest.raises(A.DraError) as e:
                    c.sync()
                assert e.value.code == A.E_INVAL, (what, r)
            for r, o in enumerate(outs):
                assert all((t.cpu().numpy() == 0x5C).all() for t in o), f"{what}: rank {r} wrote an output"
            got = None
        else:
            res = W.call(pb.claims, pb.pod_off, pb.prio, run, pb.cand_arrays() if pb.cands is not None else None,
                         pb.max_victims, fl)
            for r, x in enumerate(res):
                _same(x, ref, f"{what} rank {r}")
                assert "preempt_shard" in W.ctxs[r].last_chain(), (what, r)
            got = res[0]
        for r, c in enumerate(W.ctxs):
            assert c.get_inventory().tobytes() == pb.gpus.tobytes(), f"{what}: rank {r}'s live inventory changed"
            c.reset_inventory()
            assert c.get_inventory().tobytes() == pb.gpus.tobytes(), f"{what}: rank {r}'s pristine inventory changed"
        return got
    finally:
        W.close()


def test_sharded_random_problems(pkg):
    @settings(max_examples=N_EX or 40, deadline=None, suppress_health_check=list(HealthCheck), derandomize=N_EX == 0,
              database=None)
    @given(problems(), st.sampled_from(CONFIGS))
    def run(pb, cfg):
        _sharded(pkg, pb, *cfg, what=pb.what)
    run()


def test_sharded_fixtures(pkg, monkeypatch):
    R = pkg.records
    pbs = _fixture_problems(monkeypatch)
    for i, pb in enumerate(pbs):
        for world, kind in ((1, "even"), (2, "even"), (3, "uneven")):
            _sharded(pkg, pb, world, kind, what=f"fixture {i}")
    g, off, rc, rpo, rpr, ro = _warp_world(R)
    a = [2, 1, 2, 1, 4, 0, 0] + [2] * 30 + [0] + [1] * 31 + [0] * 7
    pb = Problem(g, off, R.default_table(), _mig(R, [R.GI_7_SLICE]), np.array([0, 1], np.uint32),
                 np.array([100], np.int32), [a], rc, rpo, rpr, ro, None, 2, 0, True, False)
    for world, kind in CONFIGS:
        got = _sharded(pkg, pb, world, kind, what="past one warp")
        assert list(got[2]) == [0]


def test_sharded_priority_sum_across_ranks(pkg):
    """the two nodes of the 64-bit sum on different ranks, in both orders: the partials carry the sum as lo / hi words"""
    for a_first in (True, False):
        for cands in (None, [[0, 1]], [[1, 0]]):
            pb, nb, vic = _sum_world(pkg.records, a_first)
            pb = dataclasses.replace(pb, cands=cands)
            for flags in (0, P.F_EXHAUSTIVE):
                got = _sharded(pkg, dataclasses.replace(pb, flags=flags), 2, "even", bounds=[0, 1, 2],
                               what=f"sum {a_first} {cands}")
                assert list(got[2]) == [nb] and list(got[5][0]) == vic + [NONE, NONE]
