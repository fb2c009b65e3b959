"""GPU suite: preemption with disruption budgets on one inventory (dra_preempt_pdb_batch, spec §14 "Disruption budgets").
Every call's eight outputs are compared byte for byte with preempt_oracle.preempt_pdb on the context's live inventory:
random problems at every lane width the pair kernel instantiates, with and without DRA_F_EXHAUSTIVE, with selectors,
victim rows shorter than the victim count, and running records that do not match the inventory.  With no budgets the
call is dra_preempt_batch, kernel chain included; a bad budget index fails with nothing written."""
import ctypes as C

import numpy as np
import pytest

import preempt_oracle as P
import preempt_oracle as PB
from preempt_problems import I32_MAX, I32_MIN, random_problem

pytestmark = pytest.mark.gpu
NONE = 0xFFFFFFFF
SENT = 0xA5
NAMES = ("pair_status", "pair_victims", "pod_node", "pod_status", "n_victims", "victims", "pair_violations",
         "pod_violations")
ALLOWED = (I32_MIN, -1, 0, 0, 1, 1, 2, 3, I32_MAX)


@pytest.fixture(scope="module")
def ctx(pkg):
    c = pkg.api.Context(device=0)
    yield c
    c.close()


def budgets(rng, n_run, n_pdb=None):
    """(run_pdb, allowed): budgets spanning nodes, NONE mixed in, now and then one budget holding most pods"""
    n_pdb = int(rng.integers(1, 6)) if n_pdb is None else n_pdb
    allowed = np.array([ALLOWED[int(i)] for i in rng.integers(0, len(ALLOWED), n_pdb)], np.int32)
    if rng.integers(0, 3) == 0:
        run_pdb = np.where(rng.integers(0, 6, n_run) > 0, 0, NONE)
    else:
        run_pdb = rng.integers(0, n_pdb + 1, n_run)
        run_pdb[run_pdb == n_pdb] = NONE
    return run_pdb.astype(np.uint32), allowed


def _check(ctx, gpus, node_off, table, claims, pod_off, prio, run, run_pdb, allowed, cands=None, mv=8, flags=0,
           what=""):
    """the device call against the oracle on `gpus` (the live inventory); returns the outputs"""
    rc, rpo, rpr, ro, roo = run
    cn, co = cands if cands is not None else (None, None)
    try:
        ref = PB.preempt_pdb(gpus, node_off, table, claims, pod_off, prio, rc, rpo, rpr, ro, run_pdb, allowed, roo, cn, co,
                            mv, P.F_EXHAUSTIVE if flags else 0)
    except ValueError:
        ref = None
    A = ctx._pkg_api
    if ref is None:
        with pytest.raises(A.DraError) as e:
            ctx.preempt_pdb(claims, pod_off, prio, rc, rpo, rpr, ro, run_pdb, allowed, roo, cn, co, mv,
                            A.F_EXHAUSTIVE if flags else 0)
        assert e.value.code == A.E_INVAL, what
        return None
    got = ctx.preempt_pdb(claims, pod_off, prio, rc, rpo, rpr, ro, run_pdb, allowed, roo, cn, co, mv,
                          A.F_EXHAUSTIVE if flags else 0)
    for name, x, y in zip(NAMES, got, ref):
        if x.tobytes() != y.tobytes():
            bad = np.flatnonzero(x.reshape(-1) != y.reshape(-1))[:5]
            pytest.fail(f"{what}: {name} differs at {bad}: device {x.reshape(-1)[bad]} oracle {y.reshape(-1)[bad]}")
    return got


def _load(ctx, pkg, table, gpus, node_off):
    ctx._pkg_api = pkg.api
    ctx.set_table(table)
    ctx.set_inventory(gpus, node_off)


def _cands(rng, n_pod, n_node, k):
    nodes = rng.integers(0, n_node + 2, size=n_pod * k).astype(np.uint32)
    return nodes, (np.arange(n_pod + 1) * k).astype(np.uint32)


@pytest.mark.parametrize("width", [4, 8, 16, 32])
def test_synth_worlds_at_every_lane_width(pkg, ctx, width):
    """Lane widths 8 (nodes of up to 8 GPUs), 16 and 32; dense and candidate forms; both flags; rows of 2 and 16."""
    rng = np.random.default_rng(width)
    for seed in range(3):
        w = pkg.synth.preempt(n_node=16, gpus_per_node=width, n_pending=40, seed=100 * width + seed)
        _load(ctx, pkg, w.table, w.gpus, w.node_off)
        run = (w.run_claims, w.run_pod_off, w.run_prio, w.run_out, None)
        n_run = len(w.run_prio)
        viol = 0
        for flags in (0, 1):
            for form in ("dense", "cands"):
                cands = None if form == "dense" else _cands(rng, len(w.prio), 16, 6)
                for mv in (2, 16):
                    run_pdb, allowed = budgets(rng, n_run)
                    got = _check(ctx, ctx.get_inventory(), w.node_off, w.table, w.claims, w.pod_off, w.prio, run,
                                 run_pdb, allowed, cands, mv, flags, f"width {width} seed {seed} f{flags} {form} mv{mv}")
                    viol += int(got[6].sum())
        assert viol > 0                                   # the budgets did bite


@pytest.mark.parametrize("seed", range(40))
def test_random_problems(pkg, ctx, seed):
    """tests/preempt_problems.py: mixed widths, mismatched records, run_out_off, int32 extremes, call-level errors"""
    pb = random_problem(seed, scale=1 + seed % 3)
    rng = np.random.default_rng(seed)
    _load(ctx, pkg, pb.table, pb.gpus, pb.node_off)
    run = (pb.run_claims, pb.run_pod_off, pb.run_prio, pb.run_out, pb.run_out_off)
    for _ in range(2):
        run_pdb, allowed = budgets(rng, len(pb.run_prio))
        _check(ctx, ctx.get_inventory(), pb.node_off, pb.table, pb.claims, pb.pod_off, pb.prio, run, run_pdb, allowed,
               pb.cand_arrays() if pb.cands is not None else None, pb.max_victims, pb.flags, f"seed {seed} {pb.what}")


def test_selectors(pkg, ctx):
    R = pkg.records
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=30, seed=7)
    attrs = np.zeros(len(w.gpus), R.ATTR_DTYPE)
    attrs["index"] = np.arange(len(w.gpus)) % 8
    attrs["mem_total_mib"] = 81920
    sels = np.stack([R.selector(("cmp", R.ATTR_INDEX, R.CMP_LT, 4)), R.selector(("cmp", R.ATTR_INDEX, R.CMP_GE, 4))])
    c = w.claims.copy()
    mig = c["kind"] == R.KIND_MIG
    c["mem_limit_mib"] = np.where(mig, (np.arange(len(c)) % 4).astype(np.uint32), 0)   # ids 0..3, 3 beyond the table
    _load(ctx, pkg, w.table, w.gpus, w.node_off)
    ctx.set_gpu_attrs(attrs)
    ctx.set_selectors(sels.reshape(-1, R.SEL_MAX_INS))
    PB.set_selectors(attrs, sels)
    try:
        rng = np.random.default_rng(3)
        run = (w.run_claims, w.run_pod_off, w.run_prio, w.run_out, None)
        for flags in (0, 1):
            run_pdb, allowed = budgets(rng, len(w.run_prio))
            _check(ctx, ctx.get_inventory(), w.node_off, w.table, c, w.pod_off, w.prio, run, run_pdb, allowed,
                   _cands(rng, len(w.prio), 12, 5), 16, flags, f"selectors f{flags}")
    finally:
        PB.set_selectors()
        ctx.set_selectors(None)
        ctx.set_gpu_attrs(None)


def test_no_budgets_is_preempt(pkg, ctx):
    """NULL budgets, n_pdb = 0 and every run_pdb NONE: dra_preempt_batch's six outputs and kernel chain, violations 0"""
    w = pkg.synth.preempt(n_node=16, gpus_per_node=8, n_pending=60, seed=3)
    _load(ctx, pkg, w.table, w.gpus, w.node_off)
    n_run = len(w.run_prio)
    args = (w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out)
    for flags in (0, pkg.api.F_EXHAUSTIVE):
        ref = ctx.preempt(*args, None, None, None, 8, flags)
        chain = ctx.last_chain()
        for run_pdb, allowed in ((None, None), (np.full(n_run, NONE, np.uint32), None),
                                 (np.full(n_run, NONE, np.uint32), np.array([0, -1], np.int32))):
            got = ctx.preempt_pdb(*args, run_pdb, allowed, None, None, None, 8, flags)
            for name, x, y in zip(NAMES, got, ref):
                assert x.tobytes() == y.tobytes(), name
            assert not got[6].any() and not got[7].any()
            assert ctx.last_chain() == chain


def test_bad_budgets_fail_with_nothing_written(pkg, ctx):
    A = pkg.api
    w = pkg.synth.preempt(n_node=8, gpus_per_node=8, n_pending=20, seed=11)
    _load(ctx, pkg, w.table, w.gpus, w.node_off)
    c = np.ascontiguousarray(w.claims)
    po, pr = np.ascontiguousarray(w.pod_off, np.uint32), np.ascontiguousarray(w.prio, np.int32)
    n_pod, n_run, n_pair = len(po) - 1, len(w.run_prio), (len(po) - 1) * 8
    run = A._running(w.run_claims, w.run_pod_off, w.run_prio, w.run_out)
    good = np.zeros(n_run, np.uint32)
    bad = good.copy()
    bad[n_run // 2] = 2                                  # n_pdb is 2
    allowed = np.array([0, 1], np.int32)
    for run_pdb, al, n_pdb in ((bad, allowed, 2), (good, None, 2), (None, allowed, 2)):
        bud = A.DisruptionBudgets(None if run_pdb is None else run_pdb.ctypes.data,
                                  None if al is None else al.ctypes.data, n_pdb)
        outs = [np.full(n, SENT, np.uint8) for n in (n_pair, 4 * n_pair, 4 * n_pair, 4 * n_pod, n_pod, 4 * n_pod,
                                                     4 * n_pod, 4 * n_pod * 4)]
        p = [o.ctypes.data_as(C.c_void_p) for o in outs]
        rc = ctx._lib.dra_preempt_pdb_batch(ctx._h, c.ctypes.data, len(c), po.ctypes.data, pr.ctypes.data, n_pod, None,
                                            None, C.byref(run), C.byref(bud), *p, 4, 0)
        assert rc == A.E_INVAL
        assert all((o == SENT).all() for o in outs)
    # the next call works
    _check(ctx, ctx.get_inventory(), w.node_off, w.table, w.claims, w.pod_off, w.prio,
           (w.run_claims, w.run_pod_off, w.run_prio, w.run_out, None), good, allowed, None, 4, 0, "after the faults")
