"""GPU suite: why preemption judged each node as it did (spec §19) through the C ABI — dra_preempt_why_batch and
dra_preempt_place_why_batch byte for byte against the CPU oracle (tests/preempt_why_oracle.py), their statuses against
dra_preempt_batch / dra_preempt_pdb_batch, their placements against dra_preempt_place_batch, and §19's consequences
against dra_unsuitable_why_batch and dra_place_pods_why_batch."""
import ctypes as C

import numpy as np
import pytest

from preempt_problems import I32_MIN, random_place_problem, random_problem
from test_preempt_why import evict_does_not_help, lost_to_an_earlier_pod  # noqa: F401  (fixtures)

import preempt_oracle as P
import preempt_why_oracle as PY
import why_oracle as Y
from oracle import oracle as O

pytestmark = pytest.mark.gpu
NONE = 0xFFFFFFFF
NAMES = ("pair_status", "pair_why", "pair_claim", "pod_why", "claim_blocks")


@pytest.fixture(scope="module")
def ctx(pkg):
    c = pkg.api.Context(device=0)
    yield c
    c.close()


def _cmp(got, ref, what):
    for name, x, y in zip(NAMES, got, ref):
        if x is None:
            continue
        y = np.ascontiguousarray(y, x.dtype).reshape(x.shape)
        if x.tobytes() != y.tobytes():
            bad = np.flatnonzero(x.ravel() != y.ravel())[:5]
            pytest.fail(f"{what}: {name} differs at {bad}: device {x.ravel()[bad]} oracle {y.ravel()[bad]}")


def _flat(cands):
    off = np.zeros(len(cands) + 1, np.uint32)
    off[1:] = np.cumsum([len(x) for x in cands])
    return np.array([n for x in cands for n in x], dtype=np.uint32), off


def _slots(pkg, claims):
    placed = claims.copy()
    placed["node"] = 0
    sl = pkg.records.claim_slots(placed, 1).astype(np.int64)
    return np.concatenate([[0], np.cumsum(sl)[:-1]]).astype(np.uint32), int(sl.sum())


def _why(ctx, w, cn, co, flags, want=True):
    """dra_preempt_why_batch on the live inventory against the oracle on w.gpus; returns the device's outputs"""
    got = ctx.preempt_why(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out,
                          getattr(w, "run_out_off", None), cn, co, flags, want, want)
    ref = PY.preempt_why(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off,
                         w.run_prio, w.run_out, getattr(w, "run_out_off", None), cn, co, flags)
    _cmp(got, ref, f"preempt_why flags {flags}")
    assert {"preempt", "unsuitable_why"} <= ctx.last_chain()
    return got


def _place_why(pkg, ctx, w, cn, co, oo, n_out, flags, want=True):
    """dra_preempt_place_why_batch from w.gpus against the oracle, then dra_preempt_place_batch from the same state"""
    roo = getattr(w, "run_out_off", None)
    ctx.set_inventory(w.gpus, w.node_off)
    got = ctx.preempt_place_why(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, roo, cn,
                                co, oo, n_out, flags, want, want)
    inv = ctx.get_inventory()
    assert {"preempt_place", "place_why"} <= ctx.last_chain()
    ref = PY.preempt_place_why(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off,
                               w.run_prio, w.run_out, roo, cn, co, oo, n_out, flags)
    if len(w.pod_off) == 1:                            # with no pending pods evicted_by is not written (the binding's zeros)
        ref = ref[:3] + (np.zeros_like(ref[3]),) + ref[4:]
    for name, x, y in zip(("out", "pod_node", "pod_status", "evicted_by"), got[:4], ref[:4]):
        assert x.tobytes() == y.tobytes(), name
    assert inv.tobytes() == ref[4].tobytes()
    _cmp(got[4:], ref[5:], f"preempt_place_why flags {flags}")
    ctx.set_inventory(w.gpus, w.node_off)
    plain = ctx.preempt_place(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, roo, cn,
                              co, oo, n_out, flags)
    for x, y in zip(plain, got[:4]):
        assert x.tobytes() == y.tobytes()
    assert ctx.get_inventory().tobytes() == inv.tobytes()
    ctx.set_inventory(w.gpus, w.node_off)
    return got


@pytest.mark.parametrize("width", [8, 16, 32])
def test_every_output_at_each_lane_width(pkg, ctx, width):
    """Synthetic preemption worlds whose nodes have `width` GPUs (the widest node sets the pair width), dense and candidate
    forms (duplicates and strays), both flags; statuses against dra_preempt_batch and dra_preempt_pdb_batch with random
    budgets, and the pairs §17 answers alike against dra_unsuitable_why_batch."""
    A = pkg.api
    w = pkg.synth.preempt(n_node=12, gpus_per_node=width, n_pending=60, seed=width)
    assert width // 2 < int(np.diff(w.node_off.astype(np.int64)).max()) <= width
    ctx.set_table(w.table)
    ctx.set_inventory(w.gpus, w.node_off)
    rng = np.random.default_rng(width)
    n_pod, n_node, n_run = len(w.pod_off) - 1, len(w.node_off) - 1, len(w.run_pod_off) - 1
    cands = _flat([list(rng.integers(0, n_node + 2, size=int(rng.integers(0, 40)))) for _ in range(n_pod)])
    seen = set()
    for cn, co in ((None, None), cands):
        for flags in (0, A.F_EXHAUSTIVE):
            st, why, claim, _, _ = _why(ctx, w, cn, co, flags, want=flags != 0)
            seen |= set(st.tolist())
            plain = ctx.preempt(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, None,
                                cn, co, 4, flags)
            assert plain[0].tobytes() == st.tobytes()
            pdb = rng.integers(0, 3, size=n_run).astype(np.uint32)
            pdb[rng.random(n_run) < 0.3] = P.NONE
            budgeted = ctx.preempt_pdb(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out,
                                       pdb, rng.integers(-1, 3, size=3).astype(np.int32), None, cn, co, 4, flags)
            assert budgeted[0].tobytes() == st.tobytes()
            if flags:                                          # consequence 3, where §19 judges on S
                u_why, u_claim, _, _ = ctx.unsuitable_why(w.claims, w.pod_off, cn, co, True)
                on_s = (st != P.NO) & (st != P.SEARCH_LIMIT)
                assert (why[on_s] == u_why[on_s]).all() and (claim[on_s] == u_claim[on_s]).all()
            oo, n_out = _slots(pkg, w.claims)
            for off in ((None, None), (oo, n_out)):
                _place_why(pkg, ctx, w, cn, co, off[0], off[1], flags, want=off[0] is not None)
    assert {P.EVICT, P.NO} <= seen


@pytest.mark.parametrize("seed", range(6))
def test_random_problems(pkg, ctx, seed):
    """preempt_problems: mixed widths, records that do not match the inventory, the int32 extremes, 0 to 33 claims, and
    call-level faults, which must fail with nothing written."""
    A = pkg.api
    for form, pb in (("14", random_problem(500 + seed, 2)), ("15", random_place_problem(700 + seed, 2)),
                     ("15", random_place_problem(900 + seed, 2))):
        ctx.set_table(pb.table)
        ctx.set_inventory(pb.gpus, pb.node_off)
        cn, co = pb.cand_arrays()
        if pb.error:
            with pytest.raises(A.DraError):
                if form == "14":
                    ctx.preempt_why(pb.claims, pb.pod_off, pb.prio, pb.run_claims, pb.run_pod_off, pb.run_prio,
                                    pb.run_out, pb.run_out_off, cn, co, pb.flags)
                else:
                    ctx.preempt_place_why(pb.claims, pb.pod_off, pb.prio, pb.run_claims, pb.run_pod_off, pb.run_prio,
                                          pb.run_out, pb.run_out_off, cn, co, pb.out_off, pb.n_out, pb.flags)
            assert ctx.get_inventory().tobytes() == pb.gpus.tobytes()
            continue
        if form == "14":
            _why(ctx, pb, cn, co, pb.flags)
        else:
            _place_why(pkg, ctx, pb, cn, co, pb.out_off, pb.n_out, pb.flags)


@pytest.mark.parametrize("flags", [0, Y.F_EXHAUSTIVE])
def test_worked_examples(pkg, ctx, evict_does_not_help, lost_to_an_earlier_pod, flags):  # noqa: F811
    f = evict_does_not_help
    ctx.set_table(f["table"]); ctx.set_inventory(f["gpus"], f["node_off"])
    got = ctx.preempt_why(f["claims"], f["pod_off"], f["prio"], f["run_claims"], f["run_pod_off"], f["run_prio"],
                          f["run_out"], None, None, None, flags)
    assert (int(got[0][0]), int(got[1][0]), int(got[2][0])) == (P.NO, Y.ST_NO_CAPACITY, 1)
    f = lost_to_an_earlier_pod
    ctx.set_inventory(f["gpus"], f["node_off"])
    got = ctx.preempt_place_why(f["claims"], f["pod_off"], f["prio"], f["run_claims"], f["run_pod_off"], f["run_prio"],
                                f["run_out"], None, None, None, None, None, flags)
    assert got[2].tolist() == [P.EVICT, P.NO] and got[3].tolist() == [NONE, 0]
    assert got[4].tolist() == [P.EVICT, P.NO] and got[5].tolist() == [Y.ST_NO_CAPACITY] * 2
    assert got[6].tolist() == [0, 1]


def test_nothing_evictable_is_place_pods_why(pkg, ctx):
    """consequence 5: no running pod below any pending pod, so the reasons are dra_place_pods_why_batch's"""
    A = pkg.api
    w = pkg.synth.preempt(n_node=10, gpus_per_node=8, n_pending=50, seed=5)
    w.prio = np.full(len(w.pod_off) - 1, I32_MIN, np.int32)
    ctx.set_table(w.table)
    oo, n_out = _slots(pkg, w.claims)
    for flags in (0, A.F_EXHAUSTIVE):
        ctx.set_inventory(w.gpus, w.node_off)
        got = ctx.preempt_place_why(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out,
                                    None, None, None, oo, n_out, flags)
        ctx.set_inventory(w.gpus, w.node_off)
        ref = ctx.place_pods_why(w.claims, w.pod_off, None, None, oo, n_out, flags)
        for x, y in zip(got[5:], ref[2:]):
            assert x.tobytes() == y.tobytes()


def test_selectors_and_search_budget(pkg, ctx):
    """Selectors (BAD_PROFILE where the selector excludes every GPU, INVALID past the selectors) and a pod whose search
    runs out of its 4096 descents: SEARCH_LIMIT with the flag, POD at the first level with no choice without it."""
    A, R = pkg.api, pkg.records
    t = R.default_table()
    g = np.zeros(8, O.GPU_DTYPE)
    g["flags"], g["node"] = 1, np.repeat([0, 1], 4)
    off = np.array([0, 4, 8], np.uint32)
    attrs = np.zeros(8, R.ATTR_DTYPE)
    attrs["index"] = np.arange(8) % 4
    sels = np.stack([R.selector(("cmp", R.ATTR_INDEX, R.CMP_EQ, 0)), R.selector(("cmp", R.ATTR_INDEX, R.CMP_GT, 9))])
    ctx.set_table(t); ctx.set_gpu_attrs(attrs); ctx.set_selectors(sels)
    O.set_selectors(attrs, sels); P.set_selectors(attrs, sels)
    try:
        small = int(np.flatnonzero(t[0]["size"] == 1)[0])
        c = np.zeros(34, O.CLAIM_DTYPE)
        c["kind"], c["profile"], c["count"] = Y.KIND_MIG, small, 1
        c[0]["mem_limit_mib"] = 1
        c[1]["mem_limit_mib"] = 2
        c[2]["mem_limit_mib"] = 5
        pod_off = np.array([0, 1, 2, 3, 33, 34], np.uint32)
        prio = np.zeros(5, np.int32)
        rc, ro = np.zeros(0, O.CLAIM_DTYPE), np.zeros(0, O.OUT_DTYPE)
        rpo, rpr = np.zeros(1, np.uint32), np.zeros(0, np.int32)
        for flags in (0, A.F_EXHAUSTIVE):
            ctx.set_inventory(g, off)
            got = ctx.preempt_why(c, pod_off, prio, rc, rpo, rpr, ro, None, None, None, flags)
            ref = PY.preempt_why(g, off, t, c, pod_off, prio, rc, rpo, rpr, ro, None, None, None, flags, attrs, sels)
            _cmp(got, ref, f"selectors {flags}")
            why = got[1].reshape(5, 2)
            assert why[1].tolist() == [Y.ST_BAD_PROFILE] * 2 and why[2].tolist() == [Y.ST_INVALID] * 2
            assert why[3].tolist() == ([Y.ST_SEARCH_LIMIT] if flags else [Y.ST_POD]) * 2
            assert got[0].reshape(5, 2)[3].tolist() == ([P.SEARCH_LIMIT] if flags else [P.NO]) * 2
            got = ctx.preempt_place_why(c, pod_off, prio, rc, rpo, rpr, ro, None, None, None, None, None, flags)
            ref = PY.preempt_place_why(g, off, t, c, pod_off, prio, rc, rpo, rpr, ro, None, None, None, None, None, flags,
                                       attrs, sels)
            _cmp(got[4:], ref[5:], f"place selectors {flags}")
            assert got[0].tobytes() == ref[0].tobytes() and ctx.get_inventory().tobytes() == ref[4].tobytes()
    finally:
        O.set_selectors(); P.set_selectors()
        ctx.set_selectors(None); ctx.set_gpu_attrs(None)


def test_refusals_and_faults_write_nothing(pkg, ctx):
    """Unknown flags, pair_why NULL with pairs, a running pod naming a GPU past the inventory (found on the device): each
    call fails with no output and no inventory word written; the next call works and writes nothing past its outputs."""
    A = pkg.api
    w = pkg.synth.preempt(n_node=6, gpus_per_node=4, n_pending=12, seed=9)
    ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
    lib, h = ctx._lib, ctx._h
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    n_pod, n_node, n_run = len(w.pod_off) - 1, len(w.node_off) - 1, len(w.run_pod_off) - 1
    n_pair, n_claim = n_pod * n_node, len(w.claims)
    cl = np.ascontiguousarray(w.claims, O.CLAIM_DTYPE)
    po, pr = np.ascontiguousarray(w.pod_off, np.uint32), np.ascontiguousarray(w.prio, np.int32)
    bad_out = w.run_out.copy()
    bad_out["gpu"][np.flatnonzero(bad_out["status"] == 0)[0]] = len(w.gpus) + 5
    oo, n_out = _slots(pkg, w.claims)
    bufs = {}

    def fresh():
        bufs.update(st=np.full(n_pair + 16, 0xAB, np.uint8), why=np.full(n_pair + 16, 0xAB, np.uint8),
                    claim=np.full(n_pair + 16, 0xABABABAB, np.uint32), pw=np.full(n_pod * Y.WHY_N + 16, 0xCD, np.uint32),
                    cb=np.full(n_claim + 16, 0xCD, np.uint32), out=np.full(n_out + 4, 0xEE, np.uint64).view(O.OUT_DTYPE),
                    node=np.full(n_pod + 4, 0xAB, np.uint32), pst=np.full(n_pod + 4, 0xAB, np.uint8),
                    ev=np.full(n_run + 4, 0xAB, np.uint32))
        return {k: v.tobytes() for k, v in bufs.items()}

    def call(which, run_out, flags, with_why=True):
        from importlib import import_module
        run = import_module("k8s-dra-driver_b200").api._running(w.run_claims, w.run_pod_off, w.run_prio, run_out)
        b = bufs
        why = p(b["why"]) if with_why else None
        if which == 14:
            return lib.dra_preempt_why_batch(h, p(cl), n_claim, p(po), p(pr), n_pod, None, None, C.byref(run), p(b["st"]),
                                             why, p(b["claim"]), p(b["pw"]), p(b["cb"]), flags)
        return lib.dra_preempt_place_why_batch(h, p(cl), n_claim, p(po), p(pr), n_pod, None, None, C.byref(run), p(oo),
                                               p(b["out"]), n_out, p(b["node"]), p(b["pst"]), p(b["ev"]), p(b["st"]), why,
                                               p(b["claim"]), p(b["pw"]), p(b["cb"]), flags)

    for which in (14, 15):
        for run_out, flags, with_why in ((w.run_out, 0x80, True), (w.run_out, 0, False), (bad_out, 0, True)):
            before = fresh()
            assert call(which, run_out, flags, with_why) == A.E_INVAL, (which, flags, with_why)
            assert {k: v.tobytes() for k, v in bufs.items()} == before, (which, flags, with_why)
            assert ctx.get_inventory().tobytes() == w.gpus.tobytes()
        before = fresh()
        assert call(which, w.run_out, A.F_EXHAUSTIVE) == A.OK
        for k, n in (("st", n_pair), ("why", n_pair), ("claim", n_pair), ("pw", n_pod * Y.WHY_N), ("cb", n_claim)):
            assert bufs[k].tobytes()[bufs[k].itemsize * n:] == before[k][bufs[k].itemsize * n:], k
        if which == 15:
            for k, n in (("out", n_out), ("node", n_pod), ("pst", n_pod), ("ev", n_run)):
                assert bufs[k].tobytes()[bufs[k].itemsize * n:] == before[k][bufs[k].itemsize * n:], k
            ctx.set_inventory(w.gpus, w.node_off)
        ref = PY.preempt_why(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off,
                             w.run_prio, w.run_out, None, None, None, A.F_EXHAUSTIVE) if which == 14 else None
        if ref is not None:
            assert bufs["why"][:n_pair].tobytes() == ref[1].tobytes()
    # no pending pods: DRA_OK without looking at the running pods
    for which in (14, 15):
        run = pkg.api._running(w.run_claims, w.run_pod_off, w.run_prio, bad_out)
        z = np.zeros(1, np.uint32)
        if which == 14:
            rc = lib.dra_preempt_why_batch(h, None, 0, p(z), None, 0, None, None, C.byref(run), None, None, None, None,
                                           None, 0)
        else:
            rc = lib.dra_preempt_place_why_batch(h, None, 0, p(z), None, 0, None, None, C.byref(run), None, None, 0, None,
                                                 None, p(np.zeros(n_run, np.uint32)), None, None, None, None, None, 0)
        assert rc == A.OK
