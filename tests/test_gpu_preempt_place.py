"""GPU suite: preempt and place (spec §15) through the C ABI — OutRecs, pod_node, pod_status, evicted_by and the live
inventory afterwards bit-exact with the CPU oracle; the call equal to its host loop on the device, and to place pods when
nothing is evictable."""
import ctypes as C

import numpy as np
import pytest

from test_preempt import error_cases

import preempt_oracle as P
import preempt_place_oracle as PP

pytestmark = pytest.mark.gpu
NONE = 0xFFFFFFFF


@pytest.fixture(scope="module")
def ctx(pkg):
    c = pkg.api.Context(device=0)
    yield c
    c.close()


def _load(ctx, w):
    ctx.set_table(w.table)
    ctx.set_inventory(w.gpus, w.node_off)


def _slots(pkg, claims):
    R = pkg.records
    placed = claims.copy()
    placed["node"] = 0
    sl = R.claim_slots(placed, 1).astype(np.int64)
    return np.concatenate([[0], np.cumsum(sl)[:-1]]).astype(np.uint32), int(sl.sum())


def _check(pkg, ctx, w, claims=None, pod_off=None, prio=None, cands=None, flags=0, what=""):
    """One call on the device against the oracle, both from the world's inventory; returns the device's outputs."""
    A = pkg.api
    claims = w.claims if claims is None else claims
    pod_off = w.pod_off if pod_off is None else pod_off
    prio = w.prio if prio is None else prio
    cn, co = (None, None) if cands is None else cands
    oo, n_out = _slots(pkg, claims)
    _load(ctx, w)
    got = ctx.preempt_place(claims, pod_off, prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, None, cn, co,
                            oo, n_out, flags)
    ref = PP.preempt_place(w.gpus, w.node_off, w.table, claims, pod_off, prio, w.run_claims, w.run_pod_off, w.run_prio,
                           w.run_out, None, cn, co, oo, n_out, PP.F_EXHAUSTIVE if flags & A.F_EXHAUSTIVE else 0)
    for name, x, y in zip(("out", "pod_node", "pod_status", "evicted_by"), got, ref):
        if x.tobytes() != y.tobytes():
            bad = np.flatnonzero(x.view(np.uint8) != y.view(np.uint8))[:5]
            pytest.fail(f"{what}: {name} differs at bytes {bad}")
    assert ctx.get_inventory().tobytes() == ref[4].tobytes(), f"{what}: inventory"
    assert "preempt_place" in ctx.last_chain()
    return got


def _random_cands(rng, n_pod, n_node, k):
    nodes = rng.integers(0, n_node + 2, size=n_pod * k).astype(np.uint32)       # duplicates and strays included
    return nodes, (np.arange(n_pod + 1) * k).astype(np.uint32)


@pytest.mark.parametrize("seed,width", [(0, 8), (1, 4), (2, 32), (3, 16)])
def test_synthetic_worlds(pkg, ctx, seed, width):
    w = pkg.synth.preempt(n_node=24, gpus_per_node=width, n_pending=120, seed=seed)
    rng = np.random.default_rng(seed)
    for flags in (0, pkg.api.F_EXHAUSTIVE):
        got = _check(pkg, ctx, w, flags=flags, what=f"dense w{width} f{flags}")
        assert (got[2] == P.EVICT).any() and (got[3] != NONE).any()
        _check(pkg, ctx, w, cands=_random_cands(rng, len(w.pod_off) - 1, 24, 6), flags=flags, what=f"cands w{width} f{flags}")


def test_selectors_and_long_pods(pkg, ctx):
    R = pkg.records
    w = pkg.synth.preempt(n_node=10, gpus_per_node=8, n_pending=30, seed=7)
    attrs = np.zeros(len(w.gpus), R.ATTR_DTYPE)
    attrs["index"] = np.arange(len(w.gpus)) % 8
    attrs["mem_total_mib"] = 81920
    sels = np.stack([R.selector(("cmp", R.ATTR_INDEX, R.CMP_LT, 4)), R.selector(("cmp", R.ATTR_INDEX, R.CMP_GE, 4))])
    c = w.claims.copy()
    mig = c["kind"] == R.KIND_MIG
    c["mem_limit_mib"] = np.where(mig, (np.arange(len(c)) % 4).astype(np.uint32), 0)   # ids 0..3, 3 beyond the table
    extra = np.zeros(65, R.CLAIM_DTYPE)                      # a pod of 32 1g claims and one of 33
    extra["kind"], extra["count"], extra["profile"] = R.KIND_MIG, 1, R.GI_1_SLICE
    c = np.concatenate([c, extra])
    pod_off = np.concatenate([w.pod_off, [len(w.claims) + 32, len(c)]]).astype(np.uint32)
    prio = np.concatenate([w.prio, [2000, 2000]]).astype(np.int32)
    ctx.set_gpu_attrs(None); ctx.set_selectors(None)
    try:
        for flags in (0, pkg.api.F_EXHAUSTIVE):
            _load(ctx, w)
            ctx.set_gpu_attrs(attrs); ctx.set_selectors(sels)
            PP.set_selectors(attrs, sels)
            got = _check_loaded(pkg, ctx, w, c, pod_off, prio, flags)
            assert got[2][-1] == P.INVALID
    finally:
        ctx.set_gpu_attrs(None); ctx.set_selectors(None)
        PP.set_selectors()


def _check_loaded(pkg, ctx, w, claims, pod_off, prio, flags):
    """_check without reloading the inventory (the selector context stays)"""
    oo, n_out = _slots(pkg, claims)
    got = ctx.preempt_place(claims, pod_off, prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, None, None, None,
                            oo, n_out, flags)
    ref = PP.preempt_place(w.gpus, w.node_off, w.table, claims, pod_off, prio, w.run_claims, w.run_pod_off, w.run_prio,
                           w.run_out, None, None, None, oo, n_out, PP.F_EXHAUSTIVE if flags else 0)
    for x, y in zip(got, ref):
        assert x.tobytes() == y.tobytes()
    assert ctx.get_inventory().tobytes() == ref[4].tobytes()
    return got


def test_time_slicing_world(pkg, ctx):
    """SHARED-heavy: every non-MIG GPU time-sliced by up to 12 pods; pending 2-GPU pods must clear whole GPUs."""
    w = pkg.synth.preempt(n_node=16, gpus_per_node=8, n_pending=80, seed=4, mig_nodes=0, shared_per_gpu=12,
                          shapes=("gpu2",))
    for flags in (0, pkg.api.F_EXHAUSTIVE):
        got = _check(pkg, ctx, w, flags=flags, what=f"time slicing f{flags}")
        assert (got[2] == P.EVICT).any()


def test_cfg2_sized_world(pkg, ctx):
    """125 nodes of 8 MIG GPUs, 1,000 pending pods, dense and with 8 candidates each."""
    w = pkg.synth.preempt(n_node=125, gpus_per_node=8, n_pending=1000, seed=12, mig_nodes=4)
    rng = np.random.default_rng(12)
    _check(pkg, ctx, w, flags=pkg.api.F_EXHAUSTIVE, what="cfg2 dense")
    _check(pkg, ctx, w, cands=_random_cands(rng, 1000, 125, 8), what="cfg2 cands")


def test_equals_the_host_loop_on_the_device(pkg, ctx):
    """A second context runs, per pod, dra_preempt_batch with that pod and the running pods not evicted yet,
    dra_deallocate_batch of its victims and dra_allocate_pods_batch on the chosen node."""
    A, R = pkg.api, pkg.records
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=40, seed=21)
    n_node, n_run = len(w.node_off) - 1, len(w.run_pod_off) - 1
    oo, n_out = _slots(pkg, w.claims)
    for flags in (0, A.F_EXHAUSTIVE):
        got = _check(pkg, ctx, w, flags=flags, what=f"host loop f{flags}")
        inv = ctx.get_inventory()
        with A.Context(device=0) as h:
            _load(h, w)
            ev = np.full(n_run, NONE, np.uint32)
            out = np.zeros(n_out, R.OUT_DTYPE)
            placed = np.zeros(n_out, bool)                   # the slots the loop writes: those of the placed pods
            for p in range(len(w.pod_off) - 1):
                c0, c1 = int(w.pod_off[p]), int(w.pod_off[p + 1])
                alive = np.flatnonzero(ev == NONE)
                keep = np.zeros(len(w.run_claims), bool)
                for r in alive:
                    keep[w.run_pod_off[r]: w.run_pod_off[r + 1]] = True
                rpo = np.concatenate([[0], np.cumsum(w.run_pod_off[alive + 1] - w.run_pod_off[alive])]).astype(np.uint32)
                _, _, pn, ps, nv, vic = h.preempt(w.claims[c0:c1], np.array([0, c1 - c0], np.uint32), w.prio[p:p + 1],
                                                  w.run_claims[keep], rpo, w.run_prio[alive], w.run_out[keep],
                                                  max_victims=max(len(alive), 1), flags=flags)
                assert pn[0] == got[1][p] and ps[0] == got[2][p], p
                victims = alive[vic[0][: nv[0]]]
                ev[victims] = p
                vk = np.zeros(len(w.run_claims), bool)
                for r in victims:
                    vk[w.run_pod_off[r]: w.run_pod_off[r + 1]] = True
                if vk.any():
                    h.deallocate(w.run_claims[vk], w.run_out[vk])
                if pn[0] != NONE and c1 > c0:
                    pod = w.claims[c0:c1].copy()
                    pod["node"] = pn[0]
                    po_ = h.allocate_pods(pod, np.array([0, c1 - c0], np.uint32), oo[c0:c1] - oo[c0],
                                          n_out - int(oo[c0]), flags)
                    n = int(R.claim_slots(pod, n_node).sum())
                    out[oo[c0]: oo[c0] + n] = po_[:n]
                    placed[oo[c0]: oo[c0] + n] = True
            assert ev.tobytes() == got[3].tobytes()
            assert placed.any() and out[placed].tobytes() == got[0][placed].tobytes()
            assert h.get_inventory().tobytes() == inv.tobytes()


def test_equals_place_pods_when_nothing_is_evictable(pkg, ctx):
    w = pkg.synth.preempt(n_node=20, gpus_per_node=8, n_pending=100, seed=8, prio_lo=500, prio_hi=600, pending_prio=500)
    oo, n_out = _slots(pkg, w.claims)
    for flags in (0, pkg.api.F_EXHAUSTIVE):
        out, node, st, ev = _check(pkg, ctx, w, flags=flags, what=f"nothing evictable f{flags}")
        inv = ctx.get_inventory()
        _load(ctx, w)
        pout, pnode = ctx.place_pods(w.claims, w.pod_off, None, None, oo, n_out, flags)
        assert out.tobytes() == pout.tobytes() and ctx.get_inventory().tobytes() == inv.tobytes()
        nonempty = np.diff(w.pod_off) > 0
        assert (node[nonempty] == pnode[nonempty]).all() and (ev == NONE).all()


def _raw(pkg, ctx, a, sentinel, slack=0):
    """dra_preempt_place_batch on sentinel-filled outputs, each `slack` elements longer than the call may write (n_out:
    a["n_out"], default 1); returns (rc, outputs)"""
    A = pkg.api
    n_pod = len(a["po"]) - 1
    n_out = a.get("n_out", 1)
    def filled(n, dtype):                                 # every byte = sentinel
        return np.full((max(n, 1) + slack) * np.dtype(dtype).itemsize, sentinel, np.uint8).view(dtype)
    outs = [filled(n_out, A.R.OUT_DTYPE), filled(n_pod, np.uint32), filled(n_pod, np.uint8), filled(len(a["rpo"]) - 1, np.uint32)]
    keep = [np.ascontiguousarray(a[k], dtype=d) if a.get(k) is not None else None for k, d in
            (("c", A.R.CLAIM_DTYPE), ("po", np.uint32), ("prio", np.int32), ("rc", A.R.CLAIM_DTYPE), ("rpo", np.uint32),
             ("rpr", np.int32), ("ro", A.R.OUT_DTYPE), ("roo", np.uint32), ("cn", np.uint32), ("co", np.uint32),
             ("oo", np.uint32))]
    c, po, prio, rc, rpo, rpr, ro, roo, cn, co, oo = keep
    run = A.RunningPods(rc.ctypes.data, len(rc), rpo.ctypes.data, len(rpo) - 1, rpr.ctypes.data,
                        None if roo is None else roo.ctypes.data, ro.ctypes.data, len(ro))
    p = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)      # noqa: E731
    rc_ = ctx._lib.dra_preempt_place_batch(ctx._h, p(c), len(c), p(po), p(prio), n_pod, p(cn), p(co), C.byref(run),
                                           p(oo), p(outs[0]), n_out, p(outs[1]), p(outs[2]), p(outs[3]), a["fl"])
    return rc_, outs


def test_call_errors_leave_the_outputs_and_the_inventory_alone(pkg, ctx, oracle):
    """Host-detected errors (flags, offsets, slots) and device-detected ones (the running pods) alike."""
    A, R = pkg.api, pkg.records
    g, off = R.make_inventory([1, 1], mig=True)
    ctx.set_table(R.default_table()); ctx.set_inventory(g, off)
    ok, cases = error_cases(g, off)
    rc_, outs = _raw(pkg, ctx, ok, 0xAB)
    assert rc_ == A.OK and outs[1][0] == 0 and outs[2][0] == P.FITS
    ctx.set_inventory(g, off)
    cases = cases + [("slot outside n_out", dict(oo=np.array([3], np.uint32)))]
    for name, kw in cases:
        rc_, outs = _raw(pkg, ctx, dict(ok, **kw), 0xAB)
        assert rc_ == A.E_INVAL, name
        assert all((o.view(np.uint8) == 0xAB).all() for o in outs), name
        assert ctx.get_inventory().tobytes() == g.tobytes(), name
    # the context keeps working
    w = pkg.synth.cfg2(2000, 16)
    ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
    out = ctx.allocate(w.claims, w.out_off, w.n_out)
    ref, inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
    assert out.tobytes() == ref.tobytes() and ctx.get_inventory().tobytes() == inv.tobytes()
    _check(pkg, ctx, pkg.synth.preempt(n_node=8, gpus_per_node=8, n_pending=16, seed=9), what="after the errors")
