"""GPU suite: preemption (spec §14) through the C ABI — all outputs bit-exact with the CPU oracle, the inventory untouched."""
import ctypes as C

import numpy as np
import pytest

from test_preempt import _flat, error_cases, mig_running

import preempt_oracle as P

pytestmark = pytest.mark.gpu
NONE = 0xFFFFFFFF


@pytest.fixture(scope="module")
def pctx(pkg):
    c = pkg.api.Context(device=0)
    yield c
    c.close()


def _check(pkg, ctx, w, claims=None, pod_off=None, prio=None, cands=None, flags=0, max_victims=16, what=""):
    """One call on the device against the oracle on the world's inventory; returns the device's outputs."""
    A = pkg.api
    claims = w.claims if claims is None else claims
    pod_off = w.pod_off if pod_off is None else pod_off
    prio = w.prio if prio is None else prio
    cn, co = (None, None) if cands is None else cands
    before = ctx.get_inventory()
    got = ctx.preempt(claims, pod_off, prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, None, cn, co,
                      max_victims, flags)
    ref = P.preempt(before, w.node_off, w.table, claims, pod_off, prio, w.run_claims, w.run_pod_off, w.run_prio,
                    w.run_out, None, cn, co, max_victims, P.F_EXHAUSTIVE if flags & A.F_EXHAUSTIVE else 0)
    for name, x, y in zip(("pair_status", "pair_victims", "pod_node", "pod_status", "n_victims", "victims"), got, ref):
        if x.tobytes() != y.tobytes():
            bad = np.flatnonzero(x.reshape(-1) != y.reshape(-1))[:5]
            pytest.fail(f"{what}: {name} differs at {bad}: device {x.reshape(-1)[bad]} oracle {y.reshape(-1)[bad]}")
    assert ctx.get_inventory().tobytes() == before.tobytes(), what
    assert "preempt" in ctx.last_chain()
    return got


def _load(ctx, w):
    ctx.set_table(w.table)
    ctx.set_inventory(w.gpus, w.node_off)


def _random_cands(rng, n_pod, n_node, k):
    nodes = rng.integers(0, n_node + 2, size=n_pod * k).astype(np.uint32)       # duplicates and strays included
    return nodes, (np.arange(n_pod + 1) * k).astype(np.uint32)


@pytest.mark.parametrize("seed,width", [(0, 8), (1, 4), (2, 32), (3, 16)])
def test_synthetic_worlds(pkg, pctx, seed, width):
    w = pkg.synth.preempt(n_node=24, gpus_per_node=width, n_pending=120, seed=seed)
    _load(pctx, w)
    rng = np.random.default_rng(seed)
    for flags in (0, pkg.api.F_EXHAUSTIVE):
        got = _check(pkg, pctx, w, flags=flags, what=f"dense w{width} f{flags}")
        assert (got[3] == P.EVICT).any()
        _check(pkg, pctx, w, cands=_random_cands(rng, len(w.pod_off) - 1, 24, 6), flags=flags, max_victims=3,
               what=f"cands w{width} f{flags}")


def test_fits_pairs_are_the_exhaustive_unsuitable_bits(pkg, pctx):
    w = pkg.synth.preempt(n_node=20, gpus_per_node=8, n_pending=60, seed=5, fill=30)
    _load(pctx, w)
    got = _check(pkg, pctx, w, flags=pkg.api.F_EXHAUSTIVE)
    bits = pctx.unsuitable(w.claims, w.pod_off, flags=pkg.api.F_EXHAUSTIVE)
    fits = np.unpackbits(bits, bitorder="little")[: len(got[0])].astype(bool)
    assert (fits == (got[0] == P.FITS)).all() and fits.any()


def test_selectors_and_long_pods(pkg, pctx):
    R = pkg.records
    w = pkg.synth.preempt(n_node=10, gpus_per_node=8, n_pending=30, seed=7)
    attrs = np.zeros(len(w.gpus), R.ATTR_DTYPE)
    attrs["index"] = np.arange(len(w.gpus)) % 8
    attrs["mem_total_mib"] = 81920
    sels = np.stack([R.selector(("cmp", R.ATTR_INDEX, R.CMP_LT, 4)), R.selector(("cmp", R.ATTR_INDEX, R.CMP_GE, 4))])
    c = w.claims.copy()
    mig = c["kind"] == R.KIND_MIG
    c["mem_limit_mib"] = np.where(mig, (np.arange(len(c)) % 4).astype(np.uint32), 0)   # ids 0..3, 3 beyond the table
    # a pod of 32 1g claims and one of 33
    extra = np.zeros(65, R.CLAIM_DTYPE)
    extra["kind"], extra["count"], extra["profile"] = R.KIND_MIG, 1, R.GI_1_SLICE
    c = np.concatenate([c, extra])
    pod_off = np.concatenate([w.pod_off, [len(w.claims) + 32, len(c)]]).astype(np.uint32)
    prio = np.concatenate([w.prio, [2000, 2000]]).astype(np.int32)
    _load(pctx, w)
    pctx.set_gpu_attrs(attrs); pctx.set_selectors(sels)
    P.set_selectors(attrs, sels)
    try:
        for flags in (0, pkg.api.F_EXHAUSTIVE):
            got = _check(pkg, pctx, w, c, pod_off, prio, flags=flags, what=f"selectors f{flags}")
            assert got[3][-1] == P.INVALID
    finally:
        pctx.set_gpu_attrs(None); pctx.set_selectors(None)
        P.set_selectors()


def test_dense_hundred_thousand_pairs(pkg, pctx):
    w = pkg.synth.preempt(n_node=250, gpus_per_node=8, n_pending=400, seed=11)
    _load(pctx, w)
    got = _check(pkg, pctx, w, flags=pkg.api.F_EXHAUSTIVE, max_victims=8, what="dense 1e5")
    assert len(got[0]) == 100_000


def test_long_reprieve_on_a_time_slicing_node(pkg, pctx):
    """1,200 time-slicing pods on one 8-GPU node; a pending 2-GPU pod of higher priority than all of them must clear two
    GPUs, so every one of them is removed and then reprieved one at a time."""
    R = pkg.records
    g, off = R.make_inventory([8, 8], mig=False)
    n = 1200
    rc = np.zeros(n, R.CLAIM_DTYPE)
    rc["kind"], rc["count"], rc["node"] = R.KIND_SHARED, 1, 0
    ro = np.zeros(n, R.OUT_DTYPE)
    ro["gpu"] = np.arange(n) % 8
    ro["profile"], ro["status"] = R.PROFILE_SHARED, R.ST_OK
    np.add.at(g["share_cnt"], ro["gpu"], 1)
    g["share_cnt"][8:] = 1                                    # node 1: every GPU shared by a pod not in the list
    w = pkg.synth.PreemptWorld(g, g, off, R.default_table(), rc, np.arange(n + 1, dtype=np.uint32),
                               (np.arange(n) % 97 - 40).astype(np.int32), ro, None, None, None)
    c = np.zeros(1, R.CLAIM_DTYPE)
    c["kind"], c["count"] = R.KIND_GPU, 2
    _load(pctx, w)
    for flags in (0, pkg.api.F_EXHAUSTIVE):
        got = _check(pkg, pctx, w, c, np.array([0, 1], np.uint32), np.array([100], np.int32), flags=flags,
                     max_victims=400, what="time slicing")
        assert list(got[3]) == [P.EVICT] and list(got[2]) == [0] and got[4][0] == 300


def test_the_full_flow(pkg, pctx, oracle):
    """Deallocate the chosen victims, then allocate the pod on pod_node: it is placed."""
    R, A = pkg.records, pkg.api
    w = pkg.synth.preempt(n_node=16, gpus_per_node=8, n_pending=24, seed=3)
    for flags in (0, A.F_EXHAUSTIVE):
        _load(pctx, w)
        st, pv, node, pst, nv, vic = _check(pkg, pctx, w, flags=flags, max_victims=64)
        done = 0
        for p in np.flatnonzero(pst == P.EVICT)[:6]:
            _load(pctx, w)
            keep = np.zeros(len(w.run_claims), bool)
            for r in vic[p][: nv[p]]:
                keep[w.run_pod_off[r]: w.run_pod_off[r + 1]] = True
            pctx.deallocate(w.run_claims[keep], w.run_out[keep])
            pod = w.claims[w.pod_off[p]: w.pod_off[p + 1]].copy()
            pod["node"] = node[p]
            oo, n_out = R.out_offsets(pod, len(w.node_off) - 1)
            out = pctx.allocate_pods(pod, np.array([0, len(pod)], np.uint32), oo, n_out, flags)
            assert (out["status"] == R.ST_OK).all()
            done += 1
        assert done


def _raw(pkg, ctx, g, a, sentinel):
    """dra_preempt_batch on sentinel-filled outputs; returns (rc, outputs)"""
    A = pkg.api
    n_pod = len(a["po"]) - 1
    n_pair = n_pod * ctx.n_node if a["co"] is None else int(a["co"][-1])
    def filled(n, dtype):                                 # every byte = sentinel
        return np.full(max(n, 1) * np.dtype(dtype).itemsize, sentinel, np.uint8).view(dtype)
    outs = [filled(n_pair, np.uint8), filled(n_pair, np.uint32)] + \
           [filled(n_pod, d) for d in (np.uint32, np.uint8, np.uint32)] + [filled(n_pod * a["mv"], np.uint32)]
    keep = [np.ascontiguousarray(a[k], dtype=d) if a[k] is not None else None for k, d in
            (("c", A.R.CLAIM_DTYPE), ("po", np.uint32), ("prio", np.int32), ("rc", A.R.CLAIM_DTYPE), ("rpo", np.uint32),
             ("rpr", np.int32), ("ro", A.R.OUT_DTYPE), ("roo", np.uint32), ("cn", np.uint32), ("co", np.uint32))]
    c, po, prio, rc, rpo, rpr, ro, roo, cn, co = keep
    run = A.RunningPods(rc.ctypes.data, len(rc), rpo.ctypes.data, len(rpo) - 1, rpr.ctypes.data,
                        None if roo is None else roo.ctypes.data, ro.ctypes.data, len(ro))
    p = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)      # noqa: E731
    rc_ = ctx._lib.dra_preempt_batch(ctx._h, p(c), len(c), p(po), p(prio), n_pod, p(cn), p(co), C.byref(run),
                                     *[p(o) for o in outs[:5]], p(outs[5]) if a.get("victims", True) else None,
                                     a["mv"], a["fl"])
    return rc_, outs


def test_call_errors_leave_the_outputs_alone(pkg, pctx, oracle):
    A, R = pkg.api, pkg.records
    g, off = R.make_inventory([1, 1], mig=True)
    pctx.set_table(R.default_table()); pctx.set_inventory(g, off)
    ok, cases = error_cases(g, off)
    rc_, outs = _raw(pkg, pctx, g, ok, 0xAB)
    assert rc_ == A.OK and outs[2][0] == 0
    for name, kw in cases + [("max_victims without a buffer", dict(victims=False))]:
        rc_, outs = _raw(pkg, pctx, g, dict(ok, **kw), 0xAB)
        assert rc_ == A.E_INVAL, name
        assert all((o.view(np.uint8) == 0xAB).all() for o in outs), name
        assert pctx.get_inventory().tobytes() == g.tobytes(), name
    # the context keeps working: an Allocate batch matches the oracle, and so does a valid preemption call
    w = pkg.synth.cfg2(2000, 16)
    pctx.set_table(w.table); pctx.set_inventory(w.gpus, w.node_off)
    out = pctx.allocate(w.claims, w.out_off, w.n_out)
    ref, inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
    assert out.tobytes() == ref.tobytes() and pctx.get_inventory().tobytes() == inv.tobytes()
    pw = pkg.synth.preempt(n_node=8, gpus_per_node=8, n_pending=16, seed=9)
    _load(pctx, pw)
    _check(pkg, pctx, pw, what="after the errors")


def test_dense_over_two_to_the_32_pairs(pkg, pctx):
    R = pkg.records
    n = 1 << 16
    g, off = R.make_inventory([1] * n, mig=True)
    pctx.set_table(R.default_table()); pctx.set_inventory(g, off)
    with pytest.raises(pkg.api.DraError):
        pctx.preempt(np.zeros(0, R.CLAIM_DTYPE), np.zeros(n + 1, np.uint32), np.zeros(n, np.int32),
                     np.zeros(0, R.CLAIM_DTYPE), np.zeros(1, np.uint32), np.zeros(0, np.int32), np.zeros(0, R.OUT_DTYPE),
                     max_victims=0)
