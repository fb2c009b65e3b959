"""GPU suite: place pods (spec §13) through the C ABI — OutRecs, pod_node and the inventory bit-exact with the oracle."""
import os
import subprocess

import numpy as np
import pytest

from test_gpu_parity import _assert_same
from test_place_pods import NONE, _flat, placed_offsets

import place_oracle as P

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pctx(pkg):
    c = pkg.api.Context(device=0)
    yield c
    c.close()


def _random_cands(rng, n_pod, n_node, k, stray=True):
    nodes = rng.integers(0, n_node + (2 if stray else 0), size=n_pod * k).astype(np.uint32)
    return nodes, (np.arange(n_pod + 1) * k).astype(np.uint32)


def _check(pkg, ctx, oracle, w, pod_off, cn, co, flags, what, out_off=None, n_out=None, start=None):
    """One call on the device against the oracle from the same starting inventory (start: the device's live state)."""
    A = pkg.api
    g0 = w.gpus if start is None else start
    out, pod_node = ctx.place_pods(w.claims, pod_off, cn, co, out_off, n_out, flags)
    oflags = (oracle.F_EXHAUSTIVE if flags & A.F_EXHAUSTIVE else 0)
    ref, ref_node, inv = P.place_pods(g0, w.node_off, w.table, w.claims, pod_off, cn, co, out_off, n_out, oflags)
    _assert_same(out, ctx.get_inventory(), ref, inv, what)
    assert pod_node.tobytes() == ref_node.tobytes(), what
    assert "place" in ctx.last_chain()
    return out, pod_node


def test_two_pods_two_nodes(pkg, pctx, oracle):
    R = pkg.records
    g, off = R.make_inventory([1, 1], mig=True)
    pctx.set_table(R.default_table()); pctx.set_inventory(g, off)
    c = np.zeros(2, dtype=R.CLAIM_DTYPE)
    c["kind"], c["count"], c["profile"] = R.KIND_MIG, 1, R.GI_7_SLICE
    pod_off = np.array([0, 1, 2], np.uint32)
    assert pctx.unsuitable(c, pod_off, *_flat([[0, 1], [0, 1]]))[0] & 0xF == 0xF
    out, pod_node = pctx.place_pods(c, pod_off, *_flat([[0, 1], [0, 1]]))
    assert list(pod_node) == [0, 1] and list(out["status"]) == [0, 0] and list(out["gpu"]) == [0, 1]
    assert "place" in pctx.last_chain()
    pctx.set_inventory(g, off)
    out, pod_node = pctx.place_pods(c, pod_off)                            # dense form: the same
    assert list(pod_node) == [0, 1]


@pytest.mark.parametrize("seed,n_pod,n_node,width", [(0, 3000, 16, 8), (1, 2500, 9, 16), (2, 2000, 5, 32)])
def test_synthetic_pods(pkg, pctx, oracle, seed, n_pod, n_node, width):
    A = pkg.api
    w, pod_off = pkg.synth.pods(n_pod, n_node, seed, gpus_per_node=width)
    rng = np.random.default_rng(seed)
    n_pod = len(pod_off) - 1
    forms = {"dense": (None, None), "random8": _random_cands(rng, n_pod, n_node, 8),
             "same order": (np.tile(np.arange(n_node, dtype=np.uint32), n_pod), (np.arange(n_pod + 1) * n_node).astype(np.uint32))}
    for name, (cn, co) in forms.items():
        for flags in (0, A.F_EXHAUSTIVE):
            pctx.set_table(w.table); pctx.set_inventory(w.gpus, w.node_off)
            out, pod_node = _check(pkg, pctx, oracle, w, pod_off, cn, co, flags, f"{name} seed {seed} flags {flags}")
            assert (pod_node != NONE).any() and (pod_node == NONE).any()


def test_more_nodes_than_resident_warps(pkg, pctx, oracle):
    """10,000 nodes: every warp owns several nodes and cycles over them."""
    w, pod_off = pkg.synth.pods(30000, 10000, 5)
    rng = np.random.default_rng(5)
    cn, co = _random_cands(rng, len(pod_off) - 1, w.n_node, 8)
    for flags in (0, pkg.api.F_EXHAUSTIVE):
        pctx.set_table(w.table); pctx.set_inventory(w.gpus, w.node_off)
        _check(pkg, pctx, oracle, w, pod_off, cn, co, flags, f"10k nodes flags {flags}")
    w, pod_off = pkg.synth.pods(2000, 10000, 7)
    pctx.set_inventory(w.gpus, w.node_off)
    _check(pkg, pctx, oracle, w, pod_off, None, None, 0, "10k nodes dense")


def test_large_batch(pkg, pctx, oracle):
    """60,000 pods over 300 nodes."""
    w, pod_off = pkg.synth.pods(60000, 300, 4)
    rng = np.random.default_rng(4)
    cn, co = _random_cands(rng, len(pod_off) - 1, w.n_node, 8)
    for flags in (0, pkg.api.F_EXHAUSTIVE):
        pctx.set_table(w.table); pctx.set_inventory(w.gpus, w.node_off)
        _check(pkg, pctx, oracle, w, pod_off, cn, co, flags, f"60k pods flags {flags}")
    pctx.set_inventory(w.gpus, w.node_off)
    _check(pkg, pctx, oracle, w, pod_off, None, None, pkg.api.F_EXHAUSTIVE, "60k pods dense")


def test_fresh_inventory_and_continuation(pkg, pctx, oracle):
    A = pkg.api
    w, pod_off = pkg.synth.pods(4000, 24, 6)
    rng = np.random.default_rng(6)
    cn, co = _random_cands(rng, len(pod_off) - 1, w.n_node, 6)
    pctx.set_table(w.table); pctx.set_inventory(w.gpus, w.node_off)
    _check(pkg, pctx, oracle, w, pod_off, cn, co, A.F_EXHAUSTIVE, "first call")
    # a second call continues from the first call's inventory
    after = pctx.get_inventory()
    _check(pkg, pctx, oracle, w, pod_off, cn, co, 0, "second call", start=after)
    # DRA_F_FRESH_INVENTORY starts from the inventory as loaded, and its result becomes the live one
    _check(pkg, pctx, oracle, w, pod_off, cn, co, A.F_EXHAUSTIVE | A.F_FRESH_INVENTORY, "fresh")


def test_single_candidate_equals_allocate_pods(pkg, pctx, oracle):
    A = pkg.api
    for seed, width in ((0, 8), (1, 16), (2, 32)):
        w, pod_off = pkg.synth.pods(3000, 12, seed, gpus_per_node=width)
        first = w.claims["node"][pod_off[:-1]].astype(np.uint32)
        co = np.arange(len(pod_off), dtype=np.uint32)
        for flags in (0, A.F_EXHAUSTIVE):
            pctx.set_table(w.table); pctx.set_inventory(w.gpus, w.node_off)
            ref = pctx.allocate_pods(w.claims, pod_off, flags=flags)
            ref_inv = pctx.get_inventory()
            pctx.set_inventory(w.gpus, w.node_off)
            out, pod_node = pctx.place_pods(w.claims, pod_off, first, co, flags=flags)
            assert out.tobytes() == ref.tobytes() and pctx.get_inventory().tobytes() == ref_inv.tobytes()


def test_mixed_pods_with_selectors(pkg, pctx, oracle):
    """Pods cut out of the 'mixed' workload: every kind, counts > 1, malformed claims, ragged nodes, selectors."""
    R = pkg.records
    for seed in range(4):
        w = pkg.synth.mixed(3000, 23, 40 + seed, invalid=seed % 2 == 0)
        attrs, sels = (None, None)
        if seed >= 2:
            attrs, sels = pkg.synth.with_selectors(w, seed)
        rng = np.random.default_rng(seed)
        cuts = np.unique(np.concatenate([[0, w.n_claim], rng.integers(0, w.n_claim, 900)])).astype(np.uint32)
        out_off, n_out = placed_offsets(R, w.claims, w.n_node)
        cn, co = _random_cands(rng, len(cuts) - 1, w.n_node, 5)
        pctx.set_table(w.table); pctx.set_inventory(w.gpus, w.node_off)
        pctx.set_gpu_attrs(attrs); pctx.set_selectors(None if sels is None else sels.reshape(-1, R.SEL_MAX_INS))
        P.set_selectors(attrs, sels)
        try:
            for flags in (0, pkg.api.F_EXHAUSTIVE):
                pctx.reset_inventory()
                out, pod_node = _check(pkg, pctx, oracle, w, cuts, cn, co, flags, f"mixed seed {seed} flags {flags}",
                                       out_off, n_out)
                # Deallocate of the result, with the claims naming the node their pod went to, restores the inventory
                placed = w.claims.copy()
                for p in range(len(cuts) - 1):
                    placed["node"][cuts[p]: cuts[p + 1]] = pod_node[p] if pod_node[p] != NONE else 0
                pctx.deallocate(placed, out, out_off)
                assert pctx.get_inventory().tobytes() == w.gpus.tobytes()
        finally:
            P.set_selectors()
            pctx.set_selectors(None); pctx.set_gpu_attrs(None)


def test_bad_arguments_change_nothing(pkg, pctx):
    R = pkg.records
    g, off = R.make_inventory([1, 1], mig=True)
    pctx.set_table(R.default_table()); pctx.set_inventory(g, off)
    c = np.zeros(2, dtype=R.CLAIM_DTYPE)
    c["kind"], c["count"], c["profile"] = R.KIND_MIG, 1, R.GI_1_SLICE
    pod_off = np.array([0, 1, 2], np.uint32)
    bad = [dict(pod_off=pod_off, out_off=np.array([0, 1], np.uint32), n_out=1),
           dict(pod_off=np.array([0, 2, 1, 2], np.uint32)),
           dict(pod_off=np.array([0, 1], np.uint32)),
           dict(pod_off=pod_off, cand_nodes=np.array([0, 1], np.uint32), cand_off=np.array([0, 2, 1], np.uint32)),
           dict(pod_off=pod_off, flags=0x100)]
    for kw in bad:
        with pytest.raises(pkg.api.DraError) as e:
            pctx.place_pods(c, **kw)
        assert e.value.code == pkg.api.E_INVAL
        assert pctx.get_inventory().tobytes() == g.tobytes()


def test_place_on_arbitrary_problems(pkg, pctx, oracle):
    from hypothesis import HealthCheck, given, settings
    from hypothesis import strategies as st
    from test_place_pods import place_problems
    n_ex = int(os.environ.get("DRA_PROP_EXAMPLES", "0"))
    R = pkg.records

    @settings(max_examples=n_ex or 120, deadline=None, suppress_health_check=list(HealthCheck), derandomize=n_ex == 0, database=None)
    @given(place_problems(), st.booleans())
    def run(prob, exhaustive):
        g, off, t, c, pod_off, cands, dense = prob
        n_node = len(off) - 1
        flags, oflags = (pkg.api.F_EXHAUSTIVE, oracle.F_EXHAUSTIVE) if exhaustive else (0, 0)
        out_off, n_out = placed_offsets(R, c, n_node)
        cn, co = (None, None) if dense else _flat(cands)
        pctx.set_table(t); pctx.set_inventory(g, off)
        out, pod_node = pctx.place_pods(c, pod_off, cn, co, out_off, n_out, flags)
        ref, ref_node, inv = P.place_pods(g, off, t, c, pod_off, cn, co, out_off, n_out, oflags)
        _assert_same(out, pctx.get_inventory(), ref, inv, "arbitrary place")
        assert pod_node.tobytes() == ref_node.tobytes()

    run()


def test_cpp_driver_place_batch(pkg):
    """Driver::PlaceBatch of the C++ host layer (tests/cpp/place_test.cpp)."""
    exe = pkg.build.build_cpp_place_test()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "place_test ok" in r.stdout
