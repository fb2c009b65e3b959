"""GPU suite: why place pods put each pod where it did (spec §18) through the C ABI — every output byte for byte the CPU
oracle's (tests/place_why_oracle.py), and out, pod_node and the inventory byte for byte dra_place_pods_batch's from the
same start state."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from test_gpu_parity import _assert_same
from test_place_pods import placed_offsets
from test_pod_capacity import R, _flat, problem

import place_oracle as P
import place_why_oracle as PW
import why_oracle as Y
from oracle import oracle as O

pytestmark = pytest.mark.gpu
WIDTHS = {8: (0, 1, 2, 3, 8, 8), 16: (0, 1, 3, 8, 9, 16), 32: (0, 2, 8, 16, 17, 32)}
NONE = 0xFFFFFFFF


@pytest.fixture(scope="module")
def pctx(pkg):
    c = pkg.api.Context(device=0)
    yield c
    c.close()


def _check(pkg, ctx, g, off, t, c, pod_off, cn=None, co=None, oo=None, n_out=None, flags=0, want=True, what="",
           attrs=None, sels=None):
    """One reasons call from the pristine inventory g (with DRA_F_FRESH_INVENTORY, after a call that changed the live
    copy) against the oracle, then dra_place_pods_batch from the same start state."""
    A = pkg.api
    ctx.set_inventory(g, off)
    if flags & A.F_FRESH_INVENTORY and len(pod_off) > 1:
        ctx.place_pods(c, pod_off, cn, co, oo, n_out, 0)              # the live copy is no longer the start state
    got = ctx.place_pods_why(c, pod_off, cn, co, oo, n_out, flags, want, want)
    inv = ctx.get_inventory()
    assert "place_why" in ctx.last_chain() or len(pod_off) == 1
    ref = PW.place_why(g, off, t, c, pod_off, cn, co, oo, n_out, flags & Y.F_EXHAUSTIVE, attrs, sels)
    _assert_same(got[0], inv, ref[0], ref[2], what)
    assert got[1].tobytes() == ref[1].tobytes(), what
    for name, x, y in zip(("pair_why", "pair_claim", "pod_why", "claim_blocks"), got[2:], ref[3:]):
        if x is None:
            assert not want and name != "pair_why", name
        elif x.tobytes() != np.ascontiguousarray(y, x.dtype).reshape(x.shape).tobytes():
            bad = np.flatnonzero(x.ravel() != np.asarray(y).ravel())[:5]
            pytest.fail(f"{what}: {name} differs at {bad}: device {x.ravel()[bad]} oracle {np.asarray(y).ravel()[bad]}")
    # dra_place_pods_batch from the same start state
    ctx.set_inventory(g, off)
    if flags & A.F_FRESH_INVENTORY and len(pod_off) > 1:
        ctx.place_pods(c, pod_off, cn, co, oo, n_out, 0)
    out, pod_node = ctx.place_pods(c, pod_off, cn, co, oo, n_out, flags)
    assert out.tobytes() == got[0].tobytes() and pod_node.tobytes() == got[1].tobytes(), what
    assert ctx.get_inventory().tobytes() == inv.tobytes(), what
    return got


@pytest.mark.parametrize("width", [8, 16, 32])
def test_random_problems_at_each_lane_width(pkg, pctx, width):
    """The pod-capacity generator (every claim kind, groups, invalid claims, 0 to 33 claims, strays, duplicates, the
    dense form) at inventories whose widest node has <= 8, 9..16 and 17..32 GPUs; both flags, DRA_F_FRESH_INVENTORY,
    with and without out_off, pair_claim and the tallies."""
    A = pkg.api
    reasons, forms = set(), set()
    for seed in range(8):
        g, off, t, c, pod_off, cands = problem(7000 * width + seed, WIDTHS[width], n_node=8, n_run=60)
        widest = int(np.diff(off.astype(np.int64)).max())
        if not width // 2 < widest <= width:
            g, off, t, c, pod_off, cands = problem(7000 * width + seed, WIDTHS[width] + (width,) * 6, n_node=8, n_run=60)
            widest = int(np.diff(off.astype(np.int64)).max())
        assert width // 2 < widest <= width, (width, seed, widest)
        pctx.set_table(t)
        cn, co = (None, None) if cands is None else _flat(cands)
        forms.add(cands is None)
        oo, n_out = placed_offsets(R, c, len(off) - 1)
        for k, (flags, want, with_off) in enumerate(((0, True, False), (A.F_EXHAUSTIVE, True, True),
                                                     (A.F_EXHAUSTIVE | A.F_FRESH_INVENTORY, False, False),
                                                     (A.F_FRESH_INVENTORY, True, True))):
            got = _check(pkg, pctx, g, off, t, c, pod_off, cn, co, oo if with_off else None, n_out if with_off else None,
                         flags, want, f"w{width} seed {seed} flags {flags} off {with_off}")
            reasons |= set(got[2].tolist())
            if not flags & A.F_EXHAUSTIVE:
                assert Y.ST_SEARCH_LIMIT not in got[2].tolist()
    assert forms == {True, False}
    assert {Y.ST_OK, Y.ST_INVALID, Y.ST_NO_CAPACITY} <= reasons


@pytest.mark.parametrize("seed", [3, 11])
def test_prefix_property_on_the_device(pkg, pctx, seed):
    """Consequence 2 on the device: with DRA_F_EXHAUSTIVE, row p equals dra_unsuitable_why_batch with the flag for pod p
    on the inventory dra_place_pods_batch leaves after pods 0..p-1 (slots with out_off: the same validity)."""
    A = pkg.api
    g, off, t, c, pod_off, cands = problem(seed, n_node=6, n_run=40)
    pctx.set_table(t)
    cn, co = (None, None) if cands is None else _flat(cands)
    oo, n_out = placed_offsets(R, c, len(off) - 1)
    got = _check(pkg, pctx, g, off, t, c, pod_off, cn, co, oo, n_out, A.F_EXHAUSTIVE, True, f"prefix seed {seed}")
    n_pod, n_node = len(pod_off) - 1, len(off) - 1
    k0 = 0
    for p in range(n_pod):
        c0, c1 = int(pod_off[p]), int(pod_off[p + 1])
        k1 = k0 + (n_node if co is None else int(co[p + 1] - co[p]))
        if p % 3 == 0 or p == n_pod - 1:
            pctx.set_inventory(g, off)
            if p:
                pctx.place_pods(c[:c0], pod_off[:p + 1], cn, None if co is None else co[:p + 1], oo[:c0], n_out,
                                A.F_EXHAUSTIVE)
            one_cn = None if co is None else cn[co[p]:co[p + 1]]
            one_co = None if co is None else np.array([0, k1 - k0], np.uint32)
            row = pctx.unsuitable_why(c[c0:c1], np.array([0, c1 - c0], np.uint32), one_cn, one_co, True)
            assert row[0].tobytes() == got[2][k0:k1].tobytes(), p
            rc = row[1].copy()
            rc[rc != Y.WHY_CLAIM_NONE] += c0
            assert rc.tobytes() == got[3][k0:k1].tobytes(), p
        k0 = k1


def _mig_pods(t, profiles_per_pod):
    claims, pod_off = [], [0]
    for pod in profiles_per_pod:
        for prof in pod:
            x = np.zeros(1, O.CLAIM_DTYPE)
            x["kind"], x["count"], x["profile"] = Y.KIND_MIG, 1, prof
            claims.append(x)
        pod_off.append(pod_off[-1] + len(pod))
    return (np.concatenate(claims) if claims else np.zeros(0, O.CLAIM_DTYPE)), np.array(pod_off, np.uint32)


def test_edges(pkg, pctx):
    """Candidates naming no node, a pod with no usable candidate, empty pods, a 33-claim pod, a GPU claim of count 2
    without out_off, the chosen node listed again later, a node listed twice before the pod fits, and a pod that lost
    the last 3g slot to the pod before it."""
    A = pkg.api
    t = R.default_table()
    pctx.set_table(t)
    g, off = R.make_inventory([1, 1], mig=True)
    g["busy"][0] = 0b1111                                  # node 0: one 3g slot left; node 1 free
    c, pod_off = _mig_pods(t, [[R.GI_3_SLICE], [R.GI_3_SLICE], [R.GI_7_SLICE], [], [R.GI_1_SLICE] * 33,
                               [R.GI_7_SLICE], [R.GI_1_SLICE]])
    gpu = np.zeros(1, O.CLAIM_DTYPE)
    gpu["kind"], gpu["count"] = Y.KIND_GPU, 2
    c = np.concatenate([c, gpu])
    pod_off = np.append(pod_off, pod_off[-1] + 1).astype(np.uint32)
    cands = [[0, 1], [0, 9, 0, 1, 1], [9, 99], [0, 1], [0, 7], [1, 0, 0], [0, 0, 1, 0], [0, 1]]
    cn, co = _flat(cands)
    for flags in (0, A.F_EXHAUSTIVE):
        got = _check(pkg, pctx, g, off, t, c, pod_off, cn, co, flags=flags, what=f"edges {flags}")
        why, claim = got[2].tolist(), got[3].tolist()
        node = got[1].tolist()
        assert node[:3] == [0, 1, NONE]
        assert why[0:2] == [Y.ST_OK, Y.ST_OK]                       # pod 0 takes node 0's last 3g slot; dry run at 1
        assert why[2:7] == [Y.ST_NO_CAPACITY, Y.WHY_NO_NODE, Y.ST_NO_CAPACITY, Y.ST_OK, Y.ST_OK]
        assert claim[2] == 1 and claim[4] == 1
        assert why[7:9] == [Y.WHY_NO_NODE, Y.WHY_NO_NODE]          # no usable candidate
        assert why[9:11] == [Y.ST_OK, Y.ST_OK] and node[3] == NONE  # empty pod
        assert why[11:13] == [Y.ST_INVALID, Y.WHY_NO_NODE] and claim[11] == Y.WHY_CLAIM_NONE
        # pod 5 (7g): node 1 is taken by pod 1's 3g, node 0 by pod 0: nowhere; listed twice, answered twice
        assert node[5] == NONE and why[13:16] == [Y.ST_NO_CAPACITY] * 3
        # pod 6 (1g): node 0 full, node 1 has room; node 0 listed again after
        assert node[6] == 1 and why[16:20] == [Y.ST_NO_CAPACITY, Y.ST_NO_CAPACITY, Y.ST_OK, Y.ST_NO_CAPACITY]
        assert why[20:22] == [Y.ST_INVALID, Y.ST_INVALID] and claim[20] == len(c) - 1   # count 2 without out_off
    oo, n_out = placed_offsets(R, c, 2)
    got = _check(pkg, pctx, g, off, t, c, pod_off, cn, co, oo, n_out, A.F_EXHAUSTIVE, what="edges with out_off")
    assert got[2].tolist()[20:22] == [Y.ST_NO_CAPACITY, Y.ST_NO_CAPACITY]   # valid with out_off; no non-MIG GPU


def test_chosen_node_listed_again_is_ok(pkg, pctx):
    """A later pair naming the chosen node is OK: the node as the pod met it, not after its own placement."""
    t = R.default_table()
    pctx.set_table(t)
    g, off = R.make_inventory([1, 1], mig=True)
    c, pod_off = _mig_pods(t, [[R.GI_7_SLICE]])
    cn, co = _flat([[0, 1, 0]])
    for flags in (0, pkg.api.F_EXHAUSTIVE):
        got = _check(pkg, pctx, g, off, t, c, pod_off, cn, co, flags=flags, what="chosen again")
        assert got[1].tolist() == [0] and got[2].tolist() == [Y.ST_OK] * 3
    got = _check(pkg, pctx, g, off, t, c, pod_off, what="dense")
    assert got[1].tolist() == [0] and got[2].tolist() == [Y.ST_OK, Y.ST_OK]


def test_selectors_and_search_budget(pkg, pctx):
    """Selectors (BAD_PROFILE where the selector excludes every GPU, INVALID past the selectors), and a pod whose search
    runs out of its 4096 descents: SEARCH_LIMIT with the flag, POD at the first level with no choice without it."""
    A = pkg.api
    t = R.default_table()
    g = np.zeros(8, O.GPU_DTYPE)
    g["flags"], g["node"] = 1, np.repeat([0, 1], 4)
    off = np.array([0, 4, 8], np.uint32)
    attrs = np.zeros(8, R.ATTR_DTYPE)
    attrs["index"] = np.arange(8) % 4
    sels = np.stack([R.selector(("cmp", R.ATTR_INDEX, R.CMP_EQ, 0)), R.selector(("cmp", R.ATTR_INDEX, R.CMP_GT, 9))])
    pctx.set_table(t); pctx.set_gpu_attrs(attrs); pctx.set_selectors(sels)
    O.set_selectors(attrs, sels); P.set_selectors(attrs, sels)
    try:
        small = int(np.flatnonzero(t[0]["size"] == 1)[0])
        c = np.zeros(34, O.CLAIM_DTYPE)
        c["kind"] = Y.KIND_MIG
        c["profile"] = small
        c[0]["mem_limit_mib"] = 1                     # index 0 only
        c[1]["mem_limit_mib"] = 2                     # no GPU
        c[2]["mem_limit_mib"] = 5                     # past the selectors: INVALID
        # pods: [0], [1], [2], then 30 one-slice claims on 4 GPUs of 7 slices (28 fit): the search gives up; then [33]
        pod_off = np.array([0, 1, 2, 3, 33, 34], np.uint32)
        for flags in (0, A.F_EXHAUSTIVE):
            got = _check(pkg, pctx, g, off, t, c, pod_off, flags=flags, what=f"selectors {flags}", attrs=attrs, sels=sels)
            why = got[2].reshape(5, 2)
            assert why[1].tolist() == [Y.ST_BAD_PROFILE] * 2 and why[2].tolist() == [Y.ST_INVALID] * 2
            if flags:
                assert why[3].tolist() == [Y.ST_SEARCH_LIMIT] * 2
            else:
                assert Y.ST_SEARCH_LIMIT not in got[2].tolist() and why[3].tolist() == [Y.ST_POD] * 2
    finally:
        O.set_selectors(); P.set_selectors()
        pctx.set_selectors(None); pctx.set_gpu_attrs(None)


def test_call_errors_write_nothing(pkg, pctx):
    """Every refusal writes nothing (outputs keep their sentinel fill, the inventory is unchanged), and the next call
    works."""
    api = pkg.api
    g, off, t, c, pod_off, _ = problem(4242, n_node=4, n_run=10)
    pctx.set_table(t); pctx.set_inventory(g, off)
    before = pctx.get_inventory()
    lib, h = pctx._lib, pctx._h
    cc = np.ascontiguousarray(c, dtype=O.CLAIM_DTYPE)
    n_pod = len(pod_off) - 1
    n_out = len(cc) + 8
    out = np.zeros(n_out, O.OUT_DTYPE)
    node = np.full(n_pod + 4, 0xABABABAB, np.uint32)
    why = np.full(n_pod * 4 + 16, 0xAB, np.uint8)
    blk = np.full(n_pod * 4 + 16, 0xABABABAB, np.uint32)
    pw = np.full((n_pod + 4) * Y.WHY_N, 0xCDCDCDCD, np.uint32)
    cb = np.full(len(cc) + 16, 0xCDCDCDCD, np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    po = np.ascontiguousarray(pod_off, np.uint32)
    bad = po.copy(); bad[-1] += 1                   # not spanning the claims
    nonmono = np.zeros(n_pod + 1, np.uint32) + 1   # cand_off not from 0

    def sentinels():
        out.view(np.uint8)[:] = 0xEE
        return out.tobytes()

    for args, flags, with_why in (((po, None, None), 0x80, True), ((bad, None, None), 0, True),
                                  ((po, np.zeros(1, np.uint32), nonmono), 0, True), ((po, None, None), 0, False)):
        o0 = sentinels()
        rc = lib.dra_place_pods_why_batch(h, p(cc), len(cc), p(args[0]), n_pod, None if args[1] is None else p(args[1]),
                                          None if args[2] is None else p(args[2]), None, p(out), n_out, p(node),
                                          p(why) if with_why else None, p(blk), p(pw), p(cb), flags)
        assert rc == api.E_INVAL
        assert out.tobytes() == o0 and (node == 0xABABABAB).all() and (why == 0xAB).all()
        assert (blk == 0xABABABAB).all() and (pw == 0xCDCDCDCD).all() and (cb == 0xCDCDCDCD).all()
        assert pctx.get_inventory().tobytes() == before.tobytes()
    # the next call works and writes nothing past its outputs
    ref = PW.place_why(before, off, t, cc, po)
    rc = lib.dra_place_pods_why_batch(h, p(cc), len(cc), p(po), n_pod, None, None, None, p(out), n_out, p(node),
                                      p(why), None, p(pw), p(cb), 0)
    assert rc == api.OK
    assert (node[:n_pod] == ref[1]).all() and (node[n_pod:] == 0xABABABAB).all()
    assert (why[:n_pod * 4] == ref[3]).all() and (why[n_pod * 4:] == 0xAB).all() and (blk == 0xABABABAB).all()
    assert (pw[:n_pod * Y.WHY_N] == ref[5].ravel()).all() and (pw[n_pod * Y.WHY_N:] == 0xCDCDCDCD).all()
    assert (cb[:len(cc)] == ref[6]).all() and (cb[len(cc):] == 0xCDCDCDCD).all()
    assert "place_why" in pctx.last_chain()


def test_dense_form_of_2_32_pairs_is_refused(pkg, pctx):
    """65,536 empty pods against 65,536 nodes: n_pod * n_node = 2^32, refused before anything is written."""
    api = pkg.api
    n = 1 << 16
    g = np.zeros(n, O.GPU_DTYPE)
    g["node"] = np.arange(n)
    pctx.set_table(R.default_table()); pctx.set_inventory(g, np.arange(n + 1, dtype=np.uint32))
    po = np.zeros(n + 1, np.uint32)
    node = np.full(n, 0xABABABAB, np.uint32)
    why = np.full(64, 0xAB, np.uint8)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    for flags in (0, O.F_EXHAUSTIVE):
        rc = pctx._lib.dra_place_pods_why_batch(pctx._h, None, 0, p(po), n, None, None, None, None, 0, p(node), p(why),
                                                None, None, None, flags)
        assert rc == api.E_INVAL and (why == 0xAB).all() and (node == 0xABABABAB).all()
    # one pod fewer is answered
    rc = pctx._lib.dra_place_pods_why_batch(pctx._h, None, 0, p(po), 1, None, None, None, None, 0, p(node),
                                            p(np.zeros(n, np.uint8)), None, None, None, 0)
    assert rc == api.OK and node[0] == NONE


def test_cpp_driver_place_batch_with_reasons(pkg):
    """Driver::PlaceBatchWithReasons of the C++ host layer (tests/cpp/place_why_test.cpp)."""
    exe = pkg.build.build_cpp_place_why_test()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "place_why_test ok" in r.stdout
