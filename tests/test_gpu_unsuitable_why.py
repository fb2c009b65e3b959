"""GPU suite: why each node is unsuitable (spec §17) through the C ABI — every output byte for byte the CPU oracle's
(tests/why_oracle.py), OK exactly where dra_unsuitable_batch sets its bit, the inventory untouched."""
import ctypes as C

import numpy as np
import pytest

from test_pod_capacity import R, _flat, problem

import why_oracle as Y
from oracle import oracle as O

pytestmark = pytest.mark.gpu
WIDTHS = {8: (0, 1, 2, 3, 8, 8), 16: (0, 1, 3, 8, 9, 16), 32: (0, 2, 8, 16, 17, 32)}


@pytest.fixture(scope="module")
def wctx(pkg):
    c = pkg.api.Context(device=0)
    yield c
    c.close()


def _check(ctx, g, off, t, claims, pod_off, cn=None, co=None, exhaustive=False, want=True, what="", attrs=None, sels=None):
    before = ctx.get_inventory()
    got = ctx.unsuitable_why(claims, pod_off, cn, co, exhaustive, want, want)
    ref = Y.why(before, off, t, claims, pod_off, cn, co, Y.F_EXHAUSTIVE if exhaustive else 0, attrs, sels)
    for name, x, y in zip(("pair_why", "pair_claim", "pod_why", "claim_blocks"), got, ref):
        if x is None:
            assert not want and name != "pair_why", name
        elif x.tobytes() != np.ascontiguousarray(y, x.dtype).reshape(x.shape).tobytes():
            bad = np.flatnonzero(x.ravel() != np.asarray(y).ravel())[:5]
            pytest.fail(f"{what}: {name} differs at {bad}: device {x.ravel()[bad]} oracle {np.asarray(y).ravel()[bad]}")
    bits = ctx.unsuitable(claims, pod_off, cn, co, O.F_EXHAUSTIVE if exhaustive else 0)
    n_pair = len(got[0])
    ok = np.unpackbits(np.asarray(bits, np.uint8), bitorder="little")[:n_pair].astype(bool)
    assert (ok == (got[0] == Y.ST_OK)).all(), what
    assert ctx.get_inventory().tobytes() == before.tobytes(), what
    return got


@pytest.mark.parametrize("width", [8, 16, 32])
def test_random_problems_at_each_lane_width(pkg, wctx, width):
    """The pod-capacity suite's generator (every claim kind, groups, invalid claims, 0 to 33 claims, strays, the dense
    form) at inventories whose widest node has <= 8, 9..16 and 17..32 GPUs, with and without the flag and the tallies."""
    reasons, forms = set(), set()
    for seed in range(12):
        g, off, t, c, pod_off, cands = problem(9000 * width + seed, WIDTHS[width], n_node=8, n_run=60)
        widest = int(np.diff(off.astype(np.int64)).max())
        if not width // 2 < widest <= width:
            g, off, t, c, pod_off, cands = problem(9000 * width + seed, WIDTHS[width] + (width,) * 6, n_node=8, n_run=60)
            widest = int(np.diff(off.astype(np.int64)).max())
        assert width // 2 < widest <= width, (width, seed, widest)
        wctx.set_table(t); wctx.set_inventory(g, off)
        cn, co = (None, None) if cands is None else _flat(cands)
        forms.add(cands is None)
        for exh, want in ((False, True), (True, True), (True, False), (False, False)):
            got = _check(wctx, g, off, t, c, pod_off, cn, co, exh, want, f"w{width} seed {seed} exh {exh}")
            reasons |= set(got[0].tolist())
    assert forms == {True, False}
    assert {Y.ST_OK, Y.ST_INVALID, Y.ST_NO_CAPACITY} <= reasons


def test_selectors_and_budget(pkg, wctx):
    """Claims with selectors (a MIG claim whose selector excludes every GPU offering its profile is BAD_PROFILE), and a
    pod whose search runs out of its 4096 descents (SEARCH_LIMIT at the level d)."""
    t = R.default_table()
    g = np.zeros(8, O.GPU_DTYPE)
    g["flags"], g["node"] = 1, np.repeat([0, 1], 4)
    off = np.array([0, 4, 8], np.uint32)
    attrs = np.zeros(8, R.ATTR_DTYPE)
    attrs["index"] = np.arange(8) % 4
    sels = np.stack([R.selector(("cmp", R.ATTR_INDEX, R.CMP_EQ, 0)), R.selector(("cmp", R.ATTR_INDEX, R.CMP_GT, 9))])
    wctx.set_table(t); wctx.set_inventory(g, off); wctx.set_gpu_attrs(attrs); wctx.set_selectors(sels)
    O.set_selectors(attrs, sels)
    try:
        small = int(np.flatnonzero(t[0]["size"] == 1)[0])
        c = np.zeros(40, O.CLAIM_DTYPE)
        c["kind"] = Y.KIND_MIG
        c["profile"] = small
        c[0]["mem_limit_mib"] = 1                     # index 0 only
        c[1]["mem_limit_mib"] = 2                     # no GPU
        c[2]["mem_limit_mib"] = 5                     # past the selectors: INVALID
        # pods: [0], [1], [2], then 30 one-slice claims on 4 GPUs of 7 slices (28 fit): the search gives up
        pod_off = np.array([0, 1, 2, 3, 33], np.uint32)
        for exh in (False, True):
            got = _check(wctx, g, off, t, c[:33], pod_off, exhaustive=exh, what=f"selectors exh {exh}",
                         attrs=attrs, sels=sels)
            assert got[0][2] == Y.ST_BAD_PROFILE and got[0][4] == Y.ST_INVALID
            if exh:                                   # 28 levels held at most: claim 3 + 28 blocks
                assert got[0][6] == Y.ST_SEARCH_LIMIT and got[1][6] == 31
    finally:
        O.set_selectors()
        wctx.set_selectors(None); wctx.set_gpu_attrs(None)


def test_call_errors_write_nothing(pkg, wctx):
    api = pkg.api
    g, off, t, c, pod_off, _ = problem(4242, n_node=4, n_run=10)
    wctx.set_table(t); wctx.set_inventory(g, off)
    lib, h = wctx._lib, wctx._h
    cc = np.ascontiguousarray(c, dtype=O.CLAIM_DTYPE)
    n_pod = len(pod_off) - 1
    why = np.full(n_pod * 4 + 16, 0xAB, np.uint8)
    blk = np.full(n_pod * 4 + 16, 0xABABABAB, np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    po = np.ascontiguousarray(pod_off, np.uint32)
    bad = po.copy(); bad[-1] += 1                   # not spanning the claims
    for args, flags in (((po, None, None), 0x80), ((bad, None, None), 0),
                        ((po, np.zeros(1, np.uint32), np.zeros(n_pod + 1, np.uint32) + 1), 0)):
        rc = lib.dra_unsuitable_why_batch(h, p(cc), len(cc), p(args[0]), n_pod, None if args[1] is None else p(args[1]),
                                          None if args[2] is None else p(args[2]), p(why), p(blk), None, None, flags)
        assert rc == api.E_INVAL
        assert (why == 0xAB).all() and (blk == 0xABABABAB).all()
    rc = lib.dra_unsuitable_why_batch(h, p(cc), len(cc), p(po), n_pod, None, None, None, None, None, None, 0)
    assert rc == api.E_INVAL                        # pairs to answer and no pair_why
    # the next call works and writes nothing past its outputs: tallies with pair_claim NULL, then every output
    pw = np.full((n_pod + 4) * Y.WHY_N, 0xCDCDCDCD, np.uint32)
    cb = np.full(len(cc) + 16, 0xCDCDCDCD, np.uint32)
    ref = Y.why(wctx.get_inventory(), off, t, cc, po)
    for claim_out in (None, blk):
        why[:] = 0xAB; blk[:] = 0xABABABAB; pw[:] = 0xCDCDCDCD; cb[:] = 0xCDCDCDCD
        rc = lib.dra_unsuitable_why_batch(h, p(cc), len(cc), p(po), n_pod, None, None, p(why),
                                          None if claim_out is None else p(claim_out), p(pw), p(cb), 0)
        assert rc == api.OK
        assert (why[:n_pod * 4] == ref[0]).all() and (why[n_pod * 4:] == 0xAB).all()
        if claim_out is None:
            assert (blk == 0xABABABAB).all()
        else:
            assert (blk[:n_pod * 4] == ref[1]).all() and (blk[n_pod * 4:] == 0xABABABAB).all()
        assert (pw[:n_pod * Y.WHY_N] == ref[2].ravel()).all() and (pw[n_pod * Y.WHY_N:] == 0xCDCDCDCD).all()
        assert (cb[:len(cc)] == ref[3]).all() and (cb[len(cc):] == 0xCDCDCDCD).all()
    assert "unsuitable_why" in wctx.last_chain()


def test_dense_form_of_2_32_pairs_is_refused(pkg, wctx):
    """65,536 empty pods against 65,536 nodes: n_pod * n_node = 2^32, refused before anything is written."""
    api = pkg.api
    n = 1 << 16
    g = np.zeros(n, O.GPU_DTYPE)
    g["node"] = np.arange(n)
    wctx.set_table(R.default_table()); wctx.set_inventory(g, np.arange(n + 1, dtype=np.uint32))
    po = np.zeros(n + 1, np.uint32)
    why = np.full(64, 0xAB, np.uint8)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    for flags in (0, O.F_EXHAUSTIVE):
        rc = wctx._lib.dra_unsuitable_why_batch(wctx._h, None, 0, p(po), n, None, None, p(why), None, None, None, flags)
        assert rc == api.E_INVAL and (why == 0xAB).all()


def test_cpp_driver_unsuitable_reasons_batch(pkg):
    """Driver::UnsuitableReasonsBatch of the C++ host layer (tests/cpp/why_test.cpp): the rendered messages."""
    import subprocess
    exe = pkg.build.build_cpp_why_test()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "why_test ok" in r.stdout
