"""GPU suite: pod capacity (spec §16) at its edges.  Every call goes through the raw ABI on sentinel-filled outputs with
slack, and every time: each output is byte for byte capacity_oracle.capacity's answer, nothing is written past an output
(nor into one that was not asked for), and the inventory, live and pristine, is unchanged.

- rounds of the pair walk: k_pods_capacity takes G = 32 / W pairs per fetch from a counter, and its grid is at most
  SMs x 8 CTAs of 8 warps, so one round of the grid is R = SMs x 8 x 8 x G pairs; walks of 1 pair to 3R + r, with the
  pairs of every fetch mixing costs from one evaluation to 65,535;
- structural limits: 32-claim pods placed many times with backtracks at position 16, 33 claims, GPU claims as wide as
  their node, zero-GPU nodes at both ends, MPS shares bounded by memory, full share counts, SEARCH_LIMIT after copies;
- 64-bit sums: pod_total above 2^32 in k_pods_capacity_sum and in the sharded merge;
- one context reused across growing and shrinking calls, widths, node counts and the other pair calls;
- walks near 2^32 pairs, which end after one pass (a 32-bit walk index once wrapped there and never stopped).

The small problems are built by the functions below; tests/test_pod_capacity_edges.py checks them on the CPU."""
import ctypes as C
import importlib

import numpy as np
import pytest

from test_pod_search_fixtures import G1, G4, claims as fx_claims, fixture_table, node as fx_node

import capacity_oracle as K

pytestmark = pytest.mark.gpu
R = importlib.import_module("k8s-dra-driver_b200").records
NONE = 0xFFFFFFFF
SENT = 0xA5
SLACK = 16
NAMES = ("pair_copies", "pair_stop", "pod_total", "pod_nodes")
DTYPES = (np.uint16, np.uint8, np.uint64, np.uint32)
EXH = K.F_EXHAUSTIVE


# ---- problems (pure numpy: the CPU suite checks them against capacity_naive) -------------------------------------------
def _claim(kind, count=1, profile=0, mem=0, group=0):
    c = np.zeros(1, R.CLAIM_DTYPE)
    c["kind"], c["count"], c["profile"], c["mem_limit_mib"], c["group"] = kind, count, profile, mem, group
    return c


def _pods(pods):
    """(claims, pod_off) of a list of claim arrays"""
    po = np.zeros(len(pods) + 1, np.uint32)
    po[1:] = np.cumsum([len(p) for p in pods])
    c = np.concatenate(pods) if po[-1] else np.zeros(0, R.CLAIM_DTYPE)
    return c, po


def _mig_pod(profiles):
    c = np.zeros(len(profiles), R.CLAIM_DTYPE)
    c["kind"], c["count"], c["profile"] = R.KIND_MIG, 1, profiles
    return c


# The palette of the walk problems (A100 table): what each costs on which node
SHARED = _claim(R.KIND_SHARED)                                   # time-slicing: up to 65,535 copies on a fresh GPU
EMPTY = np.zeros(0, R.CLAIM_DTYPE)                               # max_copies, ST_OK, no evaluation
POD33 = _mig_pod([R.GI_1_SLICE] * 33)                            # INVALID: more than 32 claims
BADGPU = _claim(R.KIND_GPU, 33)                                  # INVALID: count 33
LIMIT = _mig_pod([R.GI_1_SLICE] * 7 + [R.GI_7_SLICE])            # exhaustive: copies, then SEARCH_LIMIT on 3 GPUs
SMALL = _mig_pod([R.GI_1_SLICE, R.GI_2_SLICE])
ONEGPU = _claim(R.KIND_GPU, 1)
PALETTE = (SHARED, EMPTY, POD33, BADGPU, LIMIT, SMALL, ONEGPU)


def walk_inventory(width, n_node=6):
    """n_node nodes cycling through: a fresh plain GPU (time-slicing to 65,535), `width` MIG GPUs, a plain GPU with
    65,000 shares taken, 3 MIG GPUs (LIMIT: one copy, then SEARCH_LIMIT), no GPU, 2 MIG GPUs"""
    kinds = [(1, False, 0), (width, True, 0), (1, False, 65000), (3, True, 0), (0, True, 0), (2, True, 0)]
    per = [kinds[i % 6] for i in range(n_node)]
    g, off = R.make_inventory([k[0] for k in per], mig=True)
    for i, (n, mig, share) in enumerate(per):
        g["flags"][off[i]:off[i + 1]] = R.GPU_MIG_ENABLED if mig else 0
        g["share_cnt"][off[i]:off[i + 1]] = share
    return g, off


def walk_problem(width, n_walk, form, heavy_every=None):
    """A walk of exactly n_walk pairs.  Candidates: pod k of n_walk one-candidate pods is PALETTE[k % 7] (SHARED on the
    fresh GPU only in the first and last 64 pairs and every heavy_every-th, else on the MIG node; a stray in every 9th
    pair), so every fetch of G pairs mixes evaluations from 0 to 65,535.  Dense: n_pod x n_node = n_walk, n_node the
    smallest divisor of n_walk in [6, 64], else n_walk nodes and one pod.  Returns (g, off, claims, pod_off, cn, co)."""
    if form == "dense":
        n_node = next((d for d in range(6, 65) if n_walk % d == 0), n_walk)
        g, off = walk_inventory(width, n_node)
        n_pod = n_walk // n_node
        c, po = _pods([PALETTE[(p + 5) % 7] for p in range(n_pod)])
        return g, off, c, po, None, None
    g, off = walk_inventory(width)
    k = np.arange(n_walk)
    kind = k % 7
    node = (k // 7) % 6
    heavy = (k < 64) | (k >= n_walk - 64) | ((k % heavy_every == 0) if heavy_every else False)
    node = np.where(kind == 0, np.where(heavy, 0, 1), node)
    node = np.where(k % 9 == 8, np.where(k % 2 == 0, 6, NONE), node)
    pods = [PALETTE[i] for i in kind]
    c, po = _pods(pods)
    return g, off, c, po, node.astype(np.uint32), np.arange(n_walk + 1, dtype=np.uint32)


def deep_problems():
    """32-claim MIG pods on 32-GPU nodes of the 16-slice fixture table (W = 32): 16 x 1g, a grouped {1g, 4g}, 14 x 1g.
    First fit places none; the exhaustive search places 12 copies, every copy but a few backtracking at position 16,
    and on the first node stops with SEARCH_LIMIT after them.  A third node is half full."""
    busy = [[0x0000, 0x0100] * 16, [0x0100] * 32, [0x0100, 0x0000] * 8 + [0xFFFF] * 16]
    g = np.concatenate([fx_node(b) for b in busy])
    off = np.array([0, 32, 64, 96], np.uint32)
    g["node"] = np.repeat(np.arange(3), 32)
    deep = fx_claims(*[("mig", G1)] * 16 + [("mig", G1, 5), ("mig", G4, 5)] + [("mig", G1)] * 14)
    c, po = _pods([deep, _mig_pod([G1] * 32), deep[:16], fx_claims(*[("mig", G1)] * 33)])
    return g, off, fixture_table(), c, po


def structural_problems(width):
    """(gpus, node_off, claims, pod_off) on the A100 table, widest node `width`: GPU claims as wide as each node
    and of counts 32 and 33, zero-GPU nodes first and last, MPS shares bounded by memory, share counts at 65,534 / 65,535,
    a plain GPU UNAVAILABLE, LIMIT on 3 and 5 MIG GPUs (one and two copies, then SEARCH_LIMIT)."""
    widths = [w for w in (1, 8, 9, 16, 17, 32) if w <= width]
    # nodes: none | plain GPUs of each width | 1 (65,534 shares) | 1 (65,535) | 1 UNAVAILABLE | 2 (40960 / 12000 MiB
    # free) | MIG 3 | MIG 5 | MIG width | none
    sizes = [0] + widths + [1, 1, 1, 2, 3, 5, width, 0]
    g, off = R.make_inventory(sizes, mig=False)
    n = len(widths) + 1
    g["share_cnt"][off[n]], g["share_cnt"][off[n + 1]] = 65534, 65535
    g["flags"][off[n + 2]] = R.GPU_UNAVAILABLE
    g["mem_free_mib"][off[n + 3]:off[n + 4]] = [40960, 12000]
    g["flags"][off[n + 4]:off[n + 7]] = R.GPU_MIG_ENABLED
    pods = [_claim(R.KIND_GPU, w) for w in widths + [32, 33]]
    pods += [_claim(R.KIND_SHARED, mem=5000), _claim(R.KIND_SHARED, mem=40960), _claim(R.KIND_SHARED, mem=40961),
             SHARED, np.concatenate([SHARED, _claim(R.KIND_SHARED, mem=3000)]), LIMIT, EMPTY,
             np.concatenate([_claim(R.KIND_GPU, 1)] * 32)]
    c, po = _pods(pods)
    return g, off, c, po


# ---- the raw call ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cctx(pkg):
    c = pkg.api.Context(device=0)
    yield c
    c.close()


def _p(x):
    return None if x is None else x.ctypes.data_as(C.c_void_p)


def raw(ctx, c, po, cn=None, co=None, mc=64, fl=0, want=(True, True, True)):
    """dra_pod_capacity_batch on outputs filled with SENT and SLACK bytes past their ends; returns the four outputs
    (None where not asked for) after checking the slack and the outputs not asked for"""
    n_pod = len(po) - 1
    n_pair = n_pod * ctx.n_node if co is None else int(co[-1])
    sizes = [n_pair * 2, n_pair, n_pod * 8, n_pod * 4]
    # an output not asked for is a small sentinel buffer that is not passed: a write to it would be a wild write
    bufs = [np.full((s if i == 0 or want[i - 1] else 0) + SLACK, SENT, np.uint8) for i, s in enumerate(sizes)]
    args = [bufs[0]] + [b if w else None for b, w in zip(bufs[1:], want)]
    c = np.ascontiguousarray(c, R.CLAIM_DTYPE)
    keep = [np.ascontiguousarray(x, np.uint32) if x is not None else None for x in (po, cn, co)]
    ctx._check(ctx._lib.dra_pod_capacity_batch(ctx._h, _p(c) if len(c) else None, len(c), _p(keep[0]), n_pod, _p(keep[1]),
                                               _p(keep[2]), mc, *[_p(x) for x in args], fl))
    out = []
    for i, (b, s) in enumerate(zip(bufs, sizes)):
        assert (b[s:] == SENT).all(), f"written past {NAMES[i]}"
        if i and not want[i - 1]:
            assert (b == SENT).all(), f"{NAMES[i]} written without being asked for"
            out.append(None)
        else:
            out.append(b[:s].view(DTYPES[i]))
    return out


def same(got, ref, what):
    for name, x, y in zip(NAMES, got, ref):
        if x is not None and x.tobytes() != y.tobytes():
            bad = np.flatnonzero(x != y)[:5]
            pytest.fail(f"{what}: {name} differs at {bad}: device {x[bad]} oracle {y[bad]}")


def check(ctx, g, off, t, c, po, cn=None, co=None, mc=64, fl=0, want=(True, True, True), what="", live=None):
    """one call against the oracle on the live inventory `live` (default g, the loaded one); the live inventory is
    unchanged, and the pristine one too when live is the loaded one"""
    live = g if live is None else live
    got = raw(ctx, c, po, cn, co, mc, fl, want)
    ref = K.capacity(live, off, t, c, po, cn, co, mc, fl)
    same(got, ref, what)
    assert ctx.get_inventory().tobytes() == live.tobytes(), f"{what}: live inventory changed"
    if live is g:
        ctx.reset_inventory()
        assert ctx.get_inventory().tobytes() == g.tobytes(), f"{what}: pristine inventory changed"
    return ref


def _every_node(n_pod, n_node):
    """the dense form's pairs as candidate lists (the CPU oracle of UnsuitableNodes takes lists only)"""
    return (np.tile(np.arange(n_node, dtype=np.uint32), max(n_pod, 1))[:max(n_pod * n_node, 1)],
            (np.arange(n_pod + 1) * n_node).astype(np.uint32))


def n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- 1. rounds of the walk ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("width", [8, 16, 32])
def test_walks_around_the_rounds_of_the_grid(pkg, cctx, width):
    G = 32 // width
    rnd = n_sm() * 8 * 8 * G
    r = G + 1 if G > 1 else 7                          # not a multiple of G (W = 32: G = 1, every r is)
    t = R.default_table()
    seen = set()
    for n_walk in sorted({1, max(G - 1, 1), G + 1, 8 * G - 1, 8 * G + 1, rnd - 1, rnd, rnd + 1, 3 * rnd + r}):
        for form in ("cands", "dense"):
            g, off, c, po, cn, co = walk_problem(width, n_walk, form, heavy_every=4099)
            cctx.set_table(t); cctx.set_inventory(g, off)
            assert max(np.diff(off.astype(np.int64))) == width or n_walk < 2
            mc = 65535 if form == "cands" else 40
            for fl, want in ((0, (True, True, True)), (EXH, (True, False, True)), (EXH, (False, True, False))):
                ref = check(cctx, g, off, t, c, po, cn, co, mc, fl, want, f"w{width} n_walk {n_walk} {form} f{fl}")
                seen |= {(int(s), int(x) > 0) for s, x in zip(ref[1], ref[0])}
    assert {(K.ST_OK, True), (K.ST_POD, False), (K.ST_INVALID, False), (K.ST_SEARCH_LIMIT, True), (K.ST_POD, True)} <= seen


# ---- 2. structural limits ----------------------------------------------------------------------------------------------
def test_32_claim_pods_placed_many_times(pkg, cctx):
    g, off, t, c, po = deep_problems()
    cctx.set_table(t); cctx.set_inventory(g, off)
    rng = np.random.default_rng(1)
    cn = rng.integers(0, 4, 40).astype(np.uint32)
    co = np.array([0, 10, 20, 30, 40], np.uint32)
    for fl in (0, EXH):
        for mc in (1, 2, 11, 12, 13, 65535):
            copies, stop, _, _ = check(cctx, g, off, t, c, po, mc=mc, fl=fl, what=f"deep dense f{fl} mc {mc}")
            check(cctx, g, off, t, c, po, cn, co, mc, fl, what=f"deep cands f{fl} mc {mc}")
            if fl and mc == 65535:
                assert copies[0] == 12 and stop[0] == K.ST_SEARCH_LIMIT and copies[1] == 12 and stop[1] == K.ST_POD
                assert (stop[9:12] == K.ST_INVALID).all()
            if not fl:
                assert copies[0] == 0 and copies[3] > 0           # first fit places no deep pod but the 16-claim prefix


@pytest.mark.parametrize("width", [8, 16, 32])
def test_structural_limits_at_each_width(pkg, cctx, width):
    g, off, c, po = structural_problems(width)
    t = R.default_table()
    cctx.set_table(t); cctx.set_inventory(g, off)
    n_node = len(off) - 1
    rng = np.random.default_rng(width)
    lists = [list(rng.integers(0, n_node + 1, 9)) + [0, n_node - 1, NONE] for _ in range(len(po) - 1)]
    lists[0] = []
    cn = np.array([x for li in lists for x in li], np.uint32)
    co = np.zeros(len(lists) + 1, np.uint32)
    co[1:] = np.cumsum([len(x) for x in lists])
    stops = set()
    for fl in (0, EXH):
        for mc in (1, 8, 65535):
            ref = check(cctx, g, off, t, c, po, mc=mc, fl=fl, what=f"w{width} dense f{fl} mc {mc}")
            stops |= {(int(s), int(x) > 0) for s, x in zip(ref[1], ref[0])}
            check(cctx, g, off, t, c, po, cn, co, mc, fl, want=(True, True, False), what=f"w{width} cands f{fl} mc {mc}")
    assert (K.ST_SEARCH_LIMIT, True) in stops and (K.ST_INVALID, False) in stops and (K.ST_OK, True) in stops


# ---- 3. 64-bit sums ----------------------------------------------------------------------------------------------------
SUM_LISTS = (65538, 32 * 65537 + 33)


def sum_problem(n_list, n_node):
    """one empty pod with n_list candidates (every node, cyclically) and a one-claim pod with three: pod_total of the
    first is 65,535 x n_list > 2^32"""
    c, po = _pods([EMPTY, _mig_pod([R.GI_1_SLICE])])
    cn = np.concatenate([np.arange(n_list) % n_node, [0, n_node, 1]]).astype(np.uint32)
    return c, po, cn, np.array([0, n_list, n_list + 3], np.uint32)


def test_sums_past_two_to_the_32(pkg, cctx):
    t = R.default_table()
    g, off = R.make_inventory([1] * 65538, mig=True)
    cctx.set_table(t); cctx.set_inventory(g, off)
    for n_list in SUM_LISTS:
        c, po, cn, co = sum_problem(n_list, 65538)
        _, _, total, nodes = check(cctx, g, off, t, c, po, cn, co, 65535, 0, what=f"{n_list} candidates")
        assert int(total[0]) == 65535 * n_list > 1 << 32 and int(nodes[0]) == n_list and int(total[1]) == 14
    c, po = _pods([EMPTY])
    _, _, total, nodes = check(cctx, g, off, t, c, po, mc=65535, what="dense over 65,538 nodes")
    assert int(total[0]) == 65535 * 65538 and int(nodes[0]) == 65538


@pytest.mark.parametrize("world", [1, 2])
def test_sharded_sums_past_two_to_the_32(pkg, world):
    import shard_world as S
    t = R.default_table()
    n_node = 65538
    g, off = R.make_inventory([1] * n_node, mig=True)
    W = S.World(pkg, t, off, g, world, [0, 40000, n_node][:: (1 if world == 2 else 2)], capacity=2_200_000)
    try:
        for n_list in SUM_LISTS:
            c, po, cn, co = sum_problem(n_list, n_node)
            ref = K.capacity(g, off, t, c, po, cn, co, 65535)
            assert int(ref[2][0]) > 1 << 32
            for r, got in enumerate(S.capacity(W, c, po, (cn, co), 65535)):
                S.same(got, ref, S.CAPACITY_NAMES, f"world {world} rank {r} {n_list}")
        c, po = _pods([EMPTY, ONEGPU])
        ref = K.capacity(g, off, t, c, po, None, None, 65535)
        for r, got in enumerate(S.capacity(W, c, po, None, 65535)):
            S.same(got, ref, S.CAPACITY_NAMES, f"world {world} rank {r} dense")
        assert all(ctx.get_inventory().tobytes() == g.tobytes() for ctx in W.ctxs)
    finally:
        W.close()


# ---- 4. one context, many calls ----------------------------------------------------------------------------------------
def test_context_reused_across_calls(pkg, cctx):
    """Growing and shrinking n_pod and n_pair, both forms, every optional output on and off, inventories of W = 8 -> 32
    -> 8 and different node counts, with UnsuitableNodes, preemption and place-pods calls in between (they share the
    pod and candidate staging and pair -> pod map)."""
    import place_oracle as PL
    import preempt_oracle as PR
    from oracle import oracle as O
    t = R.default_table()
    cctx.set_table(t)
    rng = np.random.default_rng(7)
    wants = [(True, True, True), (False, False, False), (True, False, True), (False, True, False)]
    step = 0
    for width, n_node in ((8, 12), (32, 40), (8, 6), (16, 64), (8, 30)):
        g, off = walk_inventory(width, n_node)
        cctx.set_inventory(g, off)
        live = g
        for n_pod in (3, 200, 1, 57):
            c, po = _pods([PALETTE[int(i)] for i in rng.integers(0, 7, n_pod)])
            lists = [list(rng.integers(0, n_node + 1, int(rng.integers(0, 9)))) for _ in range(n_pod)]
            cn = np.array([x for li in lists for x in li] or [0], np.uint32)
            co = np.zeros(n_pod + 1, np.uint32)
            co[1:] = np.cumsum([len(x) for x in lists])
            for form in ("dense", "cands"):
                a = (None, None) if form == "dense" else (cn, co)
                fl = EXH if step % 2 else 0
                check(cctx, g, off, t, c, po, *a, mc=(5, 1, 300)[step % 3], fl=fl, want=wants[step % 4],
                      what=f"step {step} w{width} n{n_node} p{n_pod} {form}", live=live)
                step += 1
                k = step % 3
                if k == 0:
                    bits = cctx.unsuitable(c, po, *a, flags=fl)
                    ref = O.unsuitable(live, off, t, c, po, *(a if form == "cands" else _every_node(n_pod, n_node)), flags=fl)
                    assert bits.tobytes() == ref.tobytes(), f"unsuitable after step {step}"
                elif k == 1:
                    pc, ppo = _pods([SMALL, ONEGPU, EMPTY, SMALL])
                    out, pod_node = cctx.place_pods(pc, ppo, flags=fl)
                    ref_out, ref_node, live = PL.place_pods(live, off, t, pc, ppo, flags=fl)
                    assert out.tobytes() == ref_out.tobytes() and pod_node.tolist() == list(ref_node)
                    assert cctx.get_inventory().tobytes() == live.tobytes()
                else:
                    run = (EMPTY, np.zeros(1, np.uint32), np.zeros(0, np.int32), np.zeros(0, R.OUT_DTYPE), None)
                    prio = np.zeros(n_pod, np.int32)
                    got = cctx.preempt(c, po, prio, *run, *a, max_victims=2, flags=fl)
                    ref = PR.preempt(live, off, t, c, po, prio, *run, *a, max_victims=2, flags=fl)
                    assert all(x.tobytes() == y.tobytes() for x, y in zip(got, ref)), f"preempt after step {step}"
        cctx.reset_inventory()
        assert cctx.get_inventory().tobytes() == g.tobytes()


# ---- 5. near 2^32 pairs ------------------------------------------------------------------------------------------------
def _host_free():
    try:
        with open("/proc/meminfo") as f:
            return next(int(x.split()[1]) * 1024 for x in f if x.startswith("MemAvailable"))
    except (OSError, StopIteration):
        return 0


def _need(dev_bytes, host_bytes):
    import torch
    free, _ = torch.cuda.mem_get_info(0)
    if free < dev_bytes:
        pytest.skip(f"needs {dev_bytes / 2**30:.1f} GiB of device memory, {free / 2**30:.1f} GiB free")
    if _host_free() < host_bytes:
        pytest.skip(f"needs {host_bytes / 2**30:.1f} GiB of host memory, {_host_free() / 2**30:.1f} GiB available")


def limit_problem(n_node, n_pod, width):
    """n_pod pods, all empty but the first, one in the middle and the last: real pods of the walk palette"""
    g, off = walk_inventory(width, n_node)
    real = {0: SMALL, n_pod // 2: LIMIT, n_pod - 1: SHARED}
    po = np.zeros(n_pod + 1, np.uint32)
    for p, pod in real.items():
        po[p + 1:] += len(pod)
    c = np.concatenate([real[p] for p in sorted(real)])
    return g, off, c, po, real


@pytest.mark.parametrize("width", [8, 32])
def test_unsuitable_dense_at_the_pair_cap(pkg, cctx, width):
    """0xFFFFFFF0 pairs (6,960 nodes x 617,093 pods), first fit: the grid-stride walk ends after one pass; every empty
    row is suitable everywhere, every real row is the oracle's for its pod alone.  (The exhaustive form's counter walk
    is walk_fetch, as in k_pods_capacity, which test_capacity_dense_at_the_top_of_the_range runs at 2^32 - 1 pairs; at
    this size its 2^30 fetches from one counter would take minutes.)"""
    from oracle import oracle as O
    n_node, n_pod = 6960, 617093
    assert n_node * n_pod == 0xFFFFFFF0
    _need(3 << 30, 3 << 30)
    g, off, c, po, real = limit_problem(n_node, n_pod, width)
    t = R.default_table()
    cctx.set_table(t); cctx.set_inventory(g, off)
    row = n_node // 8
    for fl in (0,):
        bits = np.full(n_pod * row + SLACK, SENT, np.uint8)
        cctx._check(cctx._lib.dra_unsuitable_batch(cctx._h, _p(c), len(c), _p(po), n_pod, None, None, _p(bits), fl))
        assert (bits[n_pod * row:] == SENT).all()
        rows = bits[:n_pod * row].reshape(n_pod, row)
        for p, pod in real.items():
            ref = O.unsuitable(g, off, t, pod, np.array([0, len(pod)], np.uint32), *_every_node(1, n_node), flags=fl)
            assert rows[p].tobytes() == ref.tobytes(), f"f{fl} row {p}"
        mask = np.ones(n_pod, bool)
        mask[list(real)] = False
        assert (rows[mask] == 0xFF).all()
        assert cctx.get_inventory().tobytes() == g.tobytes()


def _rows_against_oracle(got_row, g, off, t, pod, mc, fl, what):
    ref = K.capacity(g, off, t, pod, np.array([0, len(pod)], np.uint32), None, None, mc, fl)
    same(got_row, ref, what)


def test_sharded_capacity_dense_at_the_pair_cap(pkg):
    """dra_pod_capacity_batch_global_device at world 1 over 0xFFFFFFF0 dense pairs, outputs kept on the device"""
    import torch
    import shard_world as S
    n_node, n_pod, mc = 6960, 617093, 3
    n_pair = n_node * n_pod
    _need(28 << 30, 1 << 30)
    g, off, c, po, real = limit_problem(n_node, n_pod, 8)
    t = R.default_table()
    W = S.World(pkg, t, off, g, 1, [0, n_node])
    try:
        ctx = W.ctxs[0]
        outs = [torch.full((s + SLACK,), SENT, dtype=torch.uint8, device="cuda:0")
                for s in (n_pair * 2, n_pair, n_pod * 8, n_pod * 4)]
        dc = torch.from_numpy(c.view(np.uint8).copy()).cuda()
        dpo = torch.from_numpy(po.view(np.uint8).copy()).cuda()
        torch.cuda.synchronize()
        ctx.pod_capacity_global_device(dc.data_ptr(), len(c), dpo.data_ptr(), n_pod, None, None, n_pair, mc,
                                       *[o.data_ptr() for o in outs], flags=EXH)
        ctx.sync()
        for o, s in zip(outs, (n_pair * 2, n_pair, n_pod * 8, n_pod * 4)):
            assert bool((o[s:] == SENT).all())
        copies = outs[0][:n_pair * 2].view(torch.int16).view(n_pod, n_node)
        stop = outs[1][:n_pair].view(n_pod, n_node)
        total = outs[2][:n_pod * 8].view(torch.int64)
        nodes = outs[3][:n_pod * 4].view(torch.int32)
        empty = torch.ones(n_pod, dtype=torch.bool, device="cuda:0")
        empty[list(real)] = False
        assert bool((copies[empty] == mc).all()) and bool((stop[empty] == K.ST_OK).all())
        assert bool((total[empty] == mc * n_node).all()) and bool((nodes[empty] == n_node).all())
        for p, pod in real.items():
            got = [copies[p].cpu().numpy().view(np.uint16), stop[p].cpu().numpy(),
                   total[p:p + 1].cpu().numpy().view(np.uint64), nodes[p:p + 1].cpu().numpy().view(np.uint32)]
            _rows_against_oracle(got, g, off, t, pod, mc, EXH, f"row {p}")
        assert ctx.get_inventory().tobytes() == g.tobytes()
    finally:
        W.close()


def test_capacity_dense_at_the_top_of_the_range(pkg, cctx):
    """dra_pod_capacity_batch over 2^32 - 1 dense pairs (4,369 nodes x 983,055 pods), pair_stop not asked for: the
    counter walk ends after one pass, though every warp's last fetch takes the counter past 2^32"""
    n_node, n_pod, mc = 4369, 983055, 3
    n_pair = n_node * n_pod
    assert n_pair == (1 << 32) - 1
    _need(20 << 30, 20 << 30)
    g, off, c, po, real = limit_problem(n_node, n_pod, 8)
    t = R.default_table()
    cctx.set_table(t); cctx.set_inventory(g, off)
    got = raw(cctx, c, po, mc=mc, fl=EXH, want=(False, True, True))
    copies = got[0].reshape(n_pod, n_node)
    empty = np.ones(n_pod, bool)
    empty[list(real)] = False
    for p, pod in real.items():
        _rows_against_oracle([copies[p], None, got[2][p:p + 1], got[3][p:p + 1]], g, off, t, pod, mc, EXH, f"row {p}")
    assert (got[2][empty] == mc * n_node).all() and (got[3][empty] == n_node).all()
    del got
    for lo in range(0, n_pod, 1 << 16):                  # in slices: a boolean mask over 2^32 pairs is 4 GB
        blk = copies[lo:lo + (1 << 16)]
        assert (blk[empty[lo:lo + (1 << 16)]] == mc).all(), f"rows {lo}.."
    assert cctx.get_inventory().tobytes() == g.tobytes()
