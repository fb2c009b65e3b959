"""GPU suite: Allocate at the record limits (tests/limit_problems.py) on every kernel path, byte for byte against the oracle.

Each problem reaches the packing loops where they differ from each other: 16-slice shapes and starts up to 15 (the 4-shift
plain-MIG loop), nodes of 17-32 GPUs, 31-65 claims on a node (segment boundaries, co-location runs across them, the
dead-shape memo carried between segments), SHARED segments at share count 0xFFFF and limits of 2^32 - 1.  Every Allocate
writes into a buffer longer than n_out whose tail must keep its sentinel, is compared with the oracle (OutRecs and
inventory), must have taken the expected kernel chain, and is undone by Deallocate on the device back to the pristine
inventory.  Paths:
  direct     default context: the single-launch kernel with direct host I/O
  nodirect   the single-launch kernel with the claim array staged, copy-engine transfers
  nofused    the one-CTA counting sort + one warp per node
  resident   the single-launch kernel kept up, batches by doorbell
  sorted     DRA_F_NODE_SORTED on the problem's claims stably sorted by node
  stream     padded with claims naming no node past the staged capacity: the streaming single-launch kernel
  sort       padded past the single-launch kernel's one-wave claim limit: CTA-wide histogram sort + one warp per node
  pack4      the problem tiled over more nodes than the device holds warps: warps of k_pack<4> walk several nodes
UnsuitableNodes (dense and candidate lists, with and without DRA_F_EXHAUSTIVE, as drawn and with an unnamed node of 9 or
17 GPUs appended so that the lane groups are 16 and 32 wide), pods Allocate and place pods run on the same problems."""
import os

import numpy as np
import pytest

import limit_problems as LP
import place_oracle as PO
from test_gpu_paths import STAGED_CAP, SORT8, assert_same

pytestmark = pytest.mark.gpu

R = LP.R
N_EX = int(os.environ.get("DRA_PROP_EXAMPLES", "0"))     # > 0: that many RANDOM seeds instead of the fixed ones
SEEDS = [int(s) for s in np.random.default_rng().integers(0, 1 << 30, N_EX)] if N_EX else list(range(40))
SLACK = 16
SENT = np.zeros(1, R.OUT_DTYPE)
SENT["gpu"], SENT["start"], SENT["size"], SENT["profile"], SENT["status"] = 0xA5A5A5A5, 0xA5, 0xA5, 0xA5, 0xA5
ONE_WAVE_FUSED_MAX = 14_000


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _problems():
    return [pb for pb in (LP.random_problem(s) for s in SEEDS) if len(pb.claims)]


def _pad(pb, n_claim):
    """pb with claims naming no node appended up to n_claim claims (they come back INVALID, one slot each)"""
    pad = np.zeros(n_claim - len(pb.claims), R.CLAIM_DTYPE)
    pad["kind"], pad["count"], pad["node"] = R.KIND_MIG, 1, pb.n_node
    c = np.concatenate([pb.claims, pad])
    oo, n_out = R.out_offsets(c, pb.n_node)
    return LP.Problem(pb.gpus, pb.node_off, pb.table, c, oo, n_out)


def _tile(pb, min_nodes):
    """pb repeated over at least min_nodes nodes: copy r's claims name node + r * n_node"""
    n = pb.n_node
    k = -(-min_nodes // n)
    g = np.tile(pb.gpus, k)
    w = np.diff(pb.node_off.astype(np.int64))
    off = np.zeros(k * n + 1, np.uint32)
    off[1:] = np.cumsum(np.tile(w, k))
    g["node"] = np.repeat(np.arange(k * n, dtype=np.uint32), np.tile(w, k))
    c = np.tile(pb.claims, k)
    r = np.repeat(np.arange(k, dtype=np.int64), len(pb.claims))
    node = c["node"].astype(np.int64)
    c["node"] = np.where(node < n, node + r * n, k * n).astype(np.uint32)
    oo, n_out = R.out_offsets(c, k * n)
    return LP.Problem(g, off, pb.table, c, oo, n_out)


def _alloc(c, pb, oracle, chain, flags=0, claims=None, oo=None, out=None, what=""):
    """One Allocate on context c, checked: slack, OutRecs, inventory, chain; then Deallocate back to pristine."""
    claims = pb.claims if claims is None else claims
    oo = pb.out_off if oo is None else oo
    ref, ref_inv = oracle.allocate(pb.gpus, pb.node_off, pb.table, pb.claims, pb.out_off, pb.n_out, threads=8)
    c.set_table(pb.table)
    c.set_inventory(pb.gpus, pb.node_off)
    buf = np.empty(pb.n_out + SLACK, R.OUT_DTYPE) if out is None else out[: pb.n_out + SLACK]
    buf[:] = SENT
    c.allocate(claims, oo, pb.n_out, flags=flags, out=buf)
    got_chain = c.last_chain()
    assert buf[pb.n_out:].tobytes() == SENT.tobytes() * SLACK, f"{what}: a write past n_out"
    assert_same(buf[: pb.n_out], c.get_inventory(), ref, ref_inv, what)
    assert chain(got_chain) if callable(chain) else got_chain == chain, f"{what}: took {sorted(got_chain)}"
    c.deallocate(claims, buf[: pb.n_out].copy(), oo)
    assert c.get_inventory().tobytes() == pb.gpus.tobytes(), f"{what}: Deallocate did not restore the inventory"


CFG = {"direct": 0, "nodirect": "CFG_NO_DIRECT", "nofused": "CFG_NO_FUSED", "resident": "CFG_RESIDENT", "sorted": 0,
       "stream": "CFG_NO_DIRECT", "sort": "CFG_NO_DIRECT", "pack4": 0}
CHAIN = {"direct": {"fused_direct"}, "nodirect": {"fused_staged"}, "nofused": {"bucket_small", "pack1"},
         "resident": {"serve"}, "sorted": {"sorted_prep", "pack1"}, "stream": {"fused_stream"}, "sort": SORT8 | {"pack1"},
         "pack4": lambda ch: "pack4" in ch and not ch & {"fused_staged", "fused_stream", "fused_direct"}}


def run_path(pkg, oracle, path, problems, request):
    A = pkg.api
    S = _sms()
    flags = getattr(A, CFG[path]) if CFG[path] else 0
    with A.Context(device=0, flags=flags) as c:
        out = None
        if path == "resident":
            n_c = max(len(pb.claims) for pb in problems)
            n_o = max(pb.n_out for pb in problems) + SLACK
            pins = [A.PinnedBuffer(n_c, R.CLAIM_DTYPE), A.PinnedBuffer(n_c, np.uint32), A.PinnedBuffer(n_o, R.OUT_DTYPE)]
            for b in pins:
                request.addfinalizer(b.free)         # (after the failure report, which shows arrays in these buffers)
            out = pins[2].array
        for k, pb in enumerate(problems if path != "pack4" else problems[:6]):
            what = f"{path} problem {k}"
            if path == "resident":
                n = len(pb.claims)
                pins[0].array[:n] = pb.claims
                pins[1].array[:n] = pb.out_off
                _alloc(c, pb, oracle, CHAIN[path], claims=pins[0].array[:n], oo=pins[1].array[:n], out=out, what=what)
            elif path == "sorted":
                p = np.argsort(pb.claims["node"], kind="stable")
                _alloc(c, pb, oracle, CHAIN[path], A.F_NODE_SORTED, claims=pb.claims[p], oo=pb.out_off[p], what=what)
            elif path == "stream":
                _alloc(c, _pad(pb, STAGED_CAP + 1), oracle, CHAIN[path], what=what)
            elif path == "sort":
                assert pb.n_node + 1 <= S
                _alloc(c, _pad(pb, ONE_WAVE_FUSED_MAX + 1), oracle, CHAIN[path], what=what)
            elif path == "pack4":
                _alloc(c, _tile(pb, 128 * S + 1), oracle, CHAIN[path], what=what)
            else:
                _alloc(c, pb, oracle, CHAIN[path], what=what)


@pytest.fixture(scope="module")
def problems():
    return _problems()


@pytest.mark.parametrize("path", list(CFG))
def test_allocate_on_every_path(pkg, oracle, problems, path, request):
    run_path(pkg, oracle, path, problems, request)


# ---- hand-written fixtures: the sharpest single cases -----------------------------------------------------------------
def _node(R, n_gpu, **kv):
    g, off = R.make_inventory([n_gpu], mig=kv.pop("mig", True))
    for k, v in kv.items():
        g[k] = v
    return g, off


def _claims(R, rows):
    c = np.zeros(len(rows), R.CLAIM_DTYPE)
    for i, (kind, profile, count, mem, group) in enumerate(rows):
        c[i] = (kind, profile, count, 0, mem, group)
    return c


def _fixture(name):
    U32 = LP.U32
    t = R.empty_table()
    t[3, 0] = (1, 0, 0xFFFF)                         # 1 slice anywhere, start 15 included
    t[3, 1] = (9, 0, 0x0001)                         # 9 slices at 0: the 4-shift loop
    t[3, 2] = (16, 0, 0x0001)                        # the whole GPU
    t[3, 4] = (12, 0, 0)                             # unoffered cell with a size byte above 8
    MIG, SH = R.KIND_MIG, R.KIND_SHARED
    if name == "dead_shape_in_segment_1":
        # two GPUs; 9g, 9g, then a 9g that finds no room (the shape dies in segment 0), 1g claims up to 32; the 33rd claim
        # asks 9g again in segment 1 and the 34th 1g, both NO_CAPACITY from the memo; an unoffered profile on both sides
        g, off = _node(R, 2, model=3)
        rows = [(MIG, 1, 1, 0, 0)] * 3 + [(MIG, 4, 1, 0, 0)] + [(MIG, 0, 1, 0, 0)] * 28 + \
               [(MIG, 1, 1, 0, 0), (MIG, 0, 1, 0, 0), (MIG, 4, 1, 0, 0)]
    elif name == "max_limit_after_clean_shared_segment":
        # one GPU with 2^32 - 1 MiB free: 32 time-sliced claims (segment 0, no failure), then a limit of 2^32 - 1 fits
        g, off = _node(R, 1, mig=False, mem_free_mib=U32)
        rows = [(SH, 0, 1, 0, 0)] * 32 + [(SH, 0, 1, U32, 0), (SH, 0, 1, 1, 0), (SH, 0, 1, 0, 0)]
    elif name == "share_count_at_fffe":
        # GPU 0 takes one share (to 0xFFFF) and then none, the rest go to GPU 1
        g, off = _node(R, 2, mig=False, mem_free_mib=U32)
        g["share_cnt"][0] = 0xFFFE
        rows = [(SH, 0, 1, 0, 0)] * 32 + [(SH, 0, 1, 5, 0)] * 3
    elif name == "run_across_segment_boundary":
        # 30 single slices on a 32-GPU node, then a run of four at positions 30-33, then single slices again
        g, off = _node(R, 32, model=3, busy=0xFFF0)
        rows = [(MIG, 0, 1, 0, 0)] * 30 + [(MIG, 0, 1, 0, 7)] * 4 + [(MIG, 0, 1, 0, 0)] * 31
    elif name == "whole_gpu_and_last_slice":
        g, off = _node(R, 17, model=3)
        g["busy"][:16] = 0x7FFF                      # only slice 15 free on GPUs 0..15
        rows = [(MIG, 2, 1, 0, 0)] + [(MIG, 0, 1, 0, 0)] * 17 + [(MIG, 2, 1, 0, 0)]      # the 17th 1g finds no room
    else:
        raise KeyError(name)
    c = _claims(R, rows)
    oo, n_out = R.out_offsets(c, 1)
    return LP.Problem(g, off, t, c, oo, n_out)


FIXTURES = ["dead_shape_in_segment_1", "max_limit_after_clean_shared_segment", "share_count_at_fffe",
            "run_across_segment_boundary", "whole_gpu_and_last_slice"]
EXPECT = {   # statuses the spec gives these, checked on the oracle before the device runs
    "dead_shape_in_segment_1": lambda s: list(s[:4]) == [0, 0, 1, 2] and list(s[32:]) == [1, 1, 2],
    "max_limit_after_clean_shared_segment": lambda s: list(s) == [0] * 33 + [4, 0],
    "share_count_at_fffe": lambda s: (s == 0).all(),
    "run_across_segment_boundary": lambda s: (s[30:34] == 0).all(),
    "whole_gpu_and_last_slice": lambda s: list(s) == [0] * 17 + [1, 1],
}


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture(pkg, oracle, name, request):
    pb = _fixture(name)
    ref, _ = oracle.allocate(pb.gpus, pb.node_off, pb.table, pb.claims, pb.out_off, pb.n_out)
    assert EXPECT[name](ref["status"]), ref["status"]
    for path in ("direct", "nodirect", "nofused", "resident", "sorted", "stream"):
        run_path(pkg, oracle, path, [pb], request)


# ---- UnsuitableNodes, pods Allocate, place pods --------------------------------------------------------------------------
def _extend(pb, width):
    """pb with one more node of `width` GPUs (MIG-enabled, first model of the table, empty)"""
    g, off = R.make_inventory([width], mig=True)
    g["model"] = int(np.nonzero(pb.table["start_mask"].any(axis=1))[0][0])
    g["node"] = pb.n_node
    return np.concatenate([pb.gpus, g]), np.append(pb.node_off, pb.node_off[-1] + width).astype(np.uint32)


def _cands(n_pod, n_node):
    cn, co = [], [0]
    for p in range(n_pod):
        cn += [(p + j) % n_node for j in range(p % 4)] + ([LP.NONE] if p % 5 == 0 else [])
        co.append(len(cn))
    return np.array(cn, np.uint32), np.array(co, np.uint32)


def test_unsuitable_and_pods(pkg, oracle, problems):
    A = pkg.api
    with A.Context(device=0) as c:
        for k, pb in enumerate(problems):
            claims, pod_off, oo, n_out = LP.pods(pb, k)
            n_pod = len(pod_off) - 1
            cn, co = _cands(n_pod, pb.n_node)
            c.set_table(pb.table)
            for width in (0, 9, 17):
                g, off = (pb.gpus, pb.node_off) if width == 0 else _extend(pb, width)
                n_node = len(off) - 1
                c.set_inventory(g, off)
                for flags in (0, A.F_EXHAUSTIVE):
                    what = f"problem {k} + node of {width}, flags {flags}"
                    dn = np.tile(np.arange(n_node, dtype=np.uint32), n_pod)
                    do = (np.arange(n_pod + 1) * n_node).astype(np.uint32)
                    got = c.unsuitable(claims, pod_off, flags=flags)
                    assert got.tobytes() == oracle.unsuitable(g, off, pb.table, claims, pod_off, dn, do, flags).tobytes(), what
                    got = c.unsuitable(claims, pod_off, cn, co, flags=flags)
                    want = oracle.unsuitable(pb.gpus, pb.node_off, pb.table, claims, pod_off, cn, co, flags)
                    assert got.tobytes() == want.tobytes(), f"{what}: candidate lists"
            c.set_inventory(pb.gpus, pb.node_off)
            for flags in (0, A.F_EXHAUSTIVE):
                what = f"problem {k}, flags {flags}"
                out = c.allocate_pods(claims, pod_off, oo, n_out, flags)
                ref, ref_inv = oracle.allocate_pods(pb.gpus, pb.node_off, pb.table, claims, pod_off, oo, n_out, flags)
                assert_same(out, c.get_inventory(), ref, ref_inv, f"pods Allocate, {what}")
                c.deallocate(claims, out, oo)
                assert c.get_inventory().tobytes() == pb.gpus.tobytes(), what
                for form in ((None, None), (cn, co)):
                    placed = claims.copy()
                    placed["node"] = 0
                    pl_oo, pl_n = R.out_offsets(placed, 1)
                    out, node = c.place_pods(claims, pod_off, *form, pl_oo, pl_n, flags)
                    ref, ref_node, ref_inv = PO.place_pods(pb.gpus, pb.node_off, pb.table, claims, pod_off, *form, pl_oo,
                                                           pl_n, flags)
                    assert_same(out, c.get_inventory(), ref, ref_inv, f"place pods, {what}, form {form[0] is not None}")
                    assert node.tobytes() == ref_node.tobytes(), what
                    c.set_inventory(pb.gpus, pb.node_off)
