"""CPU suite: the problems that test pods Allocate (spec §12, dra_allocate_pods_batch) at its edges, checked without a GPU.

tests/test_gpu_pods_edges.py runs these builders on the device against the C oracle, so the oracle is pinned here first:
every builder's problem gives the same bytes on oracle.allocate_pods and on oracle/naive.py's allocate_pods, and each
problem reaches the statuses it exists for.

* pod shapes and failure records: pods of 1, 31, 32 and 33 claims, empty pods, claims naming two nodes, a first claim
  naming no node before GPU claims of count 2-3 on valid nodes, GPU counts 0 and 33, MIG profiles >= 16, a selector id
  past the table, one claim invalid by §3 in an otherwise fitting pod
* nodes of 0, 1, 9, 17 and 32 GPUs, MIG and full, partly busy, with SHARED claims meeting share counts 0xFFFE / 0xFFFF
* every out_off form: none, identity, reversed, permuted, with gaps, with spare slots at the end
* the slot rule: a GPU claim has count slots only when it names a node of the inventory"""
from types import SimpleNamespace

import numpy as np
import pytest

import test_pod_search_fixtures as F
from test_pod_mode import _tbl
from test_pod_search_fixtures import _dicts

R = F.R
NONE = 0xFFFFFFFF
MIG_PROFILES = (0, 1, 2, 3, 4)                             # 1g, 2g, 3g, 4g, 7g
OUT_FORMS = ("none", "identity", "reversed", "permuted", "gaps", "spare")


def strays(n_node):
    """node fields that name no node of an n_node inventory"""
    return (n_node, n_node + 1000, NONE)


def slots(claims, n_node, have_off):
    """slots(c) of spec §1/§3, from each claim's own node field"""
    return R.claim_slots(claims, n_node, have_off)


def problem(name, g, off, t, claims, pod_off, out_off=None, n_out=None):
    """One pods call.  n_out defaults to what the out_off form needs: n_claim without out_off, the end of the last slot
    range with it."""
    off = np.asarray(off, np.uint32)
    n_node = len(off) - 1
    if out_off is not None:
        out_off = np.asarray(out_off, np.uint32)
    if n_out is None:
        n_out = len(claims) if out_off is None else int(max([int(o) + int(s) for o, s in
                                                            zip(out_off, slots(claims, n_node, True))], default=0))
    return SimpleNamespace(name=name, gpus=g, node_off=off, table=t, claims=claims, pod_off=np.asarray(pod_off, np.uint32),
                           out_off=out_off, n_out=n_out, n_node=n_node)


def owned(pb):
    """[n_out] bool: the slots some claim owns"""
    m = np.zeros(pb.n_out, bool)
    base = pb.out_off if pb.out_off is not None else np.arange(len(pb.claims))
    for b, s in zip(base, slots(pb.claims, pb.n_node, pb.out_off is not None)):
        m[int(b): int(b) + int(s)] = True
    return m


def out_form(claims, n_node, form, rng):
    """(out_off, n_out): none (slot i); ranges packed in claim order (identity), in reverse order, in a random order;
    in a random order with holes between and after them (gaps); packed with 7 spare slots at the end"""
    n = len(claims)
    if form == "none":
        return None, n
    sl = slots(claims, n_node, True).astype(np.int64)
    order = {"reversed": np.arange(n)[::-1], "permuted": rng.permutation(n), "gaps": rng.permutation(n)}.get(form, np.arange(n))
    out_off = np.zeros(n, np.uint32)
    pos = 0
    for i in order:
        pos += int(rng.integers(0, 3)) if form == "gaps" else 0
        out_off[i] = pos
        pos += int(sl[i])
    return out_off, pos + {"gaps": int(rng.integers(1, 3)), "spare": 7}.get(form, 0)


def _claims(n):
    return np.zeros(n, R.CLAIM_DTYPE)


def _mig(profiles):
    c = _claims(len(profiles))
    c["kind"], c["profile"], c["count"] = R.KIND_MIG, profiles, 1
    return c


def shapes_inventory(rng, copies=2):
    """Nodes of 0, 1, 9, 17 and 32 GPUs, MIG and full (not MIG), `copies` times.  MIG GPUs partly busy; full GPUs partly
    FULL_ALLOCATED, with less free memory, or with share counts 0xFFFE (one more share fits) and 0xFFFF (none does)."""
    widths = [0, 1, 9, 17, 32] * 2 * copies
    mig = ([True] * 5 + [False] * 5) * copies
    parts = [R.make_inventory([w], mig=m)[0] for w, m in zip(widths, mig)]
    g = np.concatenate(parts)
    off = np.zeros(len(widths) + 1, np.uint32)
    off[1:] = np.cumsum(widths)
    g["node"] = np.repeat(np.arange(len(widths)), widths)
    is_mig = (g["flags"] & R.GPU_MIG_ENABLED) != 0
    u = rng.random(len(g))
    g["busy"][is_mig & (u < 0.3)] = 0x0F
    g["busy"][is_mig & (u > 0.9)] = 0x7F
    full = ~is_mig
    g["flags"][full & (u < 0.2)] |= R.GPU_FULL_ALLOCATED
    g["share_cnt"][full & (u > 0.5) & (u < 0.65)] = 0xFFFE
    g["share_cnt"][full & (u > 0.65) & (u < 0.8)] = 0xFFFF
    g["mem_free_mib"][full & (u > 0.8)] = 5000
    for k in range(len(widths)):                              # a node's first share lands on its second GPU
        if not mig[k] and widths[k] >= 2:
            a = int(off[k])
            g["flags"][a: a + 2] = 0
            g["share_cnt"][a: a + 2] = (0xFFFF, 0xFFFE)
            g["mem_free_mib"][a: a + 2] = 40960
    return g, off, list(widths), mig


POD_KINDS = ["mixed"] * 6 + ["c1", "c31", "c32", "c33", "empty", "two_nodes", "nonode_first", "count0", "count33",
                             "prof16", "sel", "bad_fit", "stray"]


def _mixed(rng, m):
    """m claims: MIG 1g-7g, GPU claims of count 1-3, SHARED claims of 1-20 GB"""
    c = _claims(m)
    kind = rng.choice([R.KIND_MIG, R.KIND_MIG, R.KIND_GPU, R.KIND_SHARED], m)
    c["kind"] = kind
    c["profile"] = np.where(kind == R.KIND_MIG, rng.choice(MIG_PROFILES, m), 0)
    c["count"] = np.where(kind == R.KIND_GPU, rng.integers(1, 4, m), 1)
    c["mem_limit_mib"] = np.where(kind == R.KIND_SHARED, rng.integers(1, 21, m) * 1000, 0)
    return c


def shapes(seed=0, form="identity", n_pod=120, sel=True):
    """Pods of the kinds in POD_KINDS interleaved at random, each on a random node of shapes_inventory():
      c1 / c31 / c32 / c33  that many claims (c33 is INVALID), empty  no claims
      two_nodes     one claim names another node: every slot INVALID, GPU claims of count > 1 keep their count slots
      nonode_first  the first claim names no node, the rest are GPU claims of count 2-3 on valid nodes
      count0 / count33 / prof16  a GPU claim of count 0 / 33, a MIG claim of profile 16-255 (§3)
      sel           a claim naming selector 3 of an empty table (§10); sel=False: kind 3 instead (naive.py models
                    no selectors)
      bad_fit       one 1g on a node with room, plus a claim of profile 200: INVALID plus POD
      stray         every claim names the same node outside the inventory"""
    rng = np.random.default_rng(seed)
    g, off, widths, mig = shapes_inventory(rng)
    n = len(widths)
    st = strays(n)
    pods = []
    for _ in range(n_pod):
        k = POD_KINDS[int(rng.integers(len(POD_KINDS)))]
        node = int(rng.integers(n))
        if k == "c1":
            c = _mixed(rng, 1)
        elif k in ("c31", "c32", "c33"):                       # 1g claims on a MIG node with room for them
            c = _mig([R.GI_1_SLICE] * int(k[1:]))
            node = int(rng.choice([i for i in range(n) if mig[i] and widths[i] >= 9]))
        elif k == "empty":
            c = _claims(0)
        elif k == "bad_fit":
            c = _mig([R.GI_1_SLICE, R.GI_1_SLICE])
            c["profile"][int(rng.integers(2))] = 200
            node = int(rng.choice([i for i in range(n) if mig[i] and widths[i]]))
        else:
            c = _mixed(rng, int(rng.integers(1, 6)))
        c["node"] = node
        j = int(rng.integers(max(len(c), 1)))
        if k == "two_nodes":
            c = np.concatenate([c, _mixed(rng, 2)])
            c["node"][-2:] = (node + 1 + int(rng.integers(n - 1))) % n
            c["kind"][-1], c["count"][-1] = R.KIND_GPU, 3
        elif k == "nonode_first":
            c = np.concatenate([c[:1], _claims(int(rng.integers(1, 4)))])
            c["node"][0] = st[int(rng.integers(3))]
            c["kind"][1:], c["count"][1:] = R.KIND_GPU, rng.integers(2, 4, len(c) - 1)
            c["node"][1:] = rng.integers(0, n, len(c) - 1)
        elif k in ("count0", "count33"):
            c["kind"][j], c["profile"][j], c["count"][j] = R.KIND_GPU, 0, 0 if k == "count0" else 33
        elif k == "prof16":
            c["kind"][j], c["profile"][j], c["count"][j] = R.KIND_MIG, int(rng.integers(16, 256)), 1
        elif k == "sel" and sel:
            if c["kind"][j] == R.KIND_SHARED:
                c["group"][j] = 3                              # SHARED claims name their selector in group
            else:
                c["mem_limit_mib"][j] = 3                      # GPU and MIG claims in mem_limit_mib
        elif k == "sel":
            c["kind"][j] = 3
        elif k == "stray":
            c["node"] = st[int(rng.integers(3))]
        pods.append(c)
    claims = np.concatenate(pods)
    pod_off = np.zeros(n_pod + 1, np.uint32)
    pod_off[1:] = np.cumsum([len(c) for c in pods])
    out_off, n_out = out_form(claims, n, form, rng)
    return problem(f"shapes {seed} {form}", g, off, R.default_table(), claims, pod_off, out_off, n_out)


def only_empty(n_pod=40):
    g, off = R.make_inventory([1, 2, 0, 1], mig=True)
    return problem("only empty pods", g, off, R.default_table(), _claims(0), np.zeros(n_pod + 1, np.uint32))


def mostly_empty(seed=0, n_pod=1000, n_claim=10):
    """n_pod >> n_claim: 10 one-claim pods among 990 empty ones"""
    rng = np.random.default_rng(seed)
    g, off = R.make_inventory([1, 2, 0, 1], mig=True)
    c = _mig(rng.choice(MIG_PROFILES, n_claim))
    c["node"] = rng.integers(0, 4, n_claim)
    cuts = np.sort(rng.choice(np.arange(1, n_pod), n_claim - 1, replace=False))
    pod_off = np.zeros(n_pod + 1, np.uint32)
    for i, k in enumerate(cuts):
        pod_off[k:] = i + 1
    pod_off[-1] = n_claim
    return problem("mostly empty pods", g, off, R.default_table(), c, pod_off)


def boundary():
    """Calls whose slots end exactly at n_out, which must be accepted: the last slot range (a GPU claim of count 3 on a
    full node) ends at n_out; a count-5 GPU claim naming no node at out_off = n_out - 1 (one slot), alone in its pod and
    after a valid first claim of the same pod"""
    rng = np.random.default_rng(5)
    g, off, widths, mig = shapes_inventory(rng, copies=1)
    n = len(widths)
    full32 = next(i for i in range(n) if not mig[i] and widths[i] == 32)
    mig9 = next(i for i in range(n) if mig[i] and widths[i] == 9)
    t = R.default_table()
    a = _mig([R.GI_1_SLICE, R.GI_2_SLICE])
    a["node"] = mig9
    b = _claims(1)
    b["kind"], b["count"], b["node"] = R.KIND_GPU, 3, full32
    c = np.concatenate([a, b])
    out = [problem("ends at n_out", g, off, t, c, [0, 2, 3], [0, 1, 2], 5)]
    five = _claims(1)
    five["kind"], five["count"], five["node"] = R.KIND_GPU, 5, NONE
    pre = _mig([R.GI_1_SLICE])
    pre["node"] = mig9
    c = np.concatenate([pre, five])
    for where, po in (("own pod", [0, 1, 2]), ("second claim", [0, 2])):
        out.append(problem(f"count 5 naming no node at n_out - 1, {where}", g, off, t, c, po, [0, 1], 2))
    return out


# ---- checks ---------------------------------------------------------------------------------------------------------
def check_against_naive(oracle, pb, exhaustive):
    """oracle.allocate_pods and naive.allocate_pods give the same records and the same inventory"""
    from oracle import naive as N
    out, after = oracle.allocate_pods(pb.gpus, pb.node_off, pb.table, pb.claims, pb.pod_off, pb.out_off, pb.n_out,
                                      oracle.F_EXHAUSTIVE if exhaustive else 0)
    oo = None if pb.out_off is None else [int(x) for x in pb.out_off]
    nout, nafter = N.allocate_pods(_dicts(pb.gpus), [int(x) for x in pb.node_off], _tbl(pb.table), _dicts(pb.claims),
                                   [int(x) for x in pb.pod_off], exhaustive, oo)
    got = [tuple(int(v) for v in r) for r in out]
    assert len(nout) <= len(got), pb.name
    for i in range(len(got)):                               # slots no claim owns stay at the caller's zeros
        r = nout[i] if i < len(nout) else None
        assert got[i] == (r if r is not None else (0, 0, 0, 0, 0)), f"{pb.name}: slot {i}: {got[i]} != {r}"
    for a, b in zip(after, nafter):
        assert (int(a["busy"]), int(a["flags"]), int(a["mem_free_mib"]), int(a["share_cnt"])) == \
               (b["busy"], b["flags"], b["mem_free_mib"], b["share_cnt"]), pb.name
    return out, after


def pod_statuses(pb, out, p):
    """the set of statuses in pod p's slots"""
    have = pb.out_off is not None
    oo = pb.out_off if have else np.arange(len(pb.claims))
    sl = slots(pb.claims, pb.n_node, have)
    return {int(out["status"][int(oo[i]) + k]) for i in range(pb.pod_off[p], pb.pod_off[p + 1]) for k in range(sl[i])}


@pytest.mark.parametrize("form", OUT_FORMS)
def test_shapes_agree_with_naive(oracle, form):
    for seed in range(2):
        pb = shapes(seed, form, n_pod=80, sel=False)
        for exhaustive in (False, True):
            out, _ = check_against_naive(oracle, pb, exhaustive)
            st = set(out["status"][owned(pb)].tolist())
            assert {R.ST_OK, R.ST_INVALID, R.ST_POD} <= st, (pb.name, st)


def test_empty_and_boundary_problems_agree_with_naive(oracle):
    for pb in [only_empty(), mostly_empty()] + boundary():
        for exhaustive in (False, True):
            check_against_naive(oracle, pb, exhaustive)


def test_shapes_cover_their_cases(oracle):
    pb = shapes(0, "identity")
    out, after = oracle.allocate_pods(pb.gpus, pb.node_off, pb.table, pb.claims, pb.pod_off, pb.out_off, pb.n_out,
                                      oracle.F_EXHAUSTIVE)
    sizes = np.diff(pb.pod_off.astype(np.int64))
    assert {0, 1, 31, 32, 33} <= set(sizes.tolist())
    assert all(pod_statuses(pb, out, p) == {R.ST_INVALID} for p in np.flatnonzero(sizes == 33))
    assert any(pod_statuses(pb, out, p) == {R.ST_OK} for p in np.flatnonzero(sizes == 32))
    c = pb.claims
    gpu = c["kind"] == R.KIND_GPU
    assert {0, 2, 3, 33} <= set(c["count"][gpu].tolist())
    assert (c["profile"][c["kind"] == R.KIND_MIG] >= 16).any()
    sel = np.flatnonzero(((c["mem_limit_mib"] == 3) & (c["kind"] != R.KIND_SHARED)) | ((c["group"] == 3) & (c["kind"] == R.KIND_SHARED)))
    assert len(sel) and (out["status"][pb.out_off[sel]] == R.ST_INVALID).all()      # §10: a selector id past the table
    # GPU claims of count > 1 in malformed pods keep the count slots of their own node field
    first = c["node"][pb.pod_off[:-1][sizes > 0]]
    nonode = [p for p in np.flatnonzero(sizes > 0) if c["node"][pb.pod_off[p]] >= pb.n_node and
              (c["node"][pb.pod_off[p] + 1: pb.pod_off[p + 1]] < pb.n_node).any()]
    assert nonode and all(pod_statuses(pb, out, p) == {R.ST_INVALID} for p in nonode)
    assert (first >= pb.n_node).any() and (first < pb.n_node).any()
    wide = gpu & (c["count"] > 1) & (c["count"] <= R.MAX_COUNT) & (c["node"] < pb.n_node)
    assert wide.any() and (slots(c, pb.n_node, True)[wide] > 1).all()
    # INVALID plus POD in one pod: a §3-invalid claim in an otherwise fitting pod
    assert any(pod_statuses(pb, out, p) == {R.ST_INVALID, R.ST_POD} for p in range(len(sizes)))
    # shares taken on GPUs at 0xFFFE, none on GPUs at 0xFFFF
    assert ((pb.gpus["share_cnt"] == 0xFFFE) & (after["share_cnt"] == 0xFFFF)).any()
    assert (after["share_cnt"][pb.gpus["share_cnt"] == 0xFFFF] == 0xFFFF).all()
    assert (out["status"][owned(pb)] == R.ST_OK).sum() >= 30


def test_out_forms():
    for form in OUT_FORMS:
        pb = shapes(3, form)
        sl = slots(pb.claims, pb.n_node, pb.out_off is not None)
        assert sl.sum() == owned(pb).sum(), form                 # no two claims share a slot
        assert (pb.n_out > sl.sum()) == (form in ("gaps", "spare")), form
    pb = shapes(3, "reversed")
    assert pb.out_off[-1] == 0 and pb.out_off[0] == pb.n_out - slots(pb.claims[:1], pb.n_node, True)[0]


def test_slot_rule_follows_the_claims_own_node(oracle):
    """A count-5 GPU claim has five slots only when it names a node of the inventory: at out_off = n_out - 1 the oracle
    takes it naming no node, and refuses it naming a node"""
    pb = boundary()[1]
    out, _ = oracle.allocate_pods(pb.gpus, pb.node_off, pb.table, pb.claims, pb.pod_off, pb.out_off, pb.n_out)
    assert out["status"][1] == R.ST_INVALID and out["gpu"][1] == NONE
    c = pb.claims.copy()
    c["node"][1] = c["node"][0]
    with pytest.raises(ValueError):
        oracle.allocate_pods(pb.gpus, pb.node_off, pb.table, c, pb.pod_off, pb.out_off, pb.n_out)
    assert list(slots(c, pb.n_node, True)) == [1, 5] and list(slots(pb.claims, pb.n_node, True)) == [1, 1]
