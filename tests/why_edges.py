"""Problem builders for the reasons calls at their edges (spec §17, §18, §19) — TEST INFRASTRUCTURE ONLY.

`fixtures(W)` builds, for a widest node of W GPUs (W = 8, 16 or 32, so that the device evaluates each pair on W lanes),
one problem whose pods each fail for one reason at one position, laid out where the device's reason logic goes wrong:
the blocking claim at positions 0, W - 1, W and 31 (a lane-chunk shift is wrong only at W and above), MIG claims
interleaved with GPU and SHARED claims (the d-th MIG claim of the search is not at position d), co-location runs that
fail at their first member, and the search held at level d = 1, 7, 8, 16, 28 before it gives up.  Every pod carries
the (reason, position) it was built for on each node and in each mode (`Pod.want`); the CPU suite checks those against
both statements of each oracle.

The inventory uses three models of its own beside the default table's model 0:
  PIN   profiles 0 .. 13, each one slice at exactly one start (slice q): a claim of profile q has one place per GPU, so
        a co-location group of them walks its GPU level by level without choices;
  SOLE  profile 14 only, one slice at start 0;
  WIDE  profile 15 only, one slice at any of 16 starts: the claims that fill and the levels whose choices explode.
A node of width W: two PIN GPUs, one SOLE GPU, two WIDE GPUs, the rest plain (non-MIG) GPUs.  Node 0 has its SOLE GPU
full (a SOLE claim is NO_CAPACITY there), node 2 has it unavailable (BAD_PROFILE), node 1 has three plain GPUs only.
A lower-priority running pod holds one shared slot on the first plain GPU of nodes 0 and 2, for the §19 calls."""
from __future__ import annotations

import importlib
from dataclasses import dataclass, field

import numpy as np

import why_oracle as Y

R = importlib.import_module("k8s-dra-driver_b200").records
NONE = 0xFFFFFFFF
PIN, SOLE, WIDE = 2, 3, 4                      # models
P_SOLE, P_WIDE = 14, 15                        # profiles
N_PIN = 14                                     # profiles a PIN GPU offers: levels per co-location group
WIDTHS = (8, 16, 32)
POD_LEVELS = (1, 7, 8, 16, 28)
# a search level offers at most 32 GPUs x 16 starts = 512 choices, so 4096 descents need three levels of choices: the
# search runs out of budget at level 3 at the earliest, so d = 1 is asked for at 3
LIMIT_LEVELS = (3, 7, 8, 16, 28)
PRIO, RUN_PRIO = 10, 0
STRAY = 5                                       # a candidate naming no node of the 3-node inventory
MODES = ("ff", "exh", "place0", "place1", "pre0", "pre1")      # §17 first-fit / with the flag; §18, §19 without / with


def table():
    t = R.default_table()
    for q in range(N_PIN):
        t[PIN, q] = (1, 0, 1 << q)
    t[SOLE, P_SOLE] = (1, 0, 1)
    t[WIDE, P_WIDE] = (1, 0, 0xFFFF)
    return t


def claim(kind, profile=0, count=1, mem=0, group=0):
    c = np.zeros(1, R.CLAIM_DTYPE)
    c["kind"], c["profile"], c["count"], c["mem_limit_mib"], c["group"] = kind, profile, count, mem, group
    return c


def mig(profile, group=0):
    return claim(R.KIND_MIG, profile, group=group)


def gpu(count):
    return claim(R.KIND_GPU, count=count)


def shared(mem):
    return claim(R.KIND_SHARED, mem=mem)


def cat(parts):
    return np.concatenate(parts) if parts else np.zeros(0, R.CLAIM_DTYPE)


def node_gpus(W, sole):
    """one node of W GPUs: PIN, PIN, SOLE (flags `sole`), WIDE, WIDE, then plain GPUs"""
    g = np.zeros(W, R.GPU_DTYPE)
    g["mem_free_mib"] = 40960
    g["model"][:5] = (PIN, PIN, SOLE, WIDE, WIDE)
    g["flags"][:5] = R.GPU_MIG_ENABLED
    g["flags"][2] |= sole
    if not sole & R.GPU_UNAVAILABLE:
        g["busy"][2] = 1                        # full: its one start taken
    return g


def inventory(W):
    nodes = [node_gpus(W, 0), np.zeros(3, R.GPU_DTYPE), node_gpus(W, R.GPU_UNAVAILABLE)]
    nodes[1]["mem_free_mib"] = 40960
    g = np.concatenate(nodes)
    off = np.zeros(4, np.uint32)
    off[1:] = np.cumsum([len(x) for x in nodes])
    g["node"] = np.repeat(np.arange(3), [len(x) for x in nodes])
    return g, off


def running(g, off):
    """one lower-priority running pod per wide node, one shared slot of 1000 MiB on its first plain GPU (already in g)"""
    rc = cat([shared(1000), shared(1000)])
    ro = np.zeros(2, R.OUT_DTYPE)
    for i, n in enumerate((0, 2)):
        k = int(off[n]) + 5
        rc[i]["node"] = n
        g[k]["share_cnt"] += 1
        g[k]["mem_free_mib"] -= 1000
        ro[i] = (k, 0, 0, R.PROFILE_SHARED, R.ST_OK)
    return rc, np.arange(3, dtype=np.uint32), np.full(2, RUN_PRIO, np.int32), ro


@dataclass
class Pod:
    name: str
    claims: np.ndarray
    want: dict = field(default_factory=dict)    # (mode, node) -> (reason, position in the pod or None)
    cands: list = field(default_factory=lambda: [0, 1, 2])


def _all(modes, nodes, r, pos):
    return {(m, n): (r, pos) for m in modes for n in nodes}


def positions(W):
    return sorted({0, W - 1, W, 31} & set(range(32)))


def fill(n):
    """n WIDE claims: valid, each passes the pre-check, and first-fit places up to 32 of them on a wide node"""
    return cat([mig(P_WIDE)] * n)


def chain(d):
    """d co-location levels without choices after the first: profiles 0 .. 13 in group 1 on one PIN GPU, then group 2
    on the other; then the claim that fails on every branch (profile 0 in group 1: its GPU's slice 0 is taken) while it
    passes the pre-check alone"""
    lv = [mig(i % N_PIN, 1 + i // N_PIN) for i in range(d)]
    return lv, mig(0, 1)


def limited(d):
    """d levels: d - 3 without choices, then three levels of 32 choices each (a WIDE claim on either WIDE GPU); the
    claim at level d fails on every branch, so the search runs out of its 4096 descents holding d levels"""
    lv, bad = chain(d - 3)
    wide = [mig(P_WIDE, 3 if d == 3 else 0), mig(P_WIDE), mig(P_WIDE)]
    if d == 3:                                   # no PIN level: fail on the first WIDE claim's GPU, which has no profile 0
        bad = mig(0, 3)
    return lv + wide, bad


def interleave(levels, bad):
    """the MIG levels and the failing claim with a GPU, a SHARED and a GPU claim after the 1st, 3rd and 5th MIG claim:
    (claims, position of the failing claim)"""
    extra = [gpu(1), shared(100), gpu(1)]
    out = []
    for i, c in enumerate(levels + [bad]):
        out.append(c)
        if i in (0, 2, 4) and extra:
            out.append(extra.pop(0))
    out += extra
    pos = next(i for i, c in enumerate(out) if c is bad)
    return cat(out), pos


def fixture_pods(W):
    pods = []
    judged = ("exh", "place0", "place1", "pre0", "pre1")
    for p in positions(W):
        tail = [gpu(0), mig(77), fill(1)][: max(0, 31 - p)]
        c = cat([fill(p), mig(99)] + tail)
        w = _all(judged, (0, 1, 2), Y.ST_INVALID, p)
        w.update(_all(("ff",), (0, 2), Y.ST_INVALID, p))
        pods.append(Pod(f"invalid@{p}", c, w))
        # a GPU claim of W > the plain GPUs: NO_CAPACITY with out_off (INVALID without it, count != 1)
        c = cat([fill(p), gpu(W)] + ([fill(1)] if p < 31 else []))
        w = _all(judged, (0, 1, 2), Y.ST_NO_CAPACITY, p)
        w.update(_all(("ff",), (0, 2), Y.ST_NO_CAPACITY, p))
        pods.append(Pod(f"gpu_nocap@{p}", c, w))
        c = cat([fill(p), shared(50000)] + ([fill(1)] if p < 31 else []))
        w = _all(judged, (0, 1, 2), Y.ST_MEM_LIMIT, p)
        w.update(_all(("ff",), (0, 2), Y.ST_MEM_LIMIT, p))
        pods.append(Pod(f"mem_limit@{p}", c, w))
        c = cat([fill(p), mig(P_SOLE)])
        w = _all(MODES, (0,), Y.ST_NO_CAPACITY, p)
        w.update(_all(MODES, (2,), Y.ST_BAD_PROFILE, p))
        pods.append(Pod(f"precheck@{p}", c, w, [0, 0, 1, 2, 2]))        # each node listed twice in a row
        c = cat([fill(p), mig(P_SOLE, 7), mig(P_SOLE, 7)])
        pods.append(Pod(f"group@{p}", c, _all(("ff",), (0, 2), Y.ST_GROUP, p)))
        c = cat([fill(p), cat([mig(P_WIDE, 9)] * 40)])
        pods.append(Pod(f"group_cut@{p}", c, _all(("ff",), (0, 2), Y.ST_GROUP, p)))
    for d in POD_LEVELS:
        c, pos = interleave(*chain(d))
        pods.append(Pod(f"pod@d{d}", c, _all(judged, (0, 2), Y.ST_POD, pos), [0, 0, 2, 2, 2, 1]))
    for d in LIMIT_LEVELS:
        c, pos = interleave(*limited(d))
        w = _all(("exh", "place1", "pre1"), (0, 2), Y.ST_SEARCH_LIMIT, pos)
        w.update(_all(("place0", "pre0"), (0, 2), Y.ST_POD, pos))
        pods.append(Pod(f"limit@d{d}", c, w))
    # the running pod's shared slot keeps the plain GPUs from a claim of all W - 5 of them; with the victim released that
    # claim fits and the SHARED claim after it fails: §19 answers MEM_LIMIT at 1 where the calls without victims answer
    # NO_CAPACITY at 0
    w = _all(("ff", "exh", "place0", "place1"), (0, 2), Y.ST_NO_CAPACITY, 0)
    w.update(_all(("pre0", "pre1"), (0, 2), Y.ST_MEM_LIMIT, 1))
    pods.append(Pod("victim", cat([gpu(W - 5), shared(50000)]), w))
    pods.append(Pod("empty", cat([]), _all(MODES, (0, 1, 2), Y.ST_OK, None), [0, STRAY, 1, 2]))
    # placed at its first entry of node 0; the entries after it are dry runs, OK on the chosen node
    pods.append(Pod("stray", cat([shared(0)]), {(m, 0): (Y.ST_OK, None) for m in MODES},
                    [STRAY, 0, 0, 0, STRAY + 1000, NONE]))
    w = _all(("exh", "place0", "place1", "pre0", "pre1"), (0, 1, 2), Y.ST_INVALID, None)
    w.update(_all(("ff",), (0, 1, 2), Y.ST_OK, None))
    pods.append(Pod("33 claims", cat([shared(0)] * 33), w))
    return pods


class Problem:
    """One call's inputs, every call of the six alike: the inventory, the pods and their candidate lists, the running
    pods for §19; out_off (packed slots) for the slot mode of §18 and §19's placing form."""

    def __init__(self, name, gpus, node_off, tbl, pods, run=None, prio=PRIO, dense=False):
        self.name, self.gpus, self.node_off, self.table, self.pods = name, gpus, node_off, tbl, pods
        self.dense = dense                          # the dense form: every pod against every node
        self.attrs = self.sels = None               # selectors (spec §10), set on the context and the C oracle alike
        self.n_node = len(node_off) - 1
        self.claims = cat([p.claims for p in pods])
        self.pod_off = np.zeros(len(pods) + 1, np.uint32)
        self.pod_off[1:] = np.cumsum([len(p.claims) for p in pods])
        self.cands = [list(p.cands) if not dense else list(range(len(node_off) - 1)) for p in pods]
        self.cand_off = np.zeros(len(pods) + 1, np.uint32)
        self.cand_off[1:] = np.cumsum([len(x) for x in self.cands])
        self.cand_nodes = np.array([n for x in self.cands for n in x], np.uint32)
        self.prio = np.full(len(pods), prio, np.int32)
        self.run = run if run is not None else (np.zeros(0, R.CLAIM_DTYPE), np.zeros(1, np.uint32),
                                                np.zeros(0, np.int32), np.zeros(0, R.OUT_DTYPE))
        sl = slots(self.claims)
        self.out_off = np.concatenate([[0], np.cumsum(sl)[:-1]]).astype(np.uint32)
        self.n_out = int(sl.sum())

    def pairs(self):
        """(pod, node) of every pair in pair order"""
        return [(p, n) for p, x in enumerate(self.cands) for n in x]


def flat(name, gpus, node_off, tbl, claims, pod_off, cands, run=None, prio=PRIO, dense=False):
    """a Problem from flat arrays: claims split by pod_off, one candidate list per pod"""
    pods = [Pod(str(p), claims[pod_off[p]:pod_off[p + 1]], {}, [] if dense else list(cands[p]))
            for p in range(len(pod_off) - 1)]
    return Problem(name, gpus, node_off, tbl, pods, run, prio, dense)


def slots(claims):
    return np.array([int(c["count"]) if c["kind"] == R.KIND_GPU and 1 <= c["count"] <= 32 else 1 for c in claims],
                    np.uint32)


def fixtures(W):
    g, off = inventory(W)
    run = running(g, off)
    return Problem(f"fixtures w{W}", g, off, table(), fixture_pods(W), run)


# ---- §17 first-fit on long pods --------------------------------------------------------------------------------------
LONG = (32, 255, 256, 65_535)
LONGEST = 100_000


def long_pods():
    """First-fit §17 has no 32-claim limit: pods of SHARED claims of 0 MiB (65,535 of them fill a GPU's share count)
    on nodes of two plain GPUs, blocked at positions 32, 255, 256 and 65,535 by a SHARED claim no GPU has memory for or
    a GPU claim of 3, at the last claim of a 100,000-claim pod, and a 100,000-claim pod that fits."""
    g = np.zeros(4, R.GPU_DTYPE)
    g["mem_free_mib"] = 40960
    g["node"] = [0, 0, 1, 1]
    off = np.array([0, 2, 4], np.uint32)
    pods = []
    for i, k in enumerate(LONG):
        r, blk = (Y.ST_MEM_LIMIT, shared(50000)) if i % 2 == 0 else (Y.ST_NO_CAPACITY, gpu(3))
        pods.append(Pod(f"long@{k}", cat([shared(0)] * k + [blk, shared(0)]), _all(("ff",), (0, 1), r, k), [0, 1, 2]))
    pods.append(Pod(f"long@{LONGEST - 1}", cat([shared(0)] * (LONGEST - 1) + [shared(50000)]),
                    _all(("ff",), (0, 1), Y.ST_MEM_LIMIT, LONGEST - 1), [1, 0]))
    pods.append(Pod(f"long ok {LONGEST}", cat([shared(0)] * LONGEST), _all(("ff",), (0, 1), Y.ST_OK, None), [0, 3, 1]))
    return Problem("long pods", g, off, R.default_table(), pods)


# ---- tallies at scale ------------------------------------------------------------------------------------------------
def ladder(k_claims, n_cand, n_node=None, first=0):
    """nodes of 0, 1, 2, ... plain GPUs (n_node of them, widest < 33) and one pod of k_claims one-GPU claims: on the
    node of m GPUs claim m blocks (NO_CAPACITY), so candidates cycling over the nodes cycle the blocking claim over
    min(n_node, k_claims) distinct claims.  The pod's claims start at index `first` of a claims array of zero-claim
    pods before it."""
    n_node = n_node or k_claims
    widths = np.arange(n_node) % 33
    g = np.zeros(int(widths.sum()), R.GPU_DTYPE)
    g["mem_free_mib"] = 40960
    g["node"] = np.repeat(np.arange(n_node), widths)
    off = np.zeros(n_node + 1, np.uint32)
    off[1:] = np.cumsum(widths)
    return g, off, cat([gpu(1)] * k_claims), [i % n_node for i in range(n_cand)]


# ---- serial hand-off chains ------------------------------------------------------------------------------------------
def place_chain(n, mirror):
    """One-GPU MIG nodes, node at(0) full; pod i (a 7g) lists at(i), at(i+1): it finds at(i) taken by pod i - 1 and takes
    at(i + 1).  Reasons: (NO_CAPACITY, claim i) at at(i), (OK, none) at at(i + 1)."""
    at = (lambda k: n - 1 - k) if mirror else (lambda k: k)
    g, off = R.make_inventory([1] * n, mig=True)
    g["busy"][at(0)] = 0xFF
    c = cat([mig(R.GI_7_SLICE)] * (n - 1))
    pb = flat(f"chain {n} mirror {mirror}", g, off, R.default_table(), c, np.arange(n), [[at(i), at(i + 1)]
                                                                                          for i in range(n - 1)])
    why = np.tile(np.array([Y.ST_NO_CAPACITY, Y.ST_OK], np.uint8), n - 1)
    claim = np.full(2 * (n - 1), Y.WHY_CLAIM_NONE, np.uint32)
    claim[0::2] = np.arange(n - 1)
    return pb, chain_answer(why, claim, n - 1)


def pp_chain(n, mirror):
    """preempt and place across n one-GPU MIG nodes, node at(k) held by running pod k (a 7g of priority 0); pending pod i
    (a 7g of priority 1) lists at(i + 1), at(i): it evicts running pod i + 1 and takes at(i + 1), and pod i + 1 finds at(i
    + 1) held by a pod that is no victim.  Every pair: (NO_CAPACITY, claim i), on the live state or with the victims
    released."""
    at = (lambda k: n - 1 - k) if mirror else (lambda k: k)
    g, off = R.make_inventory([1] * n, mig=True)
    rc = cat([mig(R.GI_7_SLICE)] * n)
    rc["node"] = [at(k) for k in range(n)]
    ro = np.zeros(n, R.OUT_DTYPE)
    ro["gpu"], ro["start"], ro["size"], ro["profile"], ro["status"] = rc["node"], 0, 8, R.GI_7_SLICE, R.ST_OK
    g["busy"] = 0xFF
    run = (rc, np.arange(n + 1, dtype=np.uint32), np.zeros(n, np.int32), ro)
    c = cat([mig(R.GI_7_SLICE)] * (n - 1))
    pb = flat(f"pp chain {n} mirror {mirror}", g, off, R.default_table(), c, np.arange(n),
              [[at(i + 1), at(i)] for i in range(n - 1)], run, prio=1)
    why = np.full(2 * (n - 1), Y.ST_NO_CAPACITY, np.uint8)
    claim = np.repeat(np.arange(n - 1), 2).astype(np.uint32)
    return pb, chain_answer(why, claim, n - 1)


def chain_answer(why, claim, n_pod):
    rows = np.zeros((n_pod, Y.WHY_N), np.uint32)
    np.add.at(rows, (np.repeat(np.arange(n_pod), 2), why.astype(np.int64)), 1)
    blocks = np.bincount(claim[claim != Y.WHY_CLAIM_NONE].astype(np.int64), minlength=n_pod).astype(np.uint32)
    return why, claim, rows, blocks


def selector_problem(W):
    """fixtures(W)'s inventory, GPU attributes index = position in the node, and two selectors: 1 passes index 2 (the
    SOLE GPU) and 3 (a WIDE GPU), 2 passes index 3 only.  Pods of 8 WIDE claims, then a SOLE claim without a selector,
    with selector 2 (its only offering GPU hidden: BAD_PROFILE on node 0) and with selector 1 (NO_CAPACITY)."""
    g, off = inventory(W)
    attrs = np.zeros(len(g), R.ATTR_DTYPE)
    attrs["index"] = np.arange(len(g)) - np.repeat(off[:-1], np.diff(off.astype(np.int64)))
    sels = np.stack([R.selector(("cmp", R.ATTR_INDEX, R.CMP_IN_MASK, 0b1100)),
                     R.selector(("cmp", R.ATTR_INDEX, R.CMP_EQ, 3))])
    pods = []
    for sid in (0, 2, 1):
        c = cat([fill(8), mig(P_SOLE)])
        c[8]["mem_limit_mib"] = sid
        pods.append(Pod(f"sole sel {sid}", c, {}, [0, 2]))
    pb = Problem(f"selectors w{W}", g, off, table(), pods)
    pb.attrs, pb.sels = attrs, sels
    return pb
