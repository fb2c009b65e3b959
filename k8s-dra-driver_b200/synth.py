"""Seeded synthetic workloads for the five BASELINE.json configs (SURVEY.md §8d, BASELINE.md §4).

SplitMix64, base seed 0x0D5A110C, per-config seed = base + config number.  The same buffers feed the CPU
oracle and the CUDA path; nothing here reads the reference snapshot.  The reference ships no workloads of its
own for this path — the only in-tree workload shapes are the quickstart specs
(demo/specs/quickstart/gpu-test4.yaml:19-44 etc.), reproduced in tests/ as fixtures.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from . import records as R

BASE_SEED = 0x0D5A110C
_GOLDEN = np.uint64(0x9E3779B97F4A7C15)


def splitmix64(seed: int, n: int) -> np.ndarray:
    """n outputs of SplitMix64 started at `seed` (vectorised: state_i = seed + (i+1)*golden)."""
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + _GOLDEN * np.arange(1, n + 1, dtype=np.uint64)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


@dataclass
class Workload:
    name: str
    gpus: np.ndarray          # GPU_DTYPE[n_gpu]
    node_off: np.ndarray      # uint32[n_node+1]
    table: np.ndarray         # PROF_DTYPE[16,16]
    claims: np.ndarray        # CLAIM_DTYPE[n_claim], generation (unsorted) order
    out_off: np.ndarray | None = None
    n_out: int = 0

    @property
    def n_node(self) -> int:
        return len(self.node_off) - 1

    @property
    def n_gpu(self) -> int:
        return len(self.gpus)

    @property
    def n_claim(self) -> int:
        return len(self.claims)

    def node_sorted(self) -> "Workload":
        """Stable sort of the claims by node (the input order SURVEY §8d quotes for cfg2)."""
        order = np.argsort(self.claims["node"], kind="stable")
        w = Workload(self.name + "+sorted", self.gpus.copy(), self.node_off, self.table,
                     self.claims[order].copy())
        w.finish()
        return w

    def finish(self) -> "Workload":
        if not np.any((self.claims["kind"] == R.KIND_GPU) & (self.claims["count"] != 1)):
            self.out_off, self.n_out = None, self.n_claim
        else:
            self.out_off, self.n_out = R.out_offsets(self.claims, self.n_node)
        return self

    def algorithmic_bytes(self) -> int:
        """SURVEY §8(d): 16 B/claim read + 16 B/GPU read + 8 B/slot written."""
        return 16 * self.n_claim + 16 * self.n_gpu + 8 * self.n_out


def _mig_mix(n_claim: int, n_node: int, seed: int, node_base: int = 0) -> np.ndarray:
    r = splitmix64(seed, 2 * n_claim)
    pick = (r[0::2] % np.uint64(100)).astype(np.int64)
    prof = np.where(pick < 40, R.GI_1_SLICE,
                    np.where(pick < 70, R.GI_2_SLICE, np.where(pick < 90, R.GI_3_SLICE, R.GI_7_SLICE)))
    c = np.zeros(n_claim, dtype=R.CLAIM_DTYPE)
    c["kind"] = R.KIND_MIG
    c["profile"] = prof
    c["count"] = 1
    c["node"] = (r[1::2] % np.uint64(n_node)).astype(np.uint32) + np.uint32(node_base)
    return c


def cfg1() -> Workload:
    """64 full-GPU claims over one 8-GPU node: first 8 succeed (gpu 0..7), 56 fail."""
    g, off = R.make_inventory([8], mig=False)
    c = np.zeros(64, dtype=R.CLAIM_DTYPE)
    c["kind"] = R.KIND_GPU
    c["count"] = 1
    return Workload("cfg1", g, off, R.default_table(), c).finish()


def cfg2(n_claim: int = 10_000, n_node: int = 125, gpus_per_node: int = 8, seed_off: int = 2) -> Workload:
    """10k mixed 1g/2g/3g/7g MIG claims (40/30/20/10 %) over 125 nodes x 8 empty MIG-enabled GPUs."""
    g, off = R.make_inventory([gpus_per_node] * n_node, mig=True)
    c = _mig_mix(n_claim, n_node, BASE_SEED + seed_off)
    return Workload("cfg2", g, off, R.default_table(), c).finish()


def cfg3(n_claim: int = 100_000, n_node: int = 1000) -> Workload:
    """100k claims x 8k GPUs, same mix; nodes are sharded contiguously over ranks."""
    w = cfg2(n_claim, n_node, 8, seed_off=3)
    w.name = "cfg3"
    return w


def cfg3_shard(rank: int, world: int, claims_per_rank: int = 12_500, nodes_per_rank: int = 125) -> Workload:
    """Rank-local slice of a cfg3-shaped job (weak scaling: every rank owns nodes_per_rank nodes and
    the claims_per_rank claims that select them).  Node indices are LOCAL to the rank's inventory."""
    g, off = R.make_inventory([8] * nodes_per_rank, mig=True)
    c = _mig_mix(claims_per_rank, nodes_per_rank, BASE_SEED + 3 + 1000 * (rank + 1))
    return Workload(f"cfg3[{rank}/{world}]", g, off, R.default_table(), c).finish()


def cfg4(n_claim: int = 10_000, n_node: int = 125) -> Workload:
    """MPS / time-slice shared claims with a per-claim memory limit (spec §7, extension)."""
    g, off = R.make_inventory([8] * n_node, mig=False, mem_free_mib=40960)
    r = splitmix64(BASE_SEED + 4, 3 * n_claim)
    mps = (r[0::3] & np.uint64(1)).astype(bool)
    limits = np.array([1024, 2048, 4096, 8192, 10240], dtype=np.uint32)
    c = np.zeros(n_claim, dtype=R.CLAIM_DTYPE)
    c["kind"] = R.KIND_SHARED
    c["count"] = 1
    c["mem_limit_mib"] = np.where(mps, limits[(r[1::3] % np.uint64(5)).astype(np.int64)], 0)
    c["node"] = (r[2::3] % np.uint64(n_node)).astype(np.uint32)
    return Workload("cfg4", g, off, R.default_table(), c).finish()


_FRAG = np.array([0x55, 0xAA, 0x33, 0xCC, 0x0F, 0xF0, 0x5A, 0xA5, 0x7E, 0x3C, 0x66, 0x99, 0x11, 0x88],
                 dtype=np.uint16)


def cfg5(n_claim: int = 50_000, n_node: int = 64) -> Workload:
    """Adversarial fragmentation: 50k 1g claims into 512 pre-fragmented GPUs."""
    g, off = R.make_inventory([8] * n_node, mig=True)
    r = splitmix64(BASE_SEED + 5, len(g) + n_claim)
    g["busy"] = _FRAG[(r[: len(g)] % np.uint64(len(_FRAG))).astype(np.int64)]
    c = np.zeros(n_claim, dtype=R.CLAIM_DTYPE)
    c["kind"] = R.KIND_MIG
    c["profile"] = R.GI_1_SLICE
    c["count"] = 1
    c["node"] = (r[len(g):] % np.uint64(n_node)).astype(np.uint32)
    return Workload("cfg5", g, off, R.default_table(), c).finish()


def mixed(n_claim: int = 4000, n_node: int = 37, seed: int = 7, invalid: bool = True) -> Workload:
    """Everything at once, for parity fuzzing: ragged heterogeneous nodes (0..32 GPUs, two models,
    MIG and non-MIG, pre-occupied, unavailable), all three kinds, count > 1, co-location groups,
    unsupported profiles and (optionally) malformed claims."""
    r = splitmix64(BASE_SEED + 100 + seed, 8 * (n_node * 40 + n_claim) + 64)
    pos = [0]

    def take(n):
        s = pos[0]
        pos[0] += n
        return r[s: s + n]

    sizes = (take(n_node) % np.uint64(12)).astype(np.int64)
    sizes[sizes == 11] = 32          # a few full-width nodes
    sizes[:: max(1, n_node // 5)] = 0  # and some empty ones
    if n_node > 2:
        sizes[1] = 8
    g, off = R.make_inventory(list(sizes), mig=True)
    ng = len(g)
    a = take(max(ng, 1) * 4)
    g["flags"] = np.where(a[0:ng] % np.uint64(3) == 0, 0, R.GPU_MIG_ENABLED).astype(np.uint8)
    g["flags"] |= np.where(a[ng:2 * ng] % np.uint64(17) == 0, R.GPU_UNAVAILABLE, 0).astype(np.uint8)
    g["model"] = (a[2 * ng:3 * ng] % np.uint64(4) == 0).astype(np.uint8)
    pre = (a[3 * ng:4 * ng] % np.uint64(256)).astype(np.uint16)
    pre = np.where(a[3 * ng:4 * ng] % np.uint64(5) < 2, pre, 0).astype(np.uint16)
    g["busy"] = np.where(g["model"] == 1, pre & 0xF, pre)
    g["busy"] = np.where(g["flags"] & R.GPU_MIG_ENABLED, g["busy"], 0)
    g["mem_free_mib"] = 16384

    b = take(n_claim * 6)
    c = np.zeros(n_claim, dtype=R.CLAIM_DTYPE)
    k = (b[0::6] % np.uint64(10)).astype(np.int64)
    c["kind"] = np.where(k < 6, R.KIND_MIG, np.where(k < 8, R.KIND_GPU, R.KIND_SHARED))
    profs = np.array([0, 0, 0, 1, 1, 2, 3, 4, 7, 9, 5, 6], dtype=np.uint8)
    c["profile"] = profs[(b[1::6] % np.uint64(len(profs))).astype(np.int64)]
    cnt = (b[2::6] % np.uint64(8)).astype(np.int64)
    c["count"] = np.where(c["kind"] == R.KIND_GPU, np.where(cnt < 5, 1, cnt - 3), 1)
    c["node"] = (b[3::6] % np.uint64(n_node)).astype(np.uint32)
    c["mem_limit_mib"] = np.where(c["kind"] == R.KIND_SHARED,
                                  (b[4::6] % np.uint64(5)).astype(np.uint32) * 3000, 0)
    # co-location groups: runs of 2..5 consecutive MIG claims on one node share a group id
    gsel = b[5::6]
    i = 0
    gid = 1
    while i < n_claim:
        if gsel[i] % np.uint64(9) == 0:
            ln = int(gsel[i] >> np.uint64(8)) % 4 + 2
            j = min(n_claim, i + ln)
            c["kind"][i:j] = R.KIND_MIG
            c["count"][i:j] = 1
            c["mem_limit_mib"][i:j] = 0
            c["node"][i:j] = c["node"][i]
            c["group"][i:j] = gid
            small = np.array([0, 0, 1, 0, 2], dtype=np.uint8)
            c["profile"][i:j] = small[(gsel[i:j] >> np.uint64(16)).astype(np.int64) % 5]
            gid += 1
            i = j
        else:
            i += 1
    if invalid:
        bad = take(n_claim)
        c["kind"] = np.where(bad % np.uint64(97) == 0, 3, c["kind"])
        c["node"] = np.where(bad % np.uint64(89) == 1, n_node + 5, c["node"])
        c["count"] = np.where((bad % np.uint64(83) == 2) & (c["kind"] == R.KIND_GPU), 0, c["count"])
        c["count"] = np.where((bad % np.uint64(83) == 3) & (c["kind"] == R.KIND_GPU), 40, c["count"])
        c["profile"] = np.where((bad % np.uint64(79) == 4) & (c["kind"] == R.KIND_MIG), 200, c["profile"])
    w = Workload(f"mixed{seed}", g, off, R.default_table(), c)
    w.out_off, w.n_out = R.out_offsets(c, n_node)
    return w


def with_selectors(w: Workload, seed: int = 1, frac: int = 3):
    """Adds GPU attributes, a selector table (spec §10) and selector ids on ~1/frac of the claims of `w`.
    Returns (attrs, sels).  Shapes follow demo/specs/selectors/parameters.yaml:7-27 (memory / compute
    capability comparisons under and-expressions) and demo/specs/quickstart/gpu-test6.yaml:23-31
    (product match && index in a set)."""
    r = splitmix64(BASE_SEED + 900 + seed, 4 * max(w.n_gpu, 1) + 2 * w.n_claim + 8)
    ng = w.n_gpu
    a = np.zeros(ng, dtype=R.ATTR_DTYPE)
    a["mem_total_mib"] = np.array([16384, 40960, 81920], dtype=np.uint32)[(r[0:ng] % np.uint64(3)).astype(np.int64)]
    a["cc"] = np.array([0x0705, 0x0800, 0x0900], dtype=np.uint32)[(r[ng:2 * ng] % np.uint64(3)).astype(np.int64)]
    a["index"] = np.arange(ng, dtype=np.uint32) - np.repeat(w.node_off[:-1], np.diff(w.node_off)).astype(np.uint32)
    a["product"] = (r[2 * ng:3 * ng] % np.uint64(4)).astype(np.uint16)
    a["driver_major"] = np.array([535, 550, 570], dtype=np.uint16)[(r[3 * ng:4 * ng] % np.uint64(3)).astype(np.int64)]
    S_ = R.selector
    sels = np.stack([
        S_(("cmp", R.ATTR_MEMORY_MIB, R.CMP_LE, 16384), ("cmp", R.ATTR_CC, R.CMP_GE, 0x0705), "and"),   # "inference-gpu"
        S_(("cmp", R.ATTR_MEMORY_MIB, R.CMP_GE, 40960)),                                                  # "training-gpu"
        S_(("cmp", R.ATTR_PRODUCT, R.CMP_IN_MASK, 0b0110), ("cmp", R.ATTR_INDEX, R.CMP_IN_MASK, 0b01010101), "and"),
        S_(("cmp", R.ATTR_CC, R.CMP_LT, 0x0800), "not"),
        S_("and"),                                                                                         # malformed: false
        S_(),                                                                                              # empty: true
        S_(("cmp", R.ATTR_DRIVER_MAJOR, R.CMP_NE, 535), ("cmp", R.ATTR_INDEX, R.CMP_GT, 1), "or",
           ("cmp", R.ATTR_MEMORY_MIB, R.CMP_EQ, 81920), "or"),
    ])
    pick = r[4 * ng: 4 * ng + w.n_claim]
    sid = (r[4 * ng + w.n_claim: 4 * ng + 2 * w.n_claim] % np.uint64(len(sels) + 2)).astype(np.uint32) + 1   # a few beyond the table
    use = (pick % np.uint64(frac)) == 0
    c = w.claims
    gm = use & ((c["kind"] == R.KIND_GPU) | (c["kind"] == R.KIND_MIG))
    c["mem_limit_mib"] = np.where(gm, sid, c["mem_limit_mib"])
    sh = use & (c["kind"] == R.KIND_SHARED)
    c["group"] = np.where(sh, sid, c["group"])
    return a, sels


CONFIGS = {"cfg1": cfg1, "cfg2": cfg2, "cfg3": cfg3, "cfg4": cfg4, "cfg5": cfg5}


def homog(n_claim: int = 3000, n_node: int = 24, seed: int = 1, model: int = 0, wide16: bool = False,
          max_width: int = 32) -> Workload:
    """Homogeneous all-MIG nodes of widths 1..max_width with pre-occupied, fully-allocated and unavailable
    GPUs, MIG-only claims incl. unsupported profiles: the workload class of the packers' fast loops (the
    64-bit SWAR form for <= 8 GPUs x <= 8 slices, the ballot form for anything wider).  ``wide16`` swaps in a
    synthetic 16-slice part so that occupancy masks do not fit a byte."""
    r = splitmix64(BASE_SEED + 900 + seed, 8 * (n_node * 40 + n_claim) + 64)
    sizes = 1 + (r[:n_node] % np.uint64(max_width)).astype(np.int64)
    sizes[::3] = np.minimum(sizes[::3], 8)
    g, off = R.make_inventory(list(sizes), mig=True, model=model)
    ng = len(g)
    a = r[n_node: n_node + 3 * ng]
    t = R.default_table()
    if wide16:
        t[model] = 0
        t[model, R.GI_1_SLICE] = (1, 0, 0xFFFF)
        t[model, R.GI_2_SLICE] = (2, 0, 0x5555)
        t[model, R.GI_3_SLICE] = (5, 0, R.mask_of((0, 5, 10)))
        t[model, R.GI_4_SLICE] = (8, 0, R.mask_of((0, 8)))
        t[model, R.GI_7_SLICE] = (16, 0, 1)
    width = 0xFFFF if wide16 else (0xFF if model == 0 else 0xF)
    pre = (a[0:ng] % np.uint64(65536)).astype(np.uint16) & np.uint16(width)
    g["busy"] = np.where(a[0:ng] % np.uint64(4) == 0, pre, 0)
    g["flags"] |= np.where(a[ng:2 * ng] % np.uint64(13) == 0, R.GPU_UNAVAILABLE, 0).astype(np.uint8)
    g["flags"] |= np.where(a[2 * ng:3 * ng] % np.uint64(11) == 0, R.GPU_FULL_ALLOCATED, 0).astype(np.uint8)
    b = r[n_node + 3 * ng: n_node + 3 * ng + 2 * n_claim]
    c = np.zeros(n_claim, dtype=R.CLAIM_DTYPE)
    c["kind"] = R.KIND_MIG
    c["count"] = 1
    profs = np.array([0, 0, 0, 0, 1, 1, 2, 3, 4, 7, 9, 5, 12], dtype=np.uint8)
    c["profile"] = profs[(b[0::2] % np.uint64(len(profs))).astype(np.int64)]
    c["node"] = (b[1::2] % np.uint64(n_node)).astype(np.uint32)
    return Workload(f"homog{seed}", g, off, t, c).finish()


def pods(n_pod: int = 20_000, n_node: int = 64, seed: int = 0, gpus_per_node: int = 8, max_claims: int = 5,
         grouped: bool = True):
    """Pod-mode workload (spec §12): pods of 1..max_claims MIG claims of mixed profiles (the multi-request shape of
    demo/specs/quickstart/gpu-test4.yaml:19-44) over cfg5's pre-fragmented inventory — the regime where in-order
    first-fit gives false negatives.  ~1/4 of the multi-claim pods carry a co-location group (matchAttribute
    parentUUID).  Returns (Workload, pod_off)."""
    g, off = R.make_inventory([gpus_per_node] * n_node, mig=True)
    r = splitmix64(BASE_SEED + 500 + seed, len(g) + 3 * n_pod + n_pod * max_claims + 8)
    g["busy"] = _FRAG[(r[: len(g)] % np.uint64(len(_FRAG))).astype(np.int64)]
    a = r[len(g):]
    sizes = 1 + (a[:n_pod] % np.uint64(max_claims)).astype(np.int64)
    nodes = (a[n_pod: 2 * n_pod] % np.uint64(n_node)).astype(np.uint32)
    grp = (a[2 * n_pod: 3 * n_pod] % np.uint64(4) == 0) & (sizes > 1) if grouped else np.zeros(n_pod, bool)
    pod_off = np.zeros(n_pod + 1, dtype=np.uint32)
    pod_off[1:] = np.cumsum(sizes)
    n_claim = int(pod_off[-1])
    c = np.zeros(n_claim, dtype=R.CLAIM_DTYPE)
    c["kind"], c["count"] = R.KIND_MIG, 1
    pick = (a[3 * n_pod: 3 * n_pod + n_claim] % np.uint64(100)).astype(np.int64)
    c["profile"] = np.where(pick < 45, R.GI_1_SLICE, np.where(pick < 75, R.GI_2_SLICE,
                            np.where(pick < 97, R.GI_3_SLICE, R.GI_7_SLICE)))
    c["node"] = np.repeat(nodes, sizes)
    c["group"] = np.repeat(np.where(grp, np.arange(1, n_pod + 1, dtype=np.uint32), 0).astype(np.uint32), sizes)
    w = Workload(f"pods{seed}", g, off, R.default_table(), c).finish()
    return w, pod_off


@dataclass
class PreemptWorld:
    """A consistent inventory with the running pods that occupy it, and pending pods for spec §14 (preemption)."""
    gpus: np.ndarray          # GPU_DTYPE: the inventory WITH the running pods' allocations applied
    empty: np.ndarray         # GPU_DTYPE: the same inventory with nothing allocated
    node_off: np.ndarray
    table: np.ndarray
    run_claims: np.ndarray    # CLAIM_DTYPE, one OutRec slot each (run_out_off None)
    run_pod_off: np.ndarray
    run_prio: np.ndarray      # int32
    run_out: np.ndarray       # OUT_DTYPE
    claims: np.ndarray        # pending pods' claims (node fields 0: the call ignores them)
    pod_off: np.ndarray
    prio: np.ndarray          # int32


def preempt(n_node: int = 16, gpus_per_node: int = 8, n_pending: int = 64, seed: int = 0, fill: int = 90,
            mig_nodes: int = 3, prio_lo: int = -100, prio_hi: int = 1000, pending_prio: int | None = None,
            shared_per_gpu: int = 6, shapes=("3g", "7g", "2x3g", "gpu2"),
            tiles=(R.GI_1_SLICE, R.GI_1_SLICE, R.GI_2_SLICE, R.GI_2_SLICE, R.GI_3_SLICE)) -> PreemptWorld:
    """Preemption workload (spec §14), built directly — no allocator runs.  Of every 4 nodes, `mig_nodes` are MIG nodes
    whose GPUs are tiled first-fit with running pods of the `tiles` profiles (1g, 2g, 3g) until `fill` % of the 8 slices are taken (the
    fragmented regime of cfg5); the other nodes' GPUs each carry a full-GPU pod, up to `shared_per_gpu` SHARED pods (time
    slicing or an MPS memory limit), or nothing.  Running pods take 1 or 2 claims, with seeded priorities in
    [prio_lo, prio_hi); pending pods are 3g, 7g, 2x3g (one co-location group) or N-GPU ("gpuN") pods at `pending_prio` (default:
    seeded in [prio_hi / 2, prio_hi + 100))."""
    g, off = R.make_inventory([gpus_per_node] * n_node, mig=True)
    r = splitmix64(BASE_SEED + 1400 + seed, 64 * len(g) * max(shared_per_gpu, 8) + 8 * n_pending + 64)
    pos = [0]

    def nxt(m):
        v = int(r[pos[0]] % np.uint64(m))
        pos[0] += 1
        return v

    mig_node = np.array([nxt(4) < mig_nodes for _ in range(n_node)])
    g["flags"] = np.repeat(np.where(mig_node, R.GPU_MIG_ENABLED, 0), gpus_per_node).astype(np.uint8)
    empty = g.copy()
    rc, ro, pods, rprio = [], [], [], []
    size_of = {R.GI_1_SLICE: (1, range(0, 7)), R.GI_2_SLICE: (2, (0, 2, 4)), R.GI_3_SLICE: (4, (0, 4))}

    def claim(kind, prof, node, mem=0):
        c = np.zeros(1, dtype=R.CLAIM_DTYPE)[0]
        c["kind"], c["profile"], c["count"], c["node"], c["mem_limit_mib"] = kind, prof, 1, node, mem
        return c

    def out(gpu, start, size, prof):
        o = np.zeros(1, dtype=R.OUT_DTYPE)[0]
        o["gpu"], o["start"], o["size"], o["profile"], o["status"] = gpu, start, size, prof, R.ST_OK
        return o

    pending = []                # claims of the running pod being built: (claim, out)
    for n in range(n_node):
        for gi in range(off[n], off[n + 1]):
            if mig_node[n]:
                tries = 0
                while bin(int(g["busy"][gi])).count("1") * 100 < fill * 8 and tries < 24:
                    tries += 1
                    prof = tiles[nxt(len(tiles))]
                    size, starts = size_of[prof]
                    for s in starts:
                        m = ((1 << size) - 1) << s
                        if not (int(g["busy"][gi]) & m):
                            g["busy"][gi] |= m
                            pending.append((claim(R.KIND_MIG, prof, n), out(gi, s, size, prof)))
                            break
                    if pending and (nxt(4) != 0 or len(pending) == 2):
                        pods.append(pending); pending = []
            else:
                k = nxt(8)
                if k < 2:
                    g["flags"][gi] |= R.GPU_FULL_ALLOCATED
                    pods.append([(claim(R.KIND_GPU, R.PROFILE_GPU, n), out(gi, 0, 0, R.PROFILE_GPU))])
                elif k < 7:
                    for _ in range(1 + nxt(max(shared_per_gpu, 1))):
                        mem = (0, 0, 1024, 2048, 4096)[nxt(5)]
                        if g["mem_free_mib"][gi] < mem:
                            continue
                        g["mem_free_mib"][gi] -= mem
                        g["share_cnt"][gi] += 1
                        c = claim(R.KIND_SHARED, 0, n, mem)
                        c["profile"] = 0
                        pods.append([(c, out(gi, 0, 0, R.PROFILE_SHARED))])
            if pending:
                pods.append(pending); pending = []
    run_pod_off = np.zeros(len(pods) + 1, dtype=np.uint32)
    run_pod_off[1:] = np.cumsum([len(p) for p in pods])
    run_claims = np.array([c for p in pods for c, _ in p], dtype=R.CLAIM_DTYPE)
    run_out = np.array([o for p in pods for _, o in p], dtype=R.OUT_DTYPE)
    span = max(prio_hi - prio_lo, 1)
    run_prio = np.array([prio_lo + nxt(span) for _ in pods], dtype=np.int32)
    cl, pod_off, prio = [], [0], []
    for q in range(n_pending):
        shape = shapes[nxt(len(shapes))]
        if shape == "3g":
            cl.append(claim(R.KIND_MIG, R.GI_3_SLICE, 0))
        elif shape == "7g":
            cl.append(claim(R.KIND_MIG, R.GI_7_SLICE, 0))
        elif shape == "2x3g":
            for _ in range(2):
                c = claim(R.KIND_MIG, R.GI_3_SLICE, 0)
                c["group"] = q + 1
                cl.append(c)
        else:                                          # "gpu<N>": one claim of N full GPUs
            c = claim(R.KIND_GPU, 0, 0)
            c["count"] = int(shape[3:])
            cl.append(c)
        pod_off.append(len(cl))
        prio.append(pending_prio if pending_prio is not None else prio_hi // 2 + nxt(prio_hi // 2 + 100))
    return PreemptWorld(g, empty, off, R.default_table(), run_claims if len(run_claims) else np.zeros(0, R.CLAIM_DTYPE),
                        run_pod_off, run_prio, run_out if len(run_out) else np.zeros(0, R.OUT_DTYPE),
                        np.array(cl, dtype=R.CLAIM_DTYPE), np.array(pod_off, dtype=np.uint32),
                        np.array(prio, dtype=np.int32))
