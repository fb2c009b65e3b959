"""Random Allocate problems at the limits of the records and of the packing loops — TEST INFRASTRUCTURE ONLY, needs no GPU.

The packing warp cuts a node's claims into segments of 32 and picks one of three loops per segment: the lean plain-MIG loop
of a homogeneous node (3 shift steps when the node's table row has no cell larger than 8 slices, 4 otherwise), the lean
SHARED loop, or the generic step; co-location runs take the generic step and may carry over a segment boundary, and the
dead-shape memo lives across segments.  tests/test_oracle_properties.py's generator never reaches most of that (8-slice
tables, at most 9 GPUs and 24 claims per problem, benign memory values).  This one draws:
  tables      1-4 models with ids 0-15; shapes of 1-16 slices at starts anywhere in 16 bits (size 16 at 0, size 1 at 15);
              rows of shapes <= 8 slices, rows whose largest shape is exactly 9, rows with one larger shape, wide rows,
              and rows with an unoffered cell (start mask 0) whose size byte is above 8
  inventory   1-6 nodes of 0-32 GPUs (0, 1, 7, 8, 9, 15, 16, 17, 31, 32 and random), homogeneous and mixed-model nodes,
              busy over all 16 bits, every combination of the three flag bits, share counts 0, 1, 0xFFFE, 0xFFFF and
              random, free memory 0, 1, 0xFFFFFFFE, 0xFFFFFFFF and random
  claims      up to a few hundred, nodes given 31, 32, 33, 64 or 65 claims, whole segments of plain MIG or of SHARED
              claims, co-location runs started at positions 29-33 of a node's order and runs of 32 and 33 members, GPU
              counts 0-33, SHARED limits 0, 1, a GPU's free memory, 0xFFFFFFFE and 0xFFFFFFFF, the largest shape of a
              row asked again after it failed, malformed claims and claims naming no node
The same builder draws from hypothesis (`problems()`) or from a seeded numpy generator (`random_problem`).  `features()`
says, from the oracle's answer, which of the branches above a problem reached, so the suites can require that a fixed
example set keeps reaching them."""
from __future__ import annotations

import importlib
from collections import Counter
from dataclasses import dataclass

import numpy as np
from hypothesis import strategies as st

from preempt_problems import _Hyp, _Rng

R = importlib.import_module("k8s-dra-driver_b200").records
NONE = 0xFFFFFFFF
U32 = 0xFFFFFFFF
WIDTHS = (0, 1, 7, 8, 9, 15, 16, 17, 31, 32)
NODE_CLAIMS = (31, 32, 33, 64, 65)
SEG = 32


@dataclass
class Problem:
    gpus: np.ndarray
    node_off: np.ndarray
    table: np.ndarray
    claims: np.ndarray
    out_off: np.ndarray
    n_out: int

    @property
    def n_node(self):
        return len(self.node_off) - 1


def _starts(D, size):
    hi = 16 - size
    how = D.int(0, 5)
    if how == 0:
        return [0]
    if how == 1:
        return [hi]
    if how == 2:
        return list(range(0, hi + 1, max(1, size)))
    return sorted({D.int(0, hi) for _ in range(D.int(1, 4))})


def _row(D, t, m):
    """one model's row: ("small", "junk", "nine", "one_big", "wide")"""
    kind = D.pick(("small", "small", "junk", "nine", "one_big", "wide"))
    profs = sorted({D.int(0, 15) for _ in range(D.int(1, 7))})
    for p in profs:
        size = D.int(1, 16) if kind == "wide" else D.pick((1, 1, 2, 2, 3, 4, 5, 6, 7, 8))
        t[m, p] = (size, 0, R.mask_of(_starts(D, size)))
    if kind in ("nine", "one_big"):                       # exactly one shape above 8 slices
        p = D.pick(profs)
        size = 9 if kind == "nine" else D.int(9, 16)
        t[m, p] = (size, 0, R.mask_of(_starts(D, size)))
    if kind == "junk":                                    # an unoffered cell whose size byte is above 8
        free = [p for p in range(16) if p not in profs]
        t[m, D.pick(free)] = (D.pick((9, 12, 16)), 0, 0)
    return kind


def _offered(t, m):
    return [p for p in range(16) if t[m, p]["start_mask"]]


def build(D, scale: int = 1) -> Problem:
    t = R.empty_table()
    models = sorted({D.int(0, 15) for _ in range(D.int(1, 4))})
    for m in models:
        _row(D, t, m)
    n_node = D.int(1, 6)
    widths = [D.pick(WIDTHS) if D.int(0, 3) else D.int(0, 32) for _ in range(n_node)]
    g, off = R.make_inventory(widths, mig=True)
    style = []
    for n in range(n_node):
        s = D.pick(("mig", "mig", "mig", "plain", "plain", "mixed"))
        homog = D.int(0, 2) > 0
        m0 = D.pick(models)
        for i in range(int(off[n]), int(off[n + 1])):
            g["model"][i] = m0 if homog else D.pick(models)
            base = {"mig": 1, "plain": 0, "mixed": D.int(0, 1)}[s]
            g["flags"][i] = base if D.int(0, 4) else D.int(0, 7)           # all 8 combinations of the flag bits
            b = D.pick((0, 0, 1, 2, 3, 4))
            g["busy"][i] = (0, D.int(0, 0xFFFF) & D.int(0, 0xFFFF), D.int(0, 0xFF) << 8, 1 << D.int(0, 15),
                            D.int(0, 0xFFFF))[b] if b else 0
            g["mem_free_mib"][i] = D.pick((0, 1, U32 - 1, U32, U32, D.int(0, U32), 40960, 81920))
            g["share_cnt"][i] = D.pick((0, 0, 0, 0, 1, 0xFFFE, 0xFFFF, D.int(0, 0xFFFF)))
        style.append(s)

    gid = [0]
    per_node = []
    for n in range(n_node):
        gpus = range(int(off[n]), int(off[n + 1]))
        mods = sorted({int(g["model"][i]) for i in gpus}) or [D.pick(models)]
        offered = sorted({p for m in mods for p in _offered(t, m)}) or [D.int(0, 15)]
        biggest = max(offered, key=lambda p: max(int(t[m, p]["size"]) for m in mods))
        exact = D.int(0, 4) > 0
        target = D.pick(NODE_CLAIMS + NODE_CLAIMS + (0, 1, 5, 12)) if exact else D.int(0, 100 * scale)
        seq = []

        def mig(profile=None, group=0):
            c = np.zeros(1, R.CLAIM_DTYPE)[0]
            c["kind"], c["count"], c["node"], c["group"] = R.KIND_MIG, 1, n, group
            c["profile"] = profile if profile is not None else (
                D.pick(offered) if D.int(0, 9) else D.pick((D.int(0, 15), 16, 200)))
            return c

        def shared(limit=None):
            c = np.zeros(1, R.CLAIM_DTYPE)[0]
            c["kind"], c["count"], c["node"] = R.KIND_SHARED, 1, n
            eq = int(g["mem_free_mib"][D.pick(list(gpus))]) if len(gpus) else 0
            c["mem_limit_mib"] = limit if limit is not None else D.pick((0, 0, 1, eq, eq, U32 - 1, U32, 1000, 20000,
                                                                         D.int(0, U32)))
            return c

        def gpu():
            c = np.zeros(1, R.CLAIM_DTYPE)[0]
            c["kind"], c["node"] = R.KIND_GPU, n
            c["count"] = D.pick((1, 1, 1, 2, 3, D.int(1, 32), 16, 17, 31, 32, 0, 33))
            return c

        def bad():
            c = np.zeros(1, R.CLAIM_DTYPE)[0]
            c["kind"], c["node"], c["count"] = D.pick(((3, n, 1), (255, n, 1), (1, n, 1), (0, n, 0), (0, n, 33)))
            c["profile"] = D.pick((16, 200)) if c["kind"] == 1 else 0
            return c

        kinds = {"mig": ("mig", "mig", "mig", "run", "big", "bad", "mixed"),
                 "plain": ("shared", "shared", "shared", "clean_sh", "gpu", "bad", "mixed"),
                 "mixed": ("mig", "shared", "gpu", "run", "big", "mixed")}[style[n]]
        while len(seq) < target:
            blk = D.pick(kinds)
            k = D.pick((1, 2, 3, 5, 8, SEG - len(seq) % SEG, SEG))     # a block may fill the segment exactly
            if blk == "mig":
                seq += [mig() for _ in range(k)]
            elif blk == "shared":
                seq += [shared() for _ in range(k)]
            elif blk == "clean_sh":                                    # a segment of SHARED claims that all fit, then 2^32-1
                seq += [shared(0) for _ in range(SEG - len(seq) % SEG)] + [shared(U32)]
            elif blk == "gpu":
                seq += [gpu() for _ in range(min(k, 4))]
            elif blk == "bad":
                seq.append(bad())
            elif blk == "big":                                         # the largest shape, asked again later
                seq += [mig(biggest) for _ in range(D.int(1, 3))]
            elif blk == "mixed":
                seq += [D.pick((mig, shared, gpu, mig))() for _ in range(k)]
            else:                                                      # a co-location run, often across a boundary
                if D.int(0, 2):
                    at = D.int(29, 33) + SEG * D.int(0, 1)
                    while len(seq) < at:
                        seq.append(mig())
                gid[0] += 1
                size = D.pick((2, 3, 4, 5, 2, 32, 33))
                small = [p for p in offered if all(int(t[m, p]["size"]) <= 2 for m in mods)] or offered
                seq += [mig(D.pick(small), gid[0]) for _ in range(size)]
                if D.int(0, 1):                                        # a plain claim right after: the run's end
                    seq.append(mig())
        per_node.append(seq[:target] if exact else seq)

    # input order: the nodes' sequences merged at random (each keeps its own order), claims naming no node in between
    heads = [0] * n_node
    claims = []
    left = sum(len(s) for s in per_node)
    while left:
        n = D.pick([i for i in range(n_node) if heads[i] < len(per_node[i])])
        for _ in range(D.int(1, 8)):
            if heads[n] < len(per_node[n]):
                claims.append(per_node[n][heads[n]])
                heads[n] += 1
                left -= 1
        if D.int(0, 15) == 0:
            c = np.zeros(1, R.CLAIM_DTYPE)[0]
            c["kind"], c["count"], c["node"] = D.pick((0, 1, 2)), D.pick((1, 2, 40)), D.pick((n_node, n_node + 7, NONE))
            claims.append(c)
    c = np.array(claims, dtype=R.CLAIM_DTYPE) if claims else np.zeros(0, R.CLAIM_DTYPE)
    out_off, n_out = R.out_offsets(c, n_node)
    return Problem(g, off, t, c, out_off, n_out)


@st.composite
def problems(draw):
    return build(_Hyp(draw))


def random_problem(seed: int, scale: int = 1) -> Problem:
    return build(_Rng(np.random.default_rng(seed)), scale)


# ---- which branches a problem reached ----------------------------------------------------------------------------------
def _runs(c, q):
    """co-location runs of a node's order q (spec §6): [(position, length)]"""
    res, k = [], 0
    while k < len(q):
        x = c[q[k]]
        if x["kind"] == R.KIND_MIG and x["group"] and x["profile"] < 16:
            e = k + 1
            while (e < len(q) and e - k < R.MAX_GROUP and c[q[e]]["kind"] == R.KIND_MIG
                   and c[q[e]]["group"] == x["group"] and c[q[e]]["profile"] < 16):
                e += 1
            res.append((k, e - k))
            k = e
        else:
            k += 1
    return res


def _valid(x, n_node):
    if x["kind"] > 2 or x["node"] >= n_node:
        return False
    if x["kind"] == R.KIND_GPU:
        return 1 <= x["count"] <= 32
    return x["kind"] != R.KIND_MIG or x["profile"] < 16


def features(pb: Problem, out: np.ndarray) -> Counter:
    """The branches of the packing loops the problem reached, from the oracle's OutRecs `out`."""
    f = Counter()
    g, off, t, c, oo = pb.gpus, pb.node_off, pb.table, pb.claims, pb.out_off
    n_node = pb.n_node
    for n in range(n_node):
        g0, g1 = int(off[n]), int(off[n + 1])
        q = [i for i in range(len(c)) if c[i]["node"] == n]
        if len(q) in NODE_CLAIMS:
            f[f"claims_{len(q)}"] += 1
        mods = {int(g["model"][i]) for i in range(g0, g1)}
        homog = len(mods) <= 1
        sizes = {m: [int(t[m, p]["size"]) for p in range(16)] for m in mods}
        small8 = homog and all(s <= 8 for v in sizes.values() for s in v)
        row_max = max((s for v in sizes.values() for s in v), default=0)
        ok_any = any(out[oo[i]]["status"] == R.ST_OK for i in q)
        if 17 <= g1 - g0 and ok_any:
            f["node_17_32"] += 1
        if not homog and any(max(v) > 8 for v in sizes.values()) and any(max(v) <= 8 for v in sizes.values()):
            f["hetero_wide_and_small"] += 1
        runs = _runs(c, q)
        covered = set()
        for k, ln in runs:
            covered.update(range(k + 1, k + ln))
            if k // SEG != (k + ln - 1) // SEG:
                f["run_crosses_segment"] += 1
                if out[oo[q[k]]]["status"] == R.ST_OK:
                    f["run_crosses_segment_ok"] += 1
            if ln == 32:
                f["run_32"] += 1
        for k in range(len(q) - 32):
            if all(c[q[k + j]]["kind"] == R.KIND_MIG and c[q[k + j]]["group"] == c[q[k]]["group"] != 0
                   for j in range(33)):
                f["run_cut_at_33"] += 1
                break
        # replay the node: free memory / share counts as each claim sees them
        mem = {i: int(g["mem_free_mib"][i]) for i in range(g0, g1)}
        share = {i: int(g["share_cnt"][i]) for i in range(g0, g1)}
        clean_sh_seg = False                      # an all-SHARED segment without a failure came earlier
        dead = {}                                 # MIG profile -> segment where it failed
        for s0 in range(0, len(q), SEG):
            seg = range(s0, min(s0 + SEG, len(q)))
            val = [k for k in seg if _valid(c[q[k]], n_node) and k not in covered]
            in_run = any(k in covered for k in seg if k == s0)
            plain_mig = val and not in_run and all(c[q[k]]["kind"] == R.KIND_MIG and not c[q[k]]["group"] for k in val)
            all_sh = val and not in_run and all(c[q[k]]["kind"] == R.KIND_SHARED for k in val)
            fast = homog and g1 > g0 and plain_mig
            sh_fail = False
            for k in seg:
                i = q[k]
                x, o = c[i], out[oo[i]]
                ok = o["status"] == R.ST_OK
                if x["kind"] == R.KIND_MIG and _valid(x, n_node) and not x["group"]:
                    if ok and o["start"] >= 8:
                        f["start_ge8_ok"] += 1
                    if ok and o["size"] == 16:
                        f["size16_ok"] += 1
                    if fast and ok:
                        f["fast3_ok" if small8 else "fast4_ok"] += 1
                        if o["size"] >= 9:
                            f["fast_9_16_ok"] += 1
                    if fast and row_max == 9 and any(int(t[m, x["profile"]]["size"]) == 9 for m in mods):
                        f["fast_size9_row_max9"] += 1
                    if fast and not small8 and all(t[m, p]["size"] <= 8 for m in mods for p in range(16)
                                                   if t[m, p]["start_mask"]):
                        f["fast_small_row_junk_cell"] += 1
                    p = int(x["profile"])
                    if p in dead and dead[p] < s0 // SEG:
                        f["dead_shape_asked_in_later_segment"] += 1
                    if not ok and p not in dead:
                        dead[p] = s0 // SEG
                    if ok and not homog and int(g["model"][o["gpu"]]) != int(g["model"][g0]):
                        f["hetero_placed_off_lane0_model"] += 1
                if x["kind"] == R.KIND_SHARED and _valid(x, n_node):
                    lim = int(x["mem_limit_mib"])
                    if all_sh:
                        blocked = [j for j in range(g0, g1) if not (g["flags"][j] & 7) and mem[j] >= lim
                                   and share[j] == 0xFFFF and (not ok or j < o["gpu"])]
                        if blocked:
                            f["fast_sh_skips_share_ffff"] += 1
                    if ok:
                        j = int(o["gpu"])
                        if lim == mem[j] and lim:
                            f["shared_limit_eq_free_ok"] += 1
                        if lim == U32:
                            f["shared_limit_max_ok"] += 1
                            if clean_sh_seg:
                                f["limit_max_ok_after_clean_sh_segment"] += 1
                        mem[j] -= lim
                        share[j] += 1
                        if share[j] == 0xFFFF:
                            f["share_reaches_ffff"] += 1
                    else:
                        sh_fail = True
                if x["kind"] == R.KIND_GPU and ok and x["count"] >= 17:
                    f["gpu_count_17_32_ok"] += 1
            if all_sh:
                f["sh_segment"] += 1
                clean_sh_seg = clean_sh_seg or not sh_fail
    return f


POD_SIZES = (1, 2, 3, 1, 4, 2, 6, 1, 3, 33, 2, 5)


def pods(pb: Problem, first: int = 0):
    """The problem's claims cut into consecutive pods (sizes cycle through POD_SIZES from index `first`), every claim of a
    pod naming the node of its first claim.  Returns (claims, pod_off, out_off, n_out)."""
    c = pb.claims.copy()
    off, k, i = [0], first, 0
    while i < len(c):
        e = min(len(c), i + POD_SIZES[k % len(POD_SIZES)])
        c["node"][i:e] = c["node"][i]
        off.append(e)
        i, k = e, k + 1
    oo, n_out = R.out_offsets(c, pb.n_node)
    return c, np.array(off, np.uint32), oo, n_out
