"""Random spec §14 (preemption) problems for the CPU and GPU suites — TEST INFRASTRUCTURE ONLY, needs no GPU.

A problem is an inventory of mixed widths (0 to 32 GPUs per node, MIG and non-MIG nodes, models 0 and 1 of
records.default_table(), now and then an UNAVAILABLE GPU), running pods placed on it by the oracle's pods Allocate (so
their records match the inventory), optionally perturbed afterwards into records that do not match it, priorities drawn
from a pool with the int32 extremes and many ties, pending pods of 0 to 33 claims, and candidate lists with duplicates,
strays and more than 32 entries.  The same builder draws from hypothesis (`problems()`) or from a seeded numpy generator
(`random_problem`), so the GPU suite can also make larger problems of the same kind without hypothesis.  `build_place`
makes spec §15 (preempt and place) problems of the same kind, with the pending pods' out_off in one of four forms."""
from __future__ import annotations

import dataclasses
import importlib
from dataclasses import dataclass

import numpy as np
from hypothesis import strategies as st

import preempt_oracle as P
from oracle import oracle as O

R = importlib.import_module("k8s-dra-driver_b200").records
NONE = 0xFFFFFFFF
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
PRIOS = (I32_MIN, I32_MIN + 1, -1, 0, 1, I32_MAX - 1, I32_MAX, 7, 7)
WIDTHS = (0, 1, 1, 2, 2, 3, 3, 8, 9, 16, 17, 32)


@dataclass
class Problem:
    gpus: np.ndarray
    node_off: np.ndarray
    table: np.ndarray
    claims: np.ndarray            # pending pods
    pod_off: np.ndarray
    prio: np.ndarray
    cands: list | None            # one list of node indices per pod, or None: the dense form
    run_claims: np.ndarray
    run_pod_off: np.ndarray
    run_prio: np.ndarray
    run_out: np.ndarray
    run_out_off: np.ndarray | None
    max_victims: int
    flags: int                    # 0 or F_EXHAUSTIVE
    matched: bool                 # the running records are exactly what the inventory holds
    error: bool                   # a call-level error of §14: the call must fail with nothing written
    what: str = ""                # the perturbations applied

    @property
    def n_node(self):
        return len(self.node_off) - 1

    def cand_arrays(self):
        if self.cands is None:
            return None, None
        off = np.zeros(len(self.cands) + 1, np.uint32)
        off[1:] = np.cumsum([len(x) for x in self.cands])
        return np.array([n for x in self.cands for n in x], dtype=np.uint32), off

    def oracle(self, gpus=None, flags=None, max_victims=None):
        """preempt_oracle.preempt on this problem (on `gpus` when given); raises ValueError on a call-level error"""
        cn, co = self.cand_arrays()
        return P.preempt(self.gpus if gpus is None else gpus, self.node_off, self.table, self.claims, self.pod_off,
                         self.prio, self.run_claims, self.run_pod_off, self.run_prio, self.run_out, self.run_out_off, cn,
                         co, self.max_victims if max_victims is None else max_victims,
                         self.flags if flags is None else flags)


class _Hyp:
    def __init__(self, draw):
        self.d = draw

    def int(self, lo, hi):
        return self.d(st.integers(lo, hi))

    def pick(self, seq):
        return self.d(st.sampled_from(seq))


class _Rng:
    def __init__(self, rng):
        self.r = rng

    def int(self, lo, hi):
        return int(self.r.integers(lo, hi + 1))

    def pick(self, seq):
        return seq[int(self.r.integers(0, len(seq)))]


def _inventory(D, n_node):
    widths = [D.pick(WIDTHS) for _ in range(n_node)]
    if not sum(widths):
        widths[-1] = 1                                   # an inventory holds at least one GPU
    g, off = R.make_inventory(widths, mig=False)
    mig = [D.pick((0, 1, 1, 2)) for _ in range(n_node)]       # 2: MIG and non-MIG GPUs on one node
    for i in range(len(g)):
        n = int(g["node"][i])
        g["model"][i] = D.pick((0, 0, 1))
        on = mig[n] == 1 or (mig[n] == 2 and D.int(0, 1) == 1)
        g["flags"][i] = (R.GPU_MIG_ENABLED if on else 0) | D.pick((0,) * 11 + (R.GPU_UNAVAILABLE,))
        g["mem_free_mib"][i] = D.pick((40960, 81920, 16384))
    return g, off, mig


def _running_claims(D, n, mig, have_off):
    """the claims of one running pod on node n"""
    k = D.pick((1, 1, 1, 2, 3))
    c = np.zeros(k, R.CLAIM_DTYPE)
    c["node"], c["count"] = n, 1
    for i in range(k):
        kind = D.pick((R.KIND_MIG,) * 5 + (R.KIND_GPU,)) if mig else D.pick((R.KIND_GPU, R.KIND_SHARED, R.KIND_SHARED,
                                                                              R.KIND_MIG))
        c[i]["kind"] = kind
        if kind == R.KIND_MIG:
            c[i]["profile"] = D.pick((R.GI_1_SLICE, R.GI_1_SLICE, R.GI_2_SLICE, R.GI_3_SLICE))
        elif kind == R.KIND_GPU:
            c[i]["count"] = D.int(1, 4) if have_off else 1
        else:
            c[i]["mem_limit_mib"] = D.pick((0, 0, 5000, 20000))
    return c


def _slots(rc, n_node, have_off):
    return R.claim_slots(rc, n_node, have_off)


def _pending(D, n_node):
    n_pod = D.int(0, 6)
    claims, pod_off, prio = [], [0], []
    for _ in range(n_pod):
        k = D.pick((0, 1, 1, 1, 2, 2, 3, 4, 6, 33))
        gid = D.pick((0, 0, 1, 2))
        kinds = D.pick(((1,), (1,), (1,), (0, 2, 2), (0, 2, 2), (1, 1, 1, 1, 0, 0, 2, 2)))   # MIG, non-MIG or both
        for _ in range(k):
            c = np.zeros(1, R.CLAIM_DTYPE)[0]
            kind = D.pick(kinds)
            c["kind"], c["count"], c["node"] = kind, 1, D.pick((0, n_node, NONE))   # the node field is ignored
            if kind == R.KIND_MIG:
                c["profile"] = D.pick((R.GI_1_SLICE, R.GI_1_SLICE, R.GI_2_SLICE, R.GI_3_SLICE, R.GI_7_SLICE,
                                       R.GI_7_SLICE, R.GI_4_SLICE, R.GI_8_SLICE))      # 8g: offered by no model
                c["group"] = gid if D.int(0, 2) == 0 else 0
            elif kind == R.KIND_GPU:
                c["count"] = D.pick((1, 1, 2, 3, 4))
            else:
                c["mem_limit_mib"] = D.pick((0, 5000, 20000, 40960))
            if D.int(0, 24) == 0:                         # an invalid claim: unknown kind or profile, count 0 or > 32
                c["kind"], c["profile"], c["count"] = D.pick(((3, 0, 1), (1, 16, 1), (1, 200, 1), (0, 0, 0), (0, 0, 33)))
            claims.append(c)
        pod_off.append(len(claims))
        prio.append(D.pick(PRIOS + (I32_MAX, I32_MAX, I32_MAX - 1, 7, 7)))
    c = np.array(claims, dtype=R.CLAIM_DTYPE) if claims else np.zeros(0, R.CLAIM_DTYPE)
    return c, np.array(pod_off, np.uint32), np.array(prio, np.int32)


def _cands(D, n_pod, n_node):
    if D.int(0, 2) == 0:
        return None
    pool = list(range(n_node)) + [n_node, n_node + 1, NONE]
    out = []
    for _ in range(n_pod):
        k = D.pick((0, 1, 2, 3, 3, 5, 8, 33, 40))
        if k > 8:                                        # long lists: one node many times, now and then another
            a, b = D.pick(pool), D.pick(pool)
            out.append([b if D.int(0, 7) == 0 else a for _ in range(k)])
        else:
            out.append([D.pick(pool) for _ in range(k)])
    return out


def _ok_slots(rc, rpo, ro, roo, n_node):
    """[(running pod, claim, slot index)] of the OK slots"""
    have_off = roo is not None
    sl = _slots(rc, n_node, have_off)
    res = []
    for r in range(len(rpo) - 1):
        for i in range(int(rpo[r]), int(rpo[r + 1])):
            base = int(roo[i]) if have_off else i
            for k in range(int(sl[i])):
                if base + k < len(ro) and ro[base + k]["status"] == R.ST_OK:
                    res.append((r, i, base + k))
    return res


def _perturb(D, g, off, rc, rpo, rpr, ro, roo):
    """records that no longer match the inventory, still valid arguments; returns (rc, rpo, rpr, ro, roo, names)"""
    n_node = len(off) - 1
    names = []
    for _ in range(D.int(1, 3)):
        what = D.pick(("status", "mig_range", "no_node", "kind", "wrap", "retarget", "empty_pod", "no_ok",
                       "count_no_off"))
        ok = _ok_slots(rc, rpo, ro, roo, n_node)
        if what == "status" and ok:
            _, _, s = D.pick(ok)
            ro[s]["status"] = D.pick((R.ST_NO_CAPACITY, R.ST_INVALID, R.ST_POD, R.ST_SEARCH_LIMIT))
        elif what == "mig_range":
            mig = [s for _, i, s in ok if rc[i]["kind"] == R.KIND_MIG]
            if mig:
                s = D.pick(mig)
                ro[s]["start"], ro[s]["size"] = D.pick(((16, 1), (200, 4), (12, 8), (15, 16), (0, 16), (3, 20),
                                                         (8, 255), (16, 16)))
        elif what == "no_node" and len(rc):
            i = D.int(0, len(rc) - 1)
            rc[i]["node"] = D.pick((n_node, n_node + 2, NONE))
            if rc[i]["kind"] == R.KIND_GPU:
                rc[i]["count"] = D.int(2, 4)
        elif what == "kind" and len(rc):
            i = D.int(0, len(rc) - 1)
            if rc[i]["kind"] != R.KIND_GPU or rc[i]["count"] == 1:
                rc[i]["kind"] = D.pick((R.KIND_GPU, R.KIND_MIG, R.KIND_SHARED))
                if rc[i]["kind"] == R.KIND_SHARED:
                    rc[i]["mem_limit_mib"] = D.pick((0, 5000))
        elif what == "wrap":
            sh = [i for _, i, _ in ok if rc[i]["kind"] == R.KIND_SHARED]
            if sh:
                rc[D.pick(sh)]["mem_limit_mib"] = D.pick((0xFFFFFFFF, 0xFFFF0000, 0x80000000, 90000))
        elif what == "retarget" and ok:
            _, _, s = D.pick(ok)
            n = int(g["node"][ro[s]["gpu"]])
            ro[s]["gpu"] = D.int(int(off[n]), int(off[n + 1]) - 1)
        elif what == "empty_pod":
            r = D.int(0, len(rpo) - 1)
            rpo = np.insert(rpo, r, rpo[r]).astype(np.uint32)
            rpr = np.insert(rpr, min(r, len(rpr)), D.pick(PRIOS)).astype(np.int32)
        elif what == "no_ok" and ok:
            r, _, _ = D.pick(ok)
            for rr, _, s in ok:
                if rr == r:
                    ro[s]["status"] = R.ST_POD
        elif what == "count_no_off" and roo is None:
            gp = [i for i in range(len(rc)) if rc[i]["kind"] == R.KIND_GPU]
            if gp:
                rc[D.pick(gp)]["count"] = D.int(2, 4)
        else:
            continue
        names.append(what)
    return rc, rpo, rpr, ro, roo, names


def _break(D, g, off, rc, rpo, ro, roo):
    """one of §14's call-level errors on the running pods; returns (rc, rpo, ro, roo, name) or None when this problem
    has no room for the one drawn"""
    n_node = len(off) - 1
    what = D.pick(("gpu_range", "two_nodes", "slot_range"))
    ok = _ok_slots(rc, rpo, ro, roo, n_node)
    if what == "gpu_range" and ok:
        _, _, s = D.pick(ok)
        ro[s]["gpu"] = D.pick((len(g), len(g) + 3, NONE))
        return rc, rpo, ro, roo, what
    if what == "two_nodes" and ok:
        r, _, s = D.pick(ok)
        other = [i for i in range(len(g)) if g["node"][i] != g["node"][ro[s]["gpu"]]]
        both = [t for rr, _, t in ok if rr == r and t != s]
        if other and both:
            ro[D.pick(both)]["gpu"] = D.pick(other)
            return rc, rpo, ro, roo, what
        return None
    if what == "slot_range" and len(rc):
        if roo is not None:
            roo[D.int(0, len(rc) - 1)] = len(ro) + D.int(0, 2)
        else:
            ro = ro[:-1]
        return rc, rpo, ro, roo, what
    return None


def build(D, scale: int = 1) -> Problem:
    """One problem drawn through D (_Hyp or _Rng).  scale > 1 multiplies the node and running-pod counts."""
    t = R.default_table()
    n_node = D.int(1, 6 * scale)
    g, off, mig = _inventory(D, n_node)
    have_off = D.int(0, 1) == 1
    # the running pods, placed by the pods Allocate on the empty inventory: records that match it
    n_run = D.int(0, 40 * scale)
    hot = [n for n in range(n_node) if 1 <= off[n + 1] - off[n] <= 3] or list(range(n_node))   # nodes that fill up
    parts, rpo = [], [0]
    for _ in range(n_run):
        n = D.pick(hot) if D.int(0, 3) else D.int(0, n_node - 1)
        parts.append(_running_claims(D, n, mig[n], have_off))
        rpo.append(rpo[-1] + len(parts[-1]))
    for n in hot[:2 * scale]:                            # then fill some nodes up with one-claim pods
        if D.int(0, 2) == 0:
            continue
        for gi in range(int(off[n]), int(off[n + 1])):
            c = np.zeros(1, R.CLAIM_DTYPE)
            c["node"], c["count"] = n, 1
            if mig[n]:
                c["kind"], c["profile"] = R.KIND_MIG, R.GI_1_SLICE
                k = 7 if g["model"][gi] == 0 else 4
            else:
                c["kind"], c["mem_limit_mib"] = D.pick(((R.KIND_GPU, 0), (R.KIND_SHARED, 0), (R.KIND_SHARED, 20000)))
                k = 1 if c["kind"][0] == R.KIND_GPU else D.int(1, 3)
            for _ in range(k):
                parts.append(c.copy())
                rpo.append(rpo[-1] + 1)
    n_run = len(rpo) - 1
    rc =np.concatenate(parts) if parts else np.zeros(0, R.CLAIM_DTYPE)
    rpo = np.array(rpo, np.uint32)
    if have_off:
        roo, n_out = R.out_offsets(rc, n_node)
    else:
        roo, n_out = None, len(rc)
    ro, g = O.allocate_pods(g, off, t, rc, rpo, roo, n_out)
    ro = ro.copy()
    rpr = np.array([D.pick(PRIOS) for _ in range(n_run)], np.int32)
    matched, error, names = True, False, []
    if D.int(0, 3) == 0:
        rc, rpo, rpr, ro, roo, names = _perturb(D, g, off, rc, rpo, rpr, ro, roo)
        matched = not names
    if D.int(0, 11) == 0:
        b = _break(D, g, off, rc, rpo, ro, roo)
        if b is not None:
            rc, rpo, ro, roo, name = b
            matched, error, names = False, True, names + [name]
    claims, pod_off, prio = _pending(D, n_node)
    error = error and len(prio) > 0                      # with no pending pods the running pods are not examined
    return Problem(g, off, t, claims, pod_off, prio, _cands(D, len(prio), n_node), rc, rpo, rpr, ro, roo,
                   D.pick((0, 1, 3, 64)), D.pick((0, P.F_EXHAUSTIVE)), matched, error, ",".join(names))


@st.composite
def problems(draw):
    return build(_Hyp(draw))


def random_problem(seed: int, scale: int = 1) -> Problem:
    return build(_Rng(np.random.default_rng(seed)), scale)


# ---- spec §15 (preempt and place) -----------------------------------------------------------------------------------
OUT_FORMS = ("none", "packed", "gaps", "spare")


@dataclass
class PlaceProblem(Problem):
    """A §15 problem: a §14 problem with the pending pods' out_off (None: the call passes none) and n_out.  `error` is
    the §15 oracle's verdict on the call."""
    out_off: np.ndarray | None = None
    n_out: int = 0
    form: str = "none"

    def pp_oracle(self, gpus=None, flags=None, fill=None):
        """preempt_place_oracle.preempt_place on this problem (on `gpus` when given); raises ValueError on a call-level
        error"""
        import preempt_place_oracle as PP
        cn, co = self.cand_arrays()
        return PP.preempt_place(self.gpus if gpus is None else gpus, self.node_off, self.table, self.claims, self.pod_off,
                                self.prio, self.run_claims, self.run_pod_off, self.run_prio, self.run_out,
                                self.run_out_off, cn, co, self.out_off, self.n_out, self.flags if flags is None else flags,
                                fill)


def pending_out_off(D, claims, form):
    """(out_off, n_out) of the pending claims in one of OUT_FORMS; slots never overlap (where overlapping slots end up
    depends on the order in which pods on different nodes are applied, which §13 and §15 leave open)"""
    if form == "none":
        return None, len(claims)
    placed = claims.copy()
    placed["node"] = 0
    sl = R.claim_slots(placed, 1, True).astype(np.int64)
    if form == "gaps":                                   # claims laid out in a random order, with holes between them
        order = list(range(len(claims)))
        for i in range(len(order) - 1, 0, -1):
            j = D.int(0, i)
            order[i], order[j] = order[j], order[i]
        oo = np.zeros(len(claims), np.uint32)
        cur = 0
        for i in order:
            cur += D.pick((0, 0, 1, 3))
            oo[i] = cur
            cur += int(sl[i])
        return oo, cur + D.pick((0, 2))
    oo = np.concatenate([[0], np.cumsum(sl)[:-1]]).astype(np.uint32) if len(claims) else np.zeros(0, np.uint32)
    return oo, int(sl.sum()) + (D.int(1, 5) if form == "spare" else 0)


def as_place(pb: Problem, D, form: str, short: bool = False, judge: bool = True) -> PlaceProblem:
    """pb as a §15 problem, the pending out_off in `form` (drawn through D); short: n_out one slot short.  judge: set
    `error` from the oracle (otherwise pb's is kept)"""
    oo, n_out = pending_out_off(D, pb.claims, form)
    d = {f.name: getattr(pb, f.name) for f in dataclasses.fields(Problem)}
    x = PlaceProblem(**d, out_off=oo, n_out=max(n_out - 1, 0) if short else n_out, form=form)
    if judge:
        try:
            x.pp_oracle()
            x.error = False
        except ValueError:
            x.error = True
    x.what = f"{x.what} out_off {form}{' short' if short else ''}"
    return x


def build_place(D, scale: int = 1) -> PlaceProblem:
    """One §15 problem drawn through D: build()'s inventory, running pods, priorities, pending pods and candidates, and
    the pending out_off in one of OUT_FORMS.  Now and then n_out is one slot short (a call-level error)."""
    pb = build(D, scale)
    return as_place(pb, D, D.pick(OUT_FORMS), D.int(0, 15) == 0)


@st.composite
def place_problems(draw):
    return build_place(_Hyp(draw))


def random_place_problem(seed: int, scale: int = 1) -> PlaceProblem:
    return build_place(_Rng(np.random.default_rng(seed)), scale)
