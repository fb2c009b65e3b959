"""CPU suite: the fixtures of the exhaustive pod search's structural limits (spec §12), checked without a GPU.

The device search (pod_eval in dra_device.cuh) keeps its stack in two registers per lane: one bit per pod position
in `chosen`, one 4-bit start per position in `st_lo` (positions 0-15) and `st_hi` (16-31).  After a backtrack it
resumes past the (lane, start) it undid, and it counts descents against DRA_EXH_BUDGET.  The fixtures here sit on
those limits: pods of 31-33 claims, starts of 8 and above at positions 16 and above, resumes from start 15 and from
the last lane, and searches of exactly 4095, 4096 and 4097 descents.  tests/test_gpu_pod_search.py runs them on the
device against the oracle.

Each fixture is a literal node and pod.  `search` below restates the canonical search of spec §12 (GPUs ascending,
starts ascending, a descent per placement) without a budget and records every descent as (pod position, GPU,
start); the tests check that each fixture has the descent count it is named for and reaches the position, start or
lane it exists for, and that the C oracle and oracle/naive.py give it the expected status."""
import importlib

import numpy as np
import pytest

R = importlib.import_module("k8s-dra-driver_b200").records

# ---- the placement table of the fixtures ---------------------------------------------------------------------------
# model 0: the synthetic 16-slice part of synth.homog(wide16=True): 1g size 1 at any of 16 starts, 2g size 2 at even
# starts, 3g size 5 at 0/5/10, 4g size 8 at 0/8, 7g size 16 at 0.
# models 1..5: parts that offer one profile each (size 1, any of 16 starts).  A claim of profile PIN[i] can only go to
# the GPU of model 1 + i, so each level of a budget fixture has a number of choices that no other level changes, and
# the descent count is the sum of the products of the levels' choices.
PIN = (5, 6, 8, 10, 11)


def fixture_table():
    t = R.empty_table()
    t[0, R.GI_1_SLICE] = (1, 0, 0xFFFF)
    t[0, R.GI_2_SLICE] = (2, 0, 0x5555)
    t[0, R.GI_3_SLICE] = (5, 0, R.mask_of((0, 5, 10)))
    t[0, R.GI_4_SLICE] = (8, 0, R.mask_of((0, 8)))
    t[0, R.GI_7_SLICE] = (16, 0, 1)
    for i, p in enumerate(PIN):
        t[1 + i, p] = (1, 0, 0xFFFF)
    return t


G1, G2, G3, G4, G7 = R.GI_1_SLICE, R.GI_2_SLICE, R.GI_3_SLICE, R.GI_4_SLICE, R.GI_7_SLICE


def node(busy, flags=R.GPU_MIG_ENABLED, model=0):
    """One node's GPUs: busy masks, with per-GPU flags / models (scalars apply to every GPU)."""
    n = len(busy)
    g = np.zeros(n, dtype=R.GPU_DTYPE)
    g["busy"] = busy
    g["flags"] = flags
    g["model"] = model
    g["mem_free_mib"] = 40960
    return g


def claims(*specs):
    """('mig', profile[, group[, selector]]), ('gpu', count[, selector]), ('shared', mem_limit_mib[, selector])."""
    c = np.zeros(len(specs), dtype=R.CLAIM_DTYPE)
    for i, s in enumerate(specs):
        kind, a, rest = s[0], s[1], list(s[2:])
        if kind == "mig":
            c[i]["kind"], c[i]["profile"], c[i]["count"] = R.KIND_MIG, a, 1
            c[i]["group"] = rest[0] if rest else 0
            c[i]["mem_limit_mib"] = rest[1] if len(rest) > 1 else 0
        elif kind == "gpu":
            c[i]["kind"], c[i]["count"] = R.KIND_GPU, a
            c[i]["mem_limit_mib"] = rest[0] if rest else 0
        else:
            c[i]["kind"], c[i]["count"], c[i]["mem_limit_mib"] = R.KIND_SHARED, 1, a
            c[i]["group"] = rest[0] if rest else 0
    return c


def mig(*profiles, group=0):
    return claims(*[("mig", p, group) for p in profiles])


# ---- the canonical search, counted -----------------------------------------------------------------------------------
def search(gpus, table, pod, trace=True, cap=None):
    """Spec §12 step 3 on the node `gpus` for the MIG claims of `pod` (no budget; selectors are not modelled, and the
    pod's GPU / SHARED claims are assumed to succeed — they take only GPUs that are not MIG-enabled).
    Returns (placed, descents, trace): placed is None when the search was stopped after `cap` descents; trace lists
    every descent as (pod position, GPU, start).  Without a trace, failing subtrees are memoised on (level, busy
    masks, GPUs of the groups' first members): a failing subtree is explored completely, so its descent count
    depends on that state only."""
    pos = [i for i in range(len(pod)) if pod[i]["kind"] == R.KIND_MIG]
    busy = [int(b) for b in gpus["busy"]]
    usable = [(int(f) & 7) == R.GPU_MIG_ENABLED for f in gpus["flags"]]
    ent = [[(int(table[int(m), int(pod[i]["profile"])]["size"]), int(table[int(m), int(pod[i]["profile"])]["start_mask"]))
            for m in gpus["model"]] for i in pos]

    def options(lv, want):
        for g in range(len(busy)):
            size, mask = ent[lv][g]
            if not usable[g] or not mask or (want is not None and g != want):
                continue
            for s in range(16):
                m = ((1 << size) - 1) << s
                if (mask >> s) & 1 and not busy[g] & m:
                    yield g, s, m

    for lv in range(len(pos)):                           # pre-check: a claim with no placement at all sinks the pod
        if next(options(lv, None), None) is None:
            return False, 0, []
    gpu_of, n, log, memo = [None] * len(pos), [0], [], {}
    first = []                                           # level of each level's group's first member (or None)
    for lv, i in enumerate(pos):
        grp = int(pod[i]["group"])
        first.append(next((j for j in range(lv) if grp and int(pod[pos[j]]["group"]) == grp), None))

    class Cap(Exception):
        pass

    def rec(lv):
        if lv == len(pos):
            return True
        key = None
        if not trace:
            key = (lv, tuple(busy), tuple(gpu_of[j] for j in range(lv) if first[j] is None))
            if key in memo:
                n[0] += memo[key]
                return False
        n0 = n[0]
        want = gpu_of[first[lv]] if first[lv] is not None else None
        for g, s, m in list(options(lv, want)):
            n[0] += 1
            if cap is not None and n[0] > cap:
                raise Cap
            if trace:
                log.append((pos[lv], g, s))
            busy[g] |= m
            gpu_of[lv] = g
            if rec(lv + 1):
                return True
            busy[g] &= ~m
        if key is not None:
            memo[key] = n[0] - n0
        return False

    try:
        placed = rec(0)
    except Cap:
        return None, n[0], log
    return placed, n[0], log


def resumed(log):
    """The descents that were undone and followed by another choice at the same position: the points the device
    search resumes from, as (position, GPU, start)."""
    out = set()
    for k, (p, g, s) in enumerate(log):
        for p2, _, _ in log[k + 1:]:
            if p2 <= p:
                if p2 == p:
                    out.add((p, g, s))
                break
    return out


def expected_status(placed, descents):
    """Status of the exhaustive search from the counted search: the budget allows DRA_EXH_BUDGET descents."""
    if placed is None or descents > R.EXH_BUDGET:
        return R.ST_SEARCH_LIMIT
    return R.ST_OK if placed else R.ST_POD


# ---- fixtures --------------------------------------------------------------------------------------------------------
# Budget boundary.  Level 1 is a 1g on the model-0 GPU, levels 2.. are pinned profiles on their own GPUs; the claim
# after them (Z) is a model-0 profile that needs the slices of level 1's first choices.
# failing: Z needs all of GPU 0's free slices, so every leaf fails: descents = a1 + a1*a2 + a1*a2*a3 + ...
# succeeding: Z fails for level 1's first j choices and fits at the next one:
#   descents = j * (1 + a2 + a2*a3 + ...) + (levels on the successful path)
BUDGET = [
    # name, busy per GPU, models, pod, descents, placed
    ("fail_4095", [0xFFE0, 0xFFFC, 0xFFF8, 0xFE00, 0xC000], [0, 1, 2, 3, 4],
     claims(("mig", G1), ("mig", PIN[0]), ("mig", PIN[1]), ("mig", PIN[2]), ("mig", PIN[3]), ("mig", G3)), 4095, False),
    ("fail_4096", [0x0000, 0x8000, 0x0000], [0, 1, 2],
     claims(("mig", G1), ("mig", PIN[0]), ("mig", PIN[1]), ("mig", G7)), 4096, False),
    ("fail_4097", [0xFFFE, 0x0000, 0x8000, 0x0000], [0, 1, 2, 3],
     claims(("mig", G1), ("mig", PIN[0]), ("mig", PIN[1]), ("mig", PIN[2]), ("mig", G1)), 4097, False),
    ("ok_4095", [0xF800, 0xFFF8, 0xE000, 0xF000], [0, 1, 2, 3],
     claims(("mig", G1), ("mig", PIN[0]), ("mig", PIN[1]), ("mig", PIN[2]), ("mig", G4), ("mig", G1), ("mig", G1)), 4095, True),
    ("ok_4096", [0xF81F, 0xFFFE, 0xFFC0, 0xFE00, 0xC000], [0, 1, 2, 3, 4],
     claims(("mig", G1), ("mig", PIN[0]), ("mig", PIN[1]), ("mig", PIN[2]), ("mig", PIN[3]), ("mig", G3)), 4096, True),
    ("ok_4097", [0xF01F, 0xFFFE, 0xFFC0, 0xFE00, 0xC000], [0, 1, 2, 3, 4],
     claims(("mig", G1), ("mig", PIN[0]), ("mig", PIN[1]), ("mig", PIN[2]), ("mig", PIN[3]), ("mig", G3), ("mig", G1)), 4097, True),
]


def budget_fixtures():
    return [dict(name=n, gpus=node(b, model=m), pods=[p], descents=d, placed=ok) for n, b, m, p, d, ok in BUDGET]


def deep_fixtures():
    """Case 1: 32-GPU nodes of the 16-slice part and pods of 31-33 claims.  `pods` run in order on the node."""
    full = [0xFFFF] * 32
    fx = []
    # a. 32 x 1g, every GPU's lower half busy: every start is >= 8, positions 16-31 on GPUs 2 and 3
    fx.append(dict(name="deep_32_high_starts", gpus=node([0x00FF] * 32), pods=[mig(*[G1] * 32)], descents=32, placed=True,
                   reach=[(p, 2 + (p - 16) // 8, 8 + p % 8) for p in range(16, 32)]))
    # a'. 32 claims of mixed sizes: 2g / 3g / 1g at positions >= 16 with starts up to 15
    fx.append(dict(name="deep_32_mixed", gpus=node([0x0000, 0x0F0F] + [0x00FF] * 30),
                   pods=[mig(*([G1] * 12 + [G2] * 6 + [G3, G3] + [G2] * 4 + [G1] * 8))], descents=32, placed=True,
                   reach=[(16, 1, 12), (24, 2, 15), (31, 5, 9)]))
    # b. position 16 backtracks from starts 0..7 to 9, co-located with the 4g at 17 (slice 8 of GPU 1 busy)
    fx.append(dict(name="deep_backtrack_at_16", gpus=node([0x0000, 0x0100] + full[2:]),
                   pods=[claims(*[("mig", G1)] * 16 + [("mig", G1, 5), ("mig", G4, 5)])], descents=26, placed=True,
                   reach=[(16, 1, 9)], resume=[(16, 1, s) for s in range(8)]))
    # b'. the 1g at position 15 sits at start 15; its group's 2g at 16 cannot follow: back across 15/16, resume past
    # start 15, onto GPU 1
    fx.append(dict(name="deep_backtrack_across_16", gpus=node([0x0000, 0x0000] + full[2:]),
                   pods=[claims(*[("mig", G1)] * 15 + [("mig", G1, 3), ("mig", G2, 3)])], descents=18, placed=True,
                   reach=[(15, 1, 0), (16, 1, 2)], resume=[(15, 0, 15)]))
    # c. 31 GPU / SHARED claims (time-sliced SHARED claims stack on GPU 16), then one MIG claim at position 31
    flags = [0] * 20 + [R.GPU_MIG_ENABLED] * 12
    nonmig = [("gpu", 1) if k % 2 == 0 else ("shared", 0) for k in range(31)]
    fx.append(dict(name="deep_mig_at_31", gpus=node([0] * 20 + [0x00FF] + [0xFFFF] * 11, flags=flags),
                   pods=[claims(*nonmig, ("mig", G4))], descents=1, placed=True, reach=[(31, 20, 8)]))
    # d. 31 x 1g fill GPUs 0 and 1 but for one slice; the 7g needs an empty GPU.  Then a 7g and a 1g that must see the
    # node as it was before the failed pod.
    fx.append(dict(name="deep_31_then_fail", gpus=node([0x0000, 0x0000] + full[2:]),
                   pods=[mig(*([G1] * 31 + [G7])), mig(G7), mig(G1)], descents=None, placed=None))
    # e. 33 claims: malformed
    fx.append(dict(name="deep_33", gpus=node([0x0000] * 32), pods=[mig(*[G1] * 33), mig(G1)], descents=None, placed=None))
    return fx


def resume_fixtures():
    """Case 2: backtracks that resume from start 15 and from the last GPU (lane) of a 32-GPU node."""
    return [
        # 1g at GPU 0 start 15 (its only free slice), its group's 2g cannot follow: resume past (0, 15) -> GPU 1
        dict(name="resume_start_15", gpus=node([0x7FFF, 0x0000]), pods=[claims(("mig", G1, 1), ("mig", G2, 1))],
             descents=3, placed=True, reach=[(0, 1, 0), (1, 1, 2)], resume=[(0, 0, 15)]),
        # only GPU 31 is free, slice 8 busy: the 1g resumes on lane 31 from starts 0..7 before its 4g fits
        dict(name="resume_lane_31", gpus=node([0xFFFF] * 31 + [0x0100]), pods=[claims(("mig", G1, 1), ("mig", G4, 1))],
             descents=10, placed=True, reach=[(0, 31, 9), (1, 31, 0)], resume=[(0, 31, s) for s in range(8)]),
        # the same on the last GPU of an 8- and a 16-GPU node (UnsuitableNodes at W = 8 and 16 resumes on lane W - 1)
        dict(name="resume_lane_7", gpus=node([0xFFFF] * 7 + [0x0100]), pods=[claims(("mig", G1, 1), ("mig", G4, 1))],
             descents=10, placed=True, reach=[(0, 7, 9)], resume=[(0, 7, s) for s in range(8)]),
        dict(name="resume_lane_15", gpus=node([0xFFFF] * 15 + [0x0100]), pods=[claims(("mig", G1, 1), ("mig", G4, 1))],
             descents=10, placed=True, reach=[(0, 15, 9)], resume=[(0, 15, s) for s in range(8)]),
    ]


def colocation_fixtures():
    """Case 5 without selectors (the selector cases need a selector table; tests/test_gpu_pod_search.py builds them)."""
    return [
        # group 9 at positions 15 and 17, an ungrouped 1g between them: 15 x 1g fill GPU 0 to slice 14, the 2g at 15
        # goes to GPU 1, the 1g at 16 to GPU 0 slice 15, and the 2g at 17 follows its group to GPU 1
        dict(name="group_straddles_16", gpus=node([0, 0, 0]),
             pods=[claims(*[("mig", G1)] * 15 + [("mig", G2, 9), ("mig", G1), ("mig", G2, 9)])], descents=18, placed=True,
             reach=[(15, 1, 0), (16, 0, 15), (17, 1, 2)]),
        # first member at position 16 (on GPU 1 at start 8), the second at 20 must follow it there
        dict(name="group_first_at_16", gpus=node([0x0000, 0x00FF, 0x0000]),
             pods=[claims(*[("mig", G1)] * 16 + [("mig", G1, 4), ("mig", G1), ("mig", G1), ("mig", G1), ("mig", G2, 4)])],
             descents=21, placed=True, reach=[(16, 1, 8), (20, 1, 12)]),
        # two interleaved groups, A = 1 at positions 0, 2 and B = 2 at 1, 3 (slice 8 of GPU 0 busy): A's 4g fits only
        # at start 0, so A's 1g backtracks out of slices 0-7 (every choice of B's 1g is retried under each), to 9
        dict(name="groups_interleaved", gpus=node([0x0100, 0x0000, 0x0000]),
             pods=[claims(("mig", G1, 1), ("mig", G1, 2), ("mig", G4, 1), ("mig", G3, 2))], descents=398, placed=True,
             reach=[(0, 0, 9), (1, 0, 15), (2, 0, 0), (3, 0, 10)]),
        # the 4g never fits GPU 0 (slices 0 and 8 busy): its group's 1g tries all 14 free slices there, then moves
        dict(name="group_moves_member", gpus=node([0x0101, 0x0000]), pods=[claims(("mig", G1, 6), ("mig", G4, 6))],
             descents=16, placed=True, reach=[(0, 1, 0), (1, 1, 8)]),
    ]


def counted_fixtures():
    return budget_fixtures() + deep_fixtures() + resume_fixtures() + colocation_fixtures()


# ---- checks ----------------------------------------------------------------------------------------------------------
def _one_node(gpus):
    g = gpus.copy()
    g["node"] = 0
    return g, np.array([0, len(g)], np.uint32)


def _tbl(t):
    return [[(int(t[m, p]["size"]), int(t[m, p]["start_mask"])) for p in range(16)] for m in range(16)]


def _dicts(a):
    return [{k: int(x[k]) for k in a.dtype.names} for x in a]


@pytest.mark.parametrize("fx", counted_fixtures(), ids=lambda f: f["name"])
def test_fixture_reaches_what_it_is_named_for(fx):
    t = fixture_table()
    pod = fx["pods"][0]
    if fx["name"] == "deep_33":
        assert len(pod) == 33
        return
    if fx["name"] == "deep_31_then_fail":
        placed, n, log = search(fx["gpus"], t, pod, trace=False, cap=R.EXH_BUDGET + 1)
        assert placed is None and n > R.EXH_BUDGET                # the budget runs out long before the tree does
        placed, n, log = search(fx["gpus"], t, pod[:31])
        assert placed and n == 31 and (30, 1, 14) in log
        return
    placed, n, log = search(fx["gpus"], t, pod, cap=R.EXH_BUDGET + 8)
    if fx["descents"] is not None:
        assert n == fx["descents"], f"{fx['name']}: {n} descents"
    assert placed == fx["placed"]
    final = {}
    for p, g, s in log:
        final[p] = (g, s)
    for p, g, s in fx.get("reach", []):
        assert final.get(p) == (g, s), f"{fx['name']}: position {p} ends at {final.get(p)}"
    for r in fx.get("resume", []):
        assert r in resumed(log), f"{fx['name']}: no resume from {r}"


@pytest.mark.parametrize("fx", budget_fixtures(), ids=lambda f: f["name"])
def test_budget_fixture_counts_without_trace(fx):
    """The memoised count equals the traced one (the fixtures were found with it)."""
    placed, n, _ = search(fx["gpus"], fixture_table(), fx["pods"][0], trace=False)
    assert (placed, n) == (fx["placed"], fx["descents"])


@pytest.mark.parametrize("fx", counted_fixtures(), ids=lambda f: f["name"])
def test_fixture_status_in_oracle_and_naive(oracle, fx):
    """The C oracle and the Python restatement give the counted status, with and without the backtracking search."""
    from oracle import naive
    t = fixture_table()
    g, off = _one_node(fx["gpus"])
    pods = fx["pods"]
    c = np.concatenate(pods)
    pod_off = np.zeros(len(pods) + 1, np.uint32)
    pod_off[1:] = np.cumsum([len(p) for p in pods])
    for exhaustive in (False, True):
        out, after = oracle.allocate_pods(g, off, t, c, pod_off, flags=oracle.F_EXHAUSTIVE if exhaustive else 0)
        nout, nafter = naive.allocate_pods(_dicts(g), [int(x) for x in off], _tbl(t), _dicts(c), [int(x) for x in pod_off],
                                           exhaustive)
        assert [tuple(int(v) for v in r) for r in out] == nout
        assert [int(x) for x in after["busy"]] == [x["busy"] for x in nafter]
        st = set(int(s) for s in out["status"][: len(pods[0])])
        if fx["name"] == "deep_33":
            assert st == {R.ST_INVALID}
            continue
        if fx["name"] == "deep_31_then_fail":
            assert st == ({R.ST_SEARCH_LIMIT} if exhaustive else {R.ST_POD})
            assert after.tobytes() != g.tobytes()
            later = out[len(pods[0]):]
            assert list(later["status"]) == [0, 0] and list(later["gpu"]) == [0, 1] and list(later["start"]) == [0, 0]
            continue
        placed, n, _ = search(fx["gpus"], t, pods[0], trace=False, cap=R.EXH_BUDGET + 8)
        want = expected_status(placed, n) if exhaustive else None
        if exhaustive:
            assert st == {want}, f"{fx['name']}: {st} != {want}"
        elif fx["name"].startswith("fail_"):
            assert st == {R.ST_POD}
