"""CPU suite: Deallocate on one inventory (spec §9) against a plain restatement.  `released` below writes §9 as a loop over
claims and slots in Python integers: the §9 mask (`((1 << size) - 1) << start` cut to 16 bits, empty when start >= 16),
explicit u16 / u32 wrap, and the call failing with nothing changed when a claim's slot range leaves [0, n_out).  It does
not use the C oracle.  The records fed to it are arbitrary, not only ones Allocate wrote: preemption's running pods, the
C++ layer's held records and a Go caller's stored records all reach Deallocate from outside the call."""
import ctypes as C

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from oracle import oracle as O
from test_oracle_properties import problems

GPU, MIG, SHARED = 0, 1, 2
FULL_ALLOCATED = 0x02
OK = 0
NONE = 0xFFFFFFFF
EDGES = [15, 16, 31, 32, 255]                         # where a shift count or a 16-bit cut goes wrong


def slots(kind, count, node, n_node, have_off):
    """slots(c) of spec §1 / §3, as Allocate counted them: an INVALID claim has one."""
    return count if kind == GPU and node < n_node and 1 <= count <= 32 and (have_off or count == 1) else 1


def released(gpus, n_node, claims, out, out_off=None):
    """Spec §9 restated: the inventory after the call, or None when the call fails (and so changes nothing)."""
    n_gpu, n_out, have_off = len(gpus), len(out), out_off is not None
    ranges = []
    for i, c in enumerate(claims):
        base = int(out_off[i]) if have_off else i
        n = slots(int(c["kind"]), int(c["count"]), int(c["node"]), n_node, have_off)
        if base + n > n_out:
            return None
        ranges.append((base, n))
    busy = [int(x) for x in gpus["busy"]]
    flags = [int(x) for x in gpus["flags"]]
    mem = [int(x) for x in gpus["mem_free_mib"]]
    share = [int(x) for x in gpus["share_cnt"]]
    for c, (base, n) in zip(claims, ranges):
        kind = int(c["kind"])
        for k in range(base, base + n):
            o = out[k]
            g = int(o["gpu"])
            if int(o["status"]) != OK or g >= n_gpu:
                continue
            if kind == GPU:
                flags[g] &= ~FULL_ALLOCATED & 0xFF
            elif kind == MIG:
                start, size = int(o["start"]), int(o["size"])
                busy[g] &= ~((((1 << size) - 1) << start) & 0xFFFF) & 0xFFFF
            elif kind == SHARED:
                mem[g] = (mem[g] + int(c["mem_limit_mib"])) % (1 << 32)
                share[g] = (share[g] - 1) % (1 << 16)
    after = gpus.copy()
    after["busy"], after["flags"], after["mem_free_mib"], after["share_cnt"] = busy, flags, mem, share
    return after


def _edge_u8(draw):
    return draw(st.one_of(st.sampled_from(EDGES), st.integers(0, 255)))


@st.composite
def releases(draw):
    """An inventory of test_oracle_properties.problems, its GPUs' words pushed to their edges, and arbitrary claims and
    records with every slot range inside [0, n_out): kinds 0-4, GPU claims of count 0, 1, 32 and 33 naming a node or
    none, records of any status, start and size, GPUs at n_gpu - 1, n_gpu and NONE, out_off ranges that overlap, the
    same claim given twice, and SHARED releases that wrap share_cnt below 0 and mem_free_mib past 2^32."""
    g, off, _, _, _, _ = draw(problems())
    n_node, n_gpu = len(off) - 1, len(g)
    for i in range(n_gpu):
        if draw(st.booleans()):
            g["busy"][i] = draw(st.sampled_from([0xFFFF, 0x8000, 0x00FF, draw(st.integers(0, 0xFFFF))]))
            g["flags"][i] = draw(st.integers(0, 255))
            g["mem_free_mib"][i] = draw(st.sampled_from([0, 1, 0xFFFFFFFF, 0xFFFFF000]))
            g["share_cnt"][i] = draw(st.sampled_from([0, 1, 0xFFFF]))
    have_off = draw(st.booleans())
    n_claim = draw(st.integers(0, 20))
    c = np.zeros(n_claim, dtype=O.CLAIM_DTYPE)
    for i in range(n_claim):
        kind = draw(st.sampled_from([GPU, GPU, MIG, MIG, MIG, SHARED, SHARED, SHARED, 3, 4]))
        c[i] = (kind, draw(st.integers(0, 255)),
                draw(st.sampled_from([0, 1, 1, 1, 2, 32, 33])) if kind == GPU else draw(st.sampled_from([1, 0, 5])),
                draw(st.sampled_from([0, n_node - 1, n_node, NONE])),
                draw(st.sampled_from([0, 1, 1000, 0x80000000, 0xFFFFFFFF])) if kind == SHARED else draw(st.integers(0, 7)),
                draw(st.integers(0, 3)))
    sl = [slots(int(x["kind"]), int(x["count"]), int(x["node"]), n_node, have_off) for x in c]
    if have_off:
        n_out = max(sl + [0]) + draw(st.integers(0, 40))
        out_off = np.array([draw(st.integers(0, n_out - s)) for s in sl], dtype=np.uint32)   # ranges overlap freely
        if n_claim and draw(st.booleans()):                                                 # one claim given twice
            j = draw(st.integers(0, n_claim - 1))
            c = np.concatenate([c, c[j:j + 1]])
            out_off = np.concatenate([out_off, out_off[j:j + 1]])
    else:
        out_off = None
        if n_claim and draw(st.booleans()):                                                 # the same record twice
            c = np.concatenate([c, c[-1:]])
        n_out = len(c) + draw(st.integers(0, 3))
    out = np.zeros(n_out, dtype=O.OUT_DTYPE)
    for k in range(n_out):
        gpu = draw(st.sampled_from([max(n_gpu - 1, 0), n_gpu, NONE, draw(st.integers(0, max(n_gpu - 1, 0)))]))
        status = draw(st.sampled_from([OK, OK, OK, draw(st.integers(0, 255))]))
        out[k] = (gpu, _edge_u8(draw), _edge_u8(draw), draw(st.integers(0, 255)), status)
    if not have_off and len(c) > 1 and draw(st.booleans()):
        out[len(c) - 1] = out[len(c) - 2]
    return g, off, c, out, out_off


@settings(max_examples=400, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True)
@given(releases())
def test_oracle_deallocate_is_the_restatement(oracle, prob):
    g, off, c, out, out_off = prob
    n_node = len(off) - 1
    want = released(g, n_node, c, out, out_off)
    assert want is not None
    got = oracle.deallocate(g, c, out, out_off, n_node=n_node)
    assert got.tobytes() == want.tobytes()


def _one_mig_gpu_per_pair(pairs, busy=0xFFFF):
    g = np.zeros(len(pairs), dtype=O.GPU_DTYPE)
    g["busy"], g["flags"], g["node"] = busy, 1, 0
    c = np.zeros(len(pairs), dtype=O.CLAIM_DTYPE)
    c["kind"], c["count"], c["node"] = MIG, 1, 0
    out = np.zeros(len(pairs), dtype=O.OUT_DTYPE)
    out["gpu"] = np.arange(len(pairs))
    out["start"], out["size"] = [p[0] for p in pairs], [p[1] for p in pairs]
    out["profile"], out["status"] = 1, OK
    return g, c, out


def test_every_start_and_size_of_a_record(oracle):
    """Every (start, size) pair of two u8 fields, one MIG GPU with every slice busy per pair, in one call."""
    pairs = [(s, z) for s in range(256) for z in range(256)]
    g, c, out = _one_mig_gpu_per_pair(pairs)
    got = oracle.deallocate(g, c, out, None, n_node=1)
    want = released(g, 1, c, out)
    assert got.tobytes() == want.tobytes()
    m = {p: int(b) for p, b in zip(pairs, want["busy"])}
    assert m[(0, 16)] == m[(0, 32)] == m[(0, 255)] == 0 and m[(15, 1)] == 0x7FFF and m[(14, 255)] == 0x3FFF
    assert m[(16, 1)] == m[(31, 255)] == m[(32, 1)] == m[(255, 255)] == 0xFFFF and m[(0, 0)] == 0xFFFF


# The records §9 did not define before it took §14's mask: start or size of 32 and more.  (200, 4) and (40, 2) name no
# slice of a 16-slice GPU; (0, 32) names all of them.  A C shift by the raw u8 is undefined at these counts.
@pytest.mark.parametrize("start,size,busy_after", [(200, 4, 0xFFFF), (0, 32, 0x0000), (40, 2, 0xFFFF)],
                         ids=["start200_size4", "start0_size32", "start40_size2"])
def test_records_past_16_slices(oracle, start, size, busy_after):
    g, c, out = _one_mig_gpu_per_pair([(start, size)])
    assert int(released(g, 1, c, out)["busy"][0]) == busy_after
    assert int(oracle.deallocate(g, c, out, None, n_node=1)["busy"][0]) == busy_after


BAD_RANGES = ["first", "middle", "last", "beyond", "short"]


def bad_range(where):
    """Ten claims that each release something, and a slot range past n_out.  With out_off: the first, middle or last
    claim is a count-3 GPU claim whose range starts two slots before the end, or ("beyond") the middle one starts at
    0xFFFFFFFF.  Without it ("short"): n_out = n_claim - 1, so the last claim has no slot.  Returns the inventory, the
    call's arrays and `keep`, the claims a call that succeeds would keep."""
    g = np.zeros(10, dtype=O.GPU_DTYPE)
    g["busy"], g["flags"], g["mem_free_mib"], g["share_cnt"] = 0xFFFF, 1 | FULL_ALLOCATED, 100, 5
    c = np.zeros(10, dtype=O.CLAIM_DTYPE)
    c["kind"] = [MIG, GPU, SHARED, MIG, GPU, SHARED, MIG, GPU, SHARED, MIG]
    c["count"], c["node"], c["mem_limit_mib"], c["profile"] = 1, 0, 7, 1
    keep = np.ones(10, dtype=bool)
    if where == "short":
        out_off, n_out = None, 9
        keep[9] = False
    else:
        bad = {"first": 0, "middle": 5, "last": 9, "beyond": 5}[where]
        out_off, n_out = np.arange(10, dtype=np.uint32), 12
        if where == "beyond":
            out_off[bad] = NONE
        else:
            c["kind"][bad], c["count"][bad] = GPU, 3
            out_off[bad] = n_out - 2
        keep[bad] = False
    out = np.zeros(n_out, dtype=O.OUT_DTYPE)
    out["gpu"], out["start"], out["size"], out["status"] = np.arange(n_out) % 10, 0, 4, OK
    return g, c, out, out_off, keep


@pytest.mark.parametrize("where", BAD_RANGES)
def test_bad_slot_range_changes_nothing(oracle, where):
    """dra_oracle_deallocate on the caller's own buffer (the Python wrapper works on a copy): -1, and not one byte of the
    inventory written, although the other claims' records release something."""
    g, c, out, out_off, keep = bad_range(where)
    assert released(g, 1, c, out, out_off) is None
    good = released(g, 1, c[keep], out, None if out_off is None else out_off[keep])
    assert good is not None and good.tobytes() != g.tobytes()
    buf = g.copy()
    oo = None if out_off is None else out_off.ctypes.data_as(C.c_void_p)
    rc = oracle.lib().dra_oracle_deallocate(buf.ctypes.data_as(C.c_void_p), len(buf), 1, c.ctypes.data_as(C.c_void_p),
                                            len(c), oo, out.ctypes.data_as(C.c_void_p), len(out))
    assert rc == -1
    assert buf.tobytes() == g.tobytes(), "a failed Deallocate wrote the inventory"
    with pytest.raises(ValueError):
        oracle.deallocate(g, c, out, out_off, n_node=1)
