"""CPU suite, part 2: the C-ABI library builds, loads, and exports every symbol include/dra_alloc.h
declares; record layouts match; with no GPU the library refuses to create a context (no CPU fallback)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dra_alloc.h")


def _declared():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(dra_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol(pkg):
    lib = pkg.api.load()
    names = _declared()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/dra_alloc.h but not exported"
    assert set(names) == set(pkg.api.SYMBOLS), "python binding and header drifted apart"
    assert lib.dra_abi_version() == 2


def test_record_sizes_match_header(pkg, tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include "dra_alloc.h"\n#include <stdio.h>\n#include <stddef.h>\n'
                   'int main(){printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(dra_gpu_rec), sizeof(dra_claim_rec),'
                   'sizeof(dra_out_rec), sizeof(dra_prof_ent), sizeof(dra_profile_tbl),'
                   'offsetof(dra_gpu_rec, share_cnt), offsetof(dra_claim_rec, group));return 0;}')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    R = pkg.records
    assert [int(x) for x in got] == [R.GPU_DTYPE.itemsize, R.CLAIM_DTYPE.itemsize, R.OUT_DTYPE.itemsize,
                                     R.PROF_DTYPE.itemsize, 64, R.GPU_DTYPE.fields["share_cnt"][1],
                                     R.CLAIM_DTYPE.fields["group"][1]]


def test_no_gpu_means_no_context(pkg):
    """Without a CUDA device dra_ctx_create must fail loudly — the product has no CPU path."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present; covered by the gpu suite")
    with pytest.raises(pkg.api.DraError) as e:
        pkg.api.Context(device=0)
    assert e.value.code == pkg.api.E_CUDA
    assert "no CPU fallback" in str(e.value)


def test_product_does_not_touch_the_oracle():
    """oracle/ is a checker: nothing under the product package may import, link or mention it."""
    pk = os.path.join(ROOT, "k8s-dra-driver_b200")
    for dp, _, fs in os.walk(pk):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".hpp", ".h")):
                text = open(os.path.join(dp, f), errors="ignore").read()
                assert "dra_oracle" not in text and "from oracle" not in text and "import oracle" not in text, f
    so = os.path.join(pk, "libdra_alloc.so")
    if os.path.exists(so):
        out = subprocess.run(["nm", "-D", so], capture_output=True, text=True).stdout
        assert "dra_oracle" not in out


def test_kernels_are_sm90a_and_use_tma(pkg):
    """cuobjdump evidence: the cubin is sm_90a; TMA bulk copies (UBLKCP), mbarriers (SYNCS), ballots (VOTE) in SASS."""
    so = pkg.api.SO_PATH
    r = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    assert "sm_90a" in r.stdout
    for mnem in ("UBLKCP", "VOTE", "SYNCS", "LDG.E.128", "STG.E.64"):
        assert mnem in r.stdout, mnem


def test_flag_constants_match_header(pkg):
    """DRA_CFG_* / DRA_F_* / DRA_K_* / error codes of the ctypes binding are the header's."""
    text = open(HEADER).read()
    defs = {m.group(1): int(m.group(2), 0) for m in re.finditer(r"#define\s+(DRA_(?:CFG|F)_[A-Z_]+)\s+(0x[0-9a-fA-F]+)u", text)}
    A = pkg.api
    assert defs == {"DRA_CFG_USE_GRAPH": A.CFG_USE_GRAPH, "DRA_CFG_NO_FUSED": A.CFG_NO_FUSED,
                    "DRA_CFG_NO_DIRECT": A.CFG_NO_DIRECT, "DRA_CFG_RESIDENT": A.CFG_RESIDENT, "DRA_F_NODE_SORTED": A.F_NODE_SORTED,
                    "DRA_F_FRESH_INVENTORY": A.F_FRESH_INVENTORY, "DRA_F_EXHAUSTIVE": A.F_EXHAUSTIVE}
    kern = {m.group(1): int(m.group(2), 0) for m in re.finditer(r"#define\s+DRA_K_([A-Z0-9_]+)\s+(0x[0-9a-fA-F]+)u", text)}
    assert kern == {k.upper(): v for k, v in A.KERNELS.items()}
    assert len(set(kern.values())) == len(kern) and all(v & (v - 1) == 0 for v in kern.values())   # one bit each
    errs = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+(DRA_E_[A-Z]+)\s+\((-\d+)\)", text)}
    assert errs == {"DRA_E_INVAL": A.E_INVAL, "DRA_E_CUDA": A.E_CUDA, "DRA_E_NCCL": A.E_NCCL, "DRA_E_NOMEM": A.E_NOMEM,
                    "DRA_E_STATE": A.E_STATE}


def test_packer_context_stays_in_registers(pkg):
    """The packing kernels keep the node context (lane state, memo, sink) in registers: a reference into it handed
    to the out-of-line generic step once pinned the whole context in local memory (STACK 208, an LDL on every access
    of the hot loops).  What remains on the stack are the copies made for that call.  Also: the sort path's
    dependent-launch instructions and the warp reductions of the lean loops are in the SASS."""
    so = pkg.api.SO_PATH
    r = subprocess.run(["cuobjdump", "-res-usage", so], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    stacks = {}
    name = None
    for line in r.stdout.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
        m = re.search(r"STACK:(\d+)", line)
        if m and name:
            stacks[name] = int(m.group(1))
    hot = {k: v for k, v in stacks.items() if "k_fused" in k or "k_pack" in k or "k_serve" in k}
    assert len(hot) >= 4, stacks
    assert all(v <= 112 for v in hot.values()), hot        # lane state + memo + sink (incl. its send-queue words), copied for the cold call
    # pod mode (spec §12) hands a COPY of the lane state to its out-of-line evaluator: 24 bytes, off the hot paths
    pod = {k: v for k, v in stacks.items() if "k_pods" in k or "k_unsuitable" in k or "pod_eval" in k or "k_shard_compact" in k}
    assert all(v <= 64 for v in pod.values()), pod         # (the 2048-claim compaction tile is held to 64 registers: 48 bytes spill, off every hot loop)
    assert all(v == 0 for k, v in stacks.items() if k not in hot and k not in pod), stacks
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    for mnem in ("PREEXIT", "ACQBULK", "REDUX.OR", "REDUX.MIN"):
        assert mnem in sass, mnem


def test_synthetic_configs_shape(pkg):
    S = pkg.synth
    w = S.cfg2()
    assert (w.n_claim, w.n_gpu, w.n_node) == (10_000, 1000, 125)
    assert w.algorithmic_bytes() == 24 * 10_000 + 16 * 1000          # SURVEY §8(d): 256,000 B
    frac = np.bincount(w.claims["profile"], minlength=5) / w.n_claim
    assert abs(frac[0] - .4) < .02 and abs(frac[1] - .3) < .02 and abs(frac[2] - .2) < .02 and abs(frac[4] - .1) < .02
    w5 = S.cfg5()
    assert (w5.n_claim, w5.n_gpu) == (50_000, 512) and np.all(w5.gpus["busy"] != 0xFF)
    assert S.cfg2().claims.tobytes() == w.claims.tobytes()           # seeded: reproducible
