#!/usr/bin/env python
"""Multi-GPU parity check of the sharded pods Allocate (run under torchrun on the GPUs of one box; not collected by
pytest).  One process per GPU, gather buffers mapped with IPC handles (dra_shard_export / dra_peer_import).  The classic
flow on a sharded world: a sharded Allocate without DRA_F_FRESH_INVENTORY makes the ranks' inventories diverge, a sharded
exhaustive UnsuitableNodes finds a suitable node for each pod, and the sharded pods Allocate places the pods retargeted to
those nodes.  Every rank's verdict, whole table and own inventory range must equal the CPU oracle's on the real state.
Then the same pods call with first-fit, exhaustive and fresh-inventory flags on the fragmented pod workload.

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/multi_gpu_shard_pods_check.py
"""
import numpy as np
import torch
import torch.distributed as dist

import multi_gpu_rank as M
from multi_gpu_rank import dv, finish, join, pkg, report, start
from oracle import oracle as O
R = pkg.records
F_EXH, F_FRESH = pkg.api.F_EXHAUSTIVE, pkg.api.F_FRESH_INVENTORY

rank, world, dev, stream = start()
w, pod_off = pkg.synth.pods(2000, 24 * world, 11)
bounds = [w.n_node * r // world for r in range(world)] + [w.n_node]
g0, g1 = int(w.node_off[bounds[rank]]), int(w.node_off[bounds[rank + 1]])
first = int(pod_off[300])                           # the first 300 pods' claims: the sharded claim Allocate
n_pod = 1700
claims = w.claims[first:].copy()
po = (pod_off[300:] - first).astype(np.uint32)
ctx = pkg.api.Context(device=dev.index, stream=stream.cuda_stream)
ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
join(ctx, bounds, world - 1, max(w.n_claim, 1), pairs=(n_pod * w.n_node,))


def real_state():
    """Every rank's inventory over its own GPU range, assembled on every rank."""
    mine = ctx.get_inventory()
    parts = [None] * world
    dist.all_gather_object(parts, mine[g0:g1].tobytes())
    real = w.gpus.copy()
    for r in range(world):
        a, b = int(w.node_off[bounds[r]]), int(w.node_off[bounds[r + 1]])
        real[a:b] = np.frombuffer(parts[r], dtype=w.gpus.dtype)
    return real


def check(what, c, p_off, flags):
    src = w.gpus if flags & F_FRESH else real_state()
    ref, ref_inv = O.allocate_pods(src, w.node_off, w.table, c, p_off, None, len(c), O.F_EXHAUSTIVE if flags & F_EXH else 0)
    d_c, d_p = dv(c), dv(p_off)
    torch.cuda.synchronize()
    ctx.allocate_pods_global_device(d_c.data_ptr(), len(c), d_p.data_ptr(), len(p_off) - 1, None, len(c), flags)
    ctx.sync()
    got = ctx.gather_read(np.zeros(len(c), dtype=R.OUT_DTYPE))
    inv = ctx.get_inventory()
    ok = got.tobytes() == ref.tobytes() and inv[g0:g1].tobytes() == ref_inv[g0:g1].tobytes()
    st = ref["status"]
    report(f"sharded pods Allocate, {what}", ok, f"{len(p_off) - 1} pods, {int((st == 0).sum())} OK slots of {len(st)}, {world} ranks")
    return ref


# 1. sharded claim Allocate: the ranks' copies diverge outside their ranges
d_first = dv(w.claims[:first])
ctx.allocate_global_device(d_first.data_ptr(), first, None, first, 0)
ctx.gather_read(np.zeros(first, dtype=R.OUT_DTYPE))
# 2. sharded exhaustive UnsuitableNodes on the real state
n_pair = n_pod * w.n_node
d_c, d_p = dv(claims), dv(po)
bits = torch.zeros((n_pair + 7) // 8, dtype=torch.uint8, device=dev)
ctx.unsuitable_global_device(d_c.data_ptr(), len(claims), d_p.data_ptr(), n_pod, None, None, n_pair, bits.data_ptr(), F_EXH)
ctx.sync()
real = real_state()
dn = np.tile(np.arange(w.n_node, dtype=np.uint32), n_pod)
do = (np.arange(n_pod + 1, dtype=np.uint64) * w.n_node).astype(np.uint32)
ref_bits = O.unsuitable(real, w.node_off, w.table, claims, po, dn, do, flags=O.F_EXHAUSTIVE)
h = bits.cpu().numpy()
report("sharded exhaustive UnsuitableNodes", h.tobytes() == ref_bits.tobytes(), f"{n_pair} pairs")
# 3. one suitable node per pod (at most one pod per node), claims retargeted there: every pod must be placed
verdict = np.unpackbits(h, bitorder="little")[:n_pair].reshape(n_pod, w.n_node)
taken, keep = set(), []
for p in range(n_pod):
    free = [n for n in np.flatnonzero(verdict[p]) if n not in taken]
    if free:
        n = int(free[0]); taken.add(n); keep.append((p, n))
sub = np.concatenate([claims[po[p]: po[p + 1]] for p, _ in keep]).copy()
sub_off = np.zeros(len(keep) + 1, dtype=np.uint32)
sub_off[1:] = np.cumsum([po[p + 1] - po[p] for p, _ in keep])
for k, (_, n) in enumerate(keep):
    sub["node"][sub_off[k]: sub_off[k + 1]] = n
ref = check("pods on their suitable nodes, exhaustive", sub, sub_off, F_EXH)
if not (ref["status"] == 0).all():                  # the same oracle answer on every rank: each counts it
    M.fails += 1
    if rank == 0:
        print("MISMATCH: a pod the exhaustive verdict called suitable was not placed")
# 4. the fragmented workload itself, every flag; repeated calls use both table parities
for flags, name in ((0, "first-fit"), (F_EXH, "exhaustive"), (F_FRESH, "fresh first-fit"), (F_EXH | F_FRESH, "fresh exhaustive")):
    check(name, claims, po, flags)
finish([ctx])
