#!/usr/bin/env python
"""Multi-GPU parity check of the inventory sync (run under torchrun on N >= 2 GPUs of one box; not collected by pytest).  One
process per GPU, peer buffers mapped with IPC handles (dra_shard_export / dra_peer_import).  A sharded Allocate without
DRA_F_FRESH_INVENTORY and a per-rank Deallocate of half its records make the ranks' copies diverge; after
dra_shard_sync_inventory_device every rank's whole inventory must equal the CPU oracle's on ONE inventory after the same
calls.  Then the node ranges rotate (dra_set_shard_map), and a sharded Allocate plus a sync must again give the oracle's
table and state.

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/multi_gpu_shard_sync_check.py
"""
import numpy as np
import torch
import torch.distributed as dist

from multi_gpu_rank import dv, finish, join, pkg, report, start
from oracle import oracle as O
R = pkg.records

rank, world, dev, stream = start()
w = pkg.synth.mixed(4000, 200 * world + 5, 21, invalid=True)      # 2,900-5,900 GPUs: k_isync_copy runs 12-23 CTAs
ctx = pkg.api.Context(device=dev.index, stream=stream.cuda_stream)
ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
bounds = [0] + [min(w.n_node, 1 + 3 * r * r) for r in range(1, world)] + [w.n_node]     # uneven ranges
join(ctx, bounds, world - 1, w.n_out)
detail = f"{world} ranks, {w.n_gpu} GPUs"


def allocate(claims, out_off, n_out):
    d_c, d_o = dv(claims), dv(out_off)
    torch.cuda.synchronize()
    ctx.allocate_global_device(d_c.data_ptr(), len(claims), d_o.data_ptr(), n_out, 0)
    ctx.sync()
    return ctx.gather_read(np.zeros(n_out, dtype=R.OUT_DTYPE))


def sync_and_check(what, state):
    g0, g1 = int(w.node_off[bounds[rank]]), int(w.node_off[bounds[rank + 1]])
    before = ctx.get_inventory()
    dist.barrier()
    ctx.shard_sync_inventory_device()
    ctx.sync()
    inv = ctx.get_inventory()
    report(what, inv.tobytes() == state.tobytes() and inv[g0:g1].tobytes() == before[g0:g1].tobytes(), detail)


# 1. sharded Allocate, then every rank deallocates the first half of the claims' records
claims, out_off, n_out = w.claims, w.out_off, int(w.n_out)
ref, state = O.allocate(w.gpus, w.node_off, w.table, claims, out_off, n_out)
report("sharded Allocate", allocate(claims, out_off, n_out).tobytes() == ref.tobytes(), detail)
half = len(claims) // 2
ctx.deallocate(claims[:half], ref, out_off[:half])
state = O.deallocate(state, claims[:half], ref, out_off[:half], n_node=w.n_node)
sync_and_check("sync after Allocate + per-rank Deallocate", state)
# 2. rotate the ranges (and the stray rank), allocate again on the synced state, sync
bounds = [0] + [w.n_node - b for b in reversed(bounds[1:-1])] + [w.n_node]
ctx.set_shard_map(bounds, stray_rank=0)
c2 = w.claims.copy(); c2["node"] = (c2["node"] + 3) % w.n_node
o2, n2 = R.out_offsets(c2, w.n_node)
ref2, state = O.allocate(state, w.node_off, w.table, c2, o2, int(n2))
report("sharded Allocate after the re-map", allocate(c2, o2, int(n2)).tobytes() == ref2.tobytes(), detail)
sync_and_check("sync after the re-map", state)
finish([ctx])
