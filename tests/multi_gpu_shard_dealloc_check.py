#!/usr/bin/env python
"""Multi-GPU parity check of the sharded Deallocate (run under torchrun on N >= 2 GPUs of one box; not collected by pytest).
One process per GPU, peer buffers mapped with IPC handles (dra_shard_export / dra_peer_import).  A sharded Allocate with
SHARED claims, then dra_deallocate_batch_global_device of a subset straight from the gathered table: every rank's own range
must equal the CPU oracle's state on ONE inventory, every other GPU must be as that rank held it before, and after
dra_shard_sync_inventory_device every rank's whole inventory must equal the oracle's.  Then the rest of the records are
released the same way, which must give back the loaded inventory.

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/multi_gpu_shard_dealloc_check.py
"""
import ctypes as C

import numpy as np
import torch
import torch.distributed as dist

from multi_gpu_rank import dv, finish, join, pkg, report, start
from oracle import oracle as O
R = pkg.records

rank, world, dev, stream = start()
w = pkg.synth.mixed(4000, 200 * world + 5, 31, invalid=True)
rng = np.random.default_rng(31)
claims = w.claims.copy()
sh = rng.random(len(claims)) < 0.2                                  # a fifth SHARED, as cfg4
claims["kind"][sh], claims["count"][sh], claims["group"][sh] = R.KIND_SHARED, 1, 0
claims["mem_limit_mib"][sh] = rng.choice(np.array([1024, 4096, 10240], dtype=np.uint32), int(sh.sum()))
out_off, n_out = R.out_offsets(claims, w.n_node)
n_out = int(n_out)
ctx = pkg.api.Context(device=dev.index, stream=stream.cuda_stream)
ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
bounds = [0] + [min(w.n_node, 1 + 3 * r * r) for r in range(1, world)] + [w.n_node]     # uneven ranges
join(ctx, bounds, world - 1, n_out)
g0, g1 = int(w.node_off[bounds[rank]]), int(w.node_off[bounds[rank + 1]])
detail = f"{world} ranks, {w.n_gpu} GPUs"


def table_ptr():
    p, n = C.c_void_p(), C.c_uint32()
    assert ctx._lib.dra_gather_table(ctx._h, C.byref(p), C.byref(n)) == 0
    return p.value


def release(sub, sub_off, state, what):
    d_c, d_o = dv(sub), dv(sub_off)
    torch.cuda.synchronize()
    before = ctx.get_inventory()
    ctx.deallocate_global_device(d_c.data_ptr(), len(sub), d_o.data_ptr(), table_ptr(), n_out)
    ctx.sync()
    inv = ctx.get_inventory()
    report(what, inv[g0:g1].tobytes() == state[g0:g1].tobytes() and inv[:g0].tobytes() == before[:g0].tobytes()
           and inv[g1:].tobytes() == before[g1:].tobytes(), detail)
    dist.barrier()
    ctx.shard_sync_inventory_device()
    ctx.sync()
    report(f"{what}, then the sync", ctx.get_inventory().tobytes() == state.tobytes(), detail)


d_c, d_o = dv(claims), dv(out_off)
torch.cuda.synchronize()
ref, state = O.allocate(w.gpus, w.node_off, w.table, claims, out_off, n_out)
ctx.allocate_global_device(d_c.data_ptr(), len(claims), d_o.data_ptr(), n_out, 0)
ctx.sync()
report("sharded Allocate", ctx.gather_read(np.zeros(n_out, dtype=R.OUT_DTYPE)).tobytes() == ref.tobytes(), detail)
sel = rng.random(len(claims)) < 0.4
state = O.deallocate(state, claims[sel], ref, out_off[sel], n_node=w.n_node)
release(claims[sel], out_off[sel].copy(), state, "sharded Deallocate of 40% of the claims")
state = O.deallocate(state, claims[~sel], ref, out_off[~sel], n_node=w.n_node)
release(claims[~sel], out_off[~sel].copy(), state, "sharded Deallocate of the rest")
report("every record released gives back the loaded inventory", state.tobytes() == w.gpus.tobytes(), detail)
finish([ctx])
