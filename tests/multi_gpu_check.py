#!/usr/bin/env python
"""Multi-GPU parity check (run under torchrun on N >= 2 GPUs of one box; not collected by pytest — the round-end
GPU suite runs on one GPU).  Every rank allocates its shard and all-gathers; every rank then compares the WHOLE
gathered table, merged back to global input order, with the CPU oracle on the global batch.  Paths covered:
fused kernel + packet-gather tail, sort path + gather kernel, ncclAllGather, and the sharded GLOBAL batch; claims with counts > 1
(out_off), co-location groups, malformed claims.

  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tests/multi_gpu_check.py
"""
import numpy as np
import torch
import torch.distributed as dist

from multi_gpu_rank import finish, pkg, report, start
from oracle import oracle as O
R = pkg.records

rank, world, dev, stream = start()
for name, w, ctx_flags, use_peer in [
        ("fused+peer, mixed with counts/groups/invalid", pkg.synth.mixed(9000, 97, 21), 0, True),
        ("sort path+peer push/wait", pkg.synth.mixed(9000, 97, 22), pkg.api.CFG_NO_FUSED, True),
        ("fused+nccl", pkg.synth.mixed(9000, 97, 23), 0, False),
        ("fused+peer, cfg2-like", pkg.synth.cfg2(20000, 250), 0, True)]:
    ranges = pkg.shard.plan(w.claims["node"], w.n_node, world)
    lbs = [pkg.shard.local_batch(w.gpus, w.node_off, w.claims, r, ranges) for r in range(world)]
    lb = lbs[rank]
    n_per = max(b.n_out for b in lbs); n_per += n_per & 1
    ctx = pkg.api.Context(device=dev.index, stream=stream.cuda_stream, flags=ctx_flags)
    ctx.set_table(w.table); ctx.set_inventory(lb.gpus, lb.node_off)
    uid = [pkg.api.Context.comm_unique_id() if rank == 0 else None]      # one NCCL unique id per communicator
    dist.broadcast_object_list(uid, src=0)
    ctx.comm_init(uid[0], rank, world)
    if use_peer:
        hs = [None] * world
        dist.all_gather_object(hs, ctx.peer_export(n_per))
        ctx.peer_import(hs)
    d_claims = torch.from_numpy(lb.claims.view(np.uint8).copy()).to(dev)
    d_off = torch.from_numpy(lb.out_off.view(np.uint8).copy()).to(dev)
    d_all = torch.zeros(world * n_per * 8, dtype=torch.uint8, device=dev)
    for rep in range(3):      # repeated calls exercise the parity double-buffering
        ctx.allocate_gather_device(d_claims.data_ptr(), len(lb.claims), d_off.data_ptr(), None if use_peer else d_all.data_ptr(),
                                   lb.n_out, n_per, pkg.api.F_FRESH_INVENTORY)
        table = ctx.gather_read(np.zeros(world * n_per, dtype=R.OUT_DTYPE))
        parts = [(b.sel, b.out_off, table[r * n_per: r * n_per + b.n_out], b.gpu_base) for r, b in enumerate(lbs)]
        merged = pkg.shard.merge(w.n_out, w.out_off if w.out_off is not None else np.arange(w.n_claim, dtype=np.uint32), parts)
        ref, _ = O.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
        report(f"{name} rep {rep}", merged.tobytes() == ref.tobytes(), f"{w.n_claim} claims, {world} ranks")
    ctx.close()
# ---- the sharded GLOBAL batch: the same claim array on every rank, device-side range filter, global slots ----
for name, w, ctx_flags in [("global batch, fused, mixed", pkg.synth.mixed(9000, 97, 31), 0),
                           ("global batch, sort path", pkg.synth.mixed(30000, 200, 32), pkg.api.CFG_NO_FUSED),
                           ("global batch, cfg3/4", pkg.synth.cfg2(25000, 250), 0),
                           # large: every shard goes through wave-sized hist tiles, the row-wise scan and the stand-alone gather
                           ("global batch, 1M claims x 10k nodes", pkg.synth.cfg2(1_000_000, 10_000), 0)]:
    ranges = pkg.shard.plan(w.claims["node"], w.n_node, world)
    ctx = pkg.api.Context(device=dev.index, stream=stream.cuda_stream, flags=ctx_flags)
    ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
    uid = [pkg.api.Context.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    ctx.comm_init(uid[0], rank, world)
    ctx.set_shard_map([r[0] for r in ranges] + [ranges[-1][1]], stray_rank=0)
    hs = [None] * world
    dist.all_gather_object(hs, ctx.shard_export(w.n_out))
    ctx.peer_import(hs)
    d_claims = torch.from_numpy(w.claims.view(np.uint8).copy()).to(dev)
    d_off = None if w.out_off is None else torch.from_numpy(w.out_off.view(np.uint8).copy()).to(dev)
    ref, ref_inv = O.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
    for rep in range(3):
        ctx.peer_rendezvous()                       # device-side rendezvous of the ranks (what bench.py enqueues after its flush)
        ctx.allocate_global_device(d_claims.data_ptr(), w.n_claim, None if d_off is None else d_off.data_ptr(), w.n_out, pkg.api.F_FRESH_INVENTORY)
        table = ctx.gather_read(np.zeros(w.n_out, dtype=R.OUT_DTYPE))
        g0, g1 = int(w.node_off[ranges[rank][0]]), int(w.node_off[ranges[rank][1]])
        report(f"{name} rep {rep}", table.tobytes() == ref.tobytes()
               and ctx.get_inventory()[g0:g1].tobytes() == ref_inv[g0:g1].tobytes(), f"{w.n_claim} claims, {world} ranks")
    dist.barrier()
    ctx.close()
finish()
