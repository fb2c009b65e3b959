#!/usr/bin/env python
"""Multi-GPU parity check of sharded UnsuitableNodes (run under torchrun on N >= 2 GPUs of one box; not collected by
pytest).  One process per GPU, gather buffers mapped with IPC handles (dra_shard_export / dra_peer_import).  A sharded
Allocate without DRA_F_FRESH_INVENTORY first makes the ranks' inventories diverge; then every rank's whole bitmap from
dra_unsuitable_batch_global_device must equal the CPU oracle's answer on the state that Allocate left — dense and
candidate-list forms, first-fit and exhaustive, claims of every kind with counts > 1 and malformed claims.

  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tests/multi_gpu_shard_unsuitable_check.py
"""
import importlib, os, sys
import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("k8s-dra-driver_b200")
from oracle import oracle as O
R = pkg.records

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
os.environ.setdefault("NCCL_DEBUG", "WARN")
torch.cuda.set_device(local)
dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
dev = torch.device("cuda", local)
stream = torch.cuda.Stream(device=dev); torch.cuda.set_stream(stream)
fails = 0

w = pkg.synth.mixed(9000, 97, 41)
ranges = pkg.shard.plan(w.claims["node"], w.n_node, world)
n_pod = 800
pods = w.claims[:n_pod].copy()
pod_off = np.arange(n_pod + 1, dtype=np.uint32)
rng = np.random.default_rng(7)
per = rng.integers(0, 12, n_pod)
cand_off = np.zeros(n_pod + 1, dtype=np.uint32); cand_off[1:] = np.cumsum(per)
cand_nodes = rng.integers(0, w.n_node + 3, int(cand_off[-1])).astype(np.uint32)      # some name no node
ctx = pkg.api.Context(device=local, stream=stream.cuda_stream)
ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
uid = [pkg.api.Context.comm_unique_id() if rank == 0 else None]
dist.broadcast_object_list(uid, src=0)
ctx.comm_init(uid[0], rank, world)
ctx.set_shard_map([r[0] for r in ranges] + [ranges[-1][1]], stray_rank=0)
ctx.set_shard_pairs(n_pod * w.n_node)
hs = [None] * world
dist.all_gather_object(hs, ctx.shard_export(w.n_out))
ctx.peer_import(hs)


def dv(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).to(dev)


d_claims, d_off = dv(w.claims), dv(w.out_off)
ctx.allocate_global_device(d_claims.data_ptr(), w.n_claim, d_off.data_ptr(), w.n_out, 0)
ctx.gather_read(np.zeros(w.n_out, dtype=R.OUT_DTYPE))
_, real = O.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
d_pods, d_po, d_cn, d_co = dv(pods), dv(pod_off), dv(cand_nodes), dv(cand_off)
dense_cn = np.tile(np.arange(w.n_node, dtype=np.uint32), n_pod)
dense_co = (np.arange(n_pod + 1, dtype=np.uint64) * w.n_node).astype(np.uint32)
for rep in range(2):                                   # repeated calls: both staging parities, rising sequence numbers
    for flags, oflags in ((0, 0), (pkg.api.F_EXHAUSTIVE, O.F_EXHAUSTIVE)):
        for form, cn, co, dcn, dco in (("dense", dense_cn, dense_co, None, None), ("candidates", cand_nodes, cand_off, d_cn, d_co)):
            n_pair = int(co[-1])
            bits = torch.zeros((n_pair + 7) // 8, dtype=torch.uint8, device=dev)
            ctx.unsuitable_global_device(d_pods.data_ptr(), n_pod, d_po.data_ptr(), n_pod, None if dcn is None else dcn.data_ptr(),
                                         None if dco is None else dco.data_ptr(), n_pair, bits.data_ptr(), flags)
            ctx.sync()
            ref = O.unsuitable(real, w.node_off, w.table, pods, pod_off, cn, co, flags=oflags)
            ok = bits.cpu().numpy().tobytes() == ref.tobytes()
            fails += not ok
            if rank == 0:
                print(f"sharded UnsuitableNodes rep {rep}, {form}, flags {flags}: {'OK' if ok else 'MISMATCH'} ({n_pair} pairs, {world} ranks)")
dist.barrier()
ctx.close()
t = torch.tensor([fails], device=dev); dist.all_reduce(t)
if rank == 0:
    print("ALL OK" if int(t.item()) == 0 else f"{int(t.item())} FAILURES")
dist.destroy_process_group()
sys.exit(1 if int(t.item()) else 0)
