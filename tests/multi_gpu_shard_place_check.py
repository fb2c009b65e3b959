#!/usr/bin/env python
"""Multi-GPU parity check of the sharded place pods (run under torchrun on the GPUs of one box; not collected by pytest).
One process per GPU, peer buffers mapped with IPC handles (dra_shard_export / dra_peer_import), so every state word and
packet crosses NVLink.  A sharded Allocate without DRA_F_FRESH_INVENTORY first makes the ranks' inventories diverge; then
the place-pods call runs in the dense form, with 8 random candidates and with every node descending, under every flag.
Every rank's whole table, pod_node and own inventory range must equal the CPU oracle's on the real state.

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/multi_gpu_shard_place_check.py
"""
import importlib, os, sys
import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
pkg = importlib.import_module("k8s-dra-driver_b200")
import place_oracle as P
R = pkg.records
F_EXH, F_FRESH = pkg.api.F_EXHAUSTIVE, pkg.api.F_FRESH_INVENTORY

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
os.environ.setdefault("NCCL_DEBUG", "WARN")
torch.cuda.set_device(local)
dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
dev = torch.device("cuda", local)
stream = torch.cuda.Stream(device=dev); torch.cuda.set_stream(stream)
fails = 0

w, pod_off = pkg.synth.pods(2000, 24 * world, 17)
bounds = [w.n_node * r // world for r in range(world)] + [w.n_node]
g0, g1 = int(w.node_off[bounds[rank]]), int(w.node_off[bounds[rank + 1]])
first = int(pod_off[300])
claims = w.claims[first:].copy()
po = (pod_off[300:] - first).astype(np.uint32)
n_pod = len(po) - 1
ctx = pkg.api.Context(device=local, stream=stream.cuda_stream)
ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
uid = [pkg.api.Context.comm_unique_id() if rank == 0 else None]
dist.broadcast_object_list(uid, src=0)
ctx.comm_init(uid[0], rank, world)
ctx.set_shard_map(bounds, stray_rank=world - 1)
ctx.set_shard_place(n_pod)
hs = [None] * world
dist.all_gather_object(hs, ctx.shard_export(max(w.n_claim, 1)))
ctx.peer_import(hs)


def dv(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).to(dev)


def real_state():
    parts = [None] * world
    dist.all_gather_object(parts, ctx.get_inventory()[g0:g1].tobytes())
    real = w.gpus.copy()
    for r in range(world):
        a, b = int(w.node_off[bounds[r]]), int(w.node_off[bounds[r + 1]])
        real[a:b] = np.frombuffer(parts[r], dtype=w.gpus.dtype)
    return real


def check(what, cn, co, flags):
    global fails
    src = w.gpus if flags & F_FRESH else real_state()
    ref, ref_node, ref_inv = P.place_pods(src, w.node_off, w.table, claims, po, cn, co, None, len(claims),
                                          P.F_EXHAUSTIVE if flags & F_EXH else 0)
    d_c, d_p = dv(claims), dv(po)
    d_n = dv(cn) if cn is not None else None
    d_o = dv(co) if co is not None else None
    d_pn = torch.zeros(n_pod * 4, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    ctx.place_pods_global_device(d_c.data_ptr(), len(claims), d_p.data_ptr(), n_pod, d_n.data_ptr() if d_n is not None else None,
                                 d_o.data_ptr() if d_o is not None else None, int(co[-1]) if co is not None else 0, None,
                                 len(claims), d_pn.data_ptr(), flags)
    ctx.sync()
    got = ctx.gather_read(np.zeros(len(claims), dtype=R.OUT_DTYPE))
    node = d_pn.cpu().numpy().view(np.uint32)
    inv = ctx.get_inventory()
    ok = got.tobytes() == ref.tobytes() and node.tobytes() == ref_node.tobytes() and inv[g0:g1].tobytes() == ref_inv[g0:g1].tobytes()
    t = torch.tensor([0 if ok else 1], device=dev); dist.all_reduce(t)
    fails += int(t.item()) != 0
    if rank == 0:
        print(f"sharded place pods, {what}: {'OK' if int(t.item()) == 0 else 'MISMATCH'} "
              f"({n_pod} pods, {int((ref_node != 0xFFFFFFFF).sum())} placed, {world} ranks)")


d_first = dv(w.claims[:first])
ctx.allocate_global_device(d_first.data_ptr(), first, None, first, 0)
ctx.gather_read(np.zeros(first, dtype=R.OUT_DTYPE))
rng = np.random.default_rng(5)
asc = np.tile(np.arange(w.n_node, dtype=np.uint32), n_pod)
every = (np.arange(n_pod + 1) * w.n_node).astype(np.uint32)
forms = {"dense": (None, None),
         "8 random": (rng.integers(0, w.n_node + 2, n_pod * 8).astype(np.uint32), (np.arange(n_pod + 1) * 8).astype(np.uint32)),
         "descending": (asc[::-1].copy(), every)}
for name, (cn, co) in forms.items():
    for flags, fname in ((0, "first-fit"), (F_EXH, "exhaustive"), (F_FRESH, "fresh first-fit"), (F_EXH | F_FRESH, "fresh exhaustive")):
        check(f"{name}, {fname}", cn, co, flags)
dist.barrier()
ctx.close()
t = torch.tensor([fails], device=dev); dist.all_reduce(t)
if rank == 0:
    print("ALL OK" if int(t.item()) == 0 else f"{int(t.item())} FAILURES")
dist.destroy_process_group()
sys.exit(1 if int(t.item()) else 0)
