#!/usr/bin/env python
"""Multi-GPU parity check of the sharded preemption call with disruption budgets (run under torchrun on the GPUs of one
box; not collected by pytest).  One process per GPU, peer buffers mapped with IPC handles (dra_shard_export /
dra_peer_import), so every partial and its violation count crosses NVLink.  Each rank holds the real world on its own node
range and the empty inventory elsewhere; budgets span the ranks' nodes; the call runs in the dense form and with 16 random
candidates, under both flags.  Every rank's eight outputs must equal the CPU oracle's on the real world, and no rank's
inventory may change.

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/multi_gpu_shard_preempt_pdb_check.py
"""
import importlib, os, sys
import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
pkg = importlib.import_module("k8s-dra-driver_b200")
import preempt_oracle as P
import preempt_oracle as PB
R = pkg.records
F_EXH = pkg.api.F_EXHAUSTIVE

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
os.environ.setdefault("NCCL_DEBUG", "WARN")
torch.cuda.set_device(local)
dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
dev = torch.device("cuda", local)
stream = torch.cuda.Stream(device=dev); torch.cuda.set_stream(stream)
fails = 0

w = pkg.synth.preempt(n_node=32 * world, gpus_per_node=8, n_pending=200, seed=23)
n_node = len(w.node_off) - 1
n_pod = len(w.pod_off) - 1
bounds = [n_node * r // world for r in range(world)] + [n_node]
g0, g1 = int(w.node_off[bounds[rank]]), int(w.node_off[bounds[rank + 1]])
mine = w.empty.copy()
mine[g0:g1] = w.gpus[g0:g1]
ctx = pkg.api.Context(device=local, stream=stream.cuda_stream)
ctx.set_table(w.table); ctx.set_inventory(mine, w.node_off)
uid = [pkg.api.Context.comm_unique_id() if rank == 0 else None]
dist.broadcast_object_list(uid, src=0)
ctx.comm_init(uid[0], rank, world)
ctx.set_shard_map(bounds, stray_rank=0)
ctx.set_shard_preempt(n_pod, n_pod * n_node, 16)
hs = [None] * world
dist.all_gather_object(hs, ctx.shard_export(max(len(w.run_claims), 1)))
ctx.peer_import(hs)


def dv(a):
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).to(dev) if a.nbytes else torch.zeros(16, dtype=torch.uint8, device=dev)


brng = np.random.default_rng(11)
allowed = np.array([0, 1, 2, -1], np.int32)
run_pdb = brng.integers(0, 5, len(w.run_prio)).astype(np.uint32)
run_pdb[run_pdb == 4] = 0xFFFFFFFF
keep = [dv(x) for x in (w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, run_pdb, allowed)]
run = pkg.api.RunningPods(keep[3].data_ptr(), len(w.run_claims), keep[4].data_ptr(), len(w.run_pod_off) - 1,
                          keep[5].data_ptr(), None, keep[6].data_ptr(), len(w.run_out))
bud = pkg.api.DisruptionBudgets(keep[7].data_ptr(), keep[8].data_ptr(), len(allowed))


def check(what, cn, co, flags):
    global fails
    ref = PB.preempt_pdb(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off,
                        w.run_prio, w.run_out, run_pdb, allowed, None, cn, co, 16, P.F_EXHAUSTIVE if flags & F_EXH else 0)
    n_pair = n_pod * n_node if co is None else int(co[-1])
    d_n = dv(cn) if cn is not None else None
    d_o = dv(co) if co is not None else None
    sizes = (n_pair, n_pair * 4, n_pod * 4, n_pod, n_pod * 4, n_pod * 16 * 4, n_pair * 4, n_pod * 4)
    outs = [torch.zeros(s + 16, dtype=torch.uint8, device=dev) for s in sizes]
    torch.cuda.synchronize()
    p = [o.data_ptr() for o in outs]
    ctx.preempt_pdb_global_device(keep[0].data_ptr(), len(w.claims), keep[1].data_ptr(), keep[2].data_ptr(), n_pod,
                                  d_n.data_ptr() if d_n is not None else None, d_o.data_ptr() if d_o is not None else None,
                                  n_pair, run, bud, p[0], p[1], p[6], p[2], p[3], p[4], p[7], p[5], 16, flags)
    ctx.sync()
    dt = (np.uint8, np.uint32, np.uint32, np.uint8, np.uint32, np.uint32, np.uint32, np.uint32)
    got = [o.cpu().numpy()[:s].view(d) for o, s, d in zip(outs, sizes, dt)]
    ok = all(x.tobytes() == y.tobytes() for x, y in zip(got, ref)) and ctx.get_inventory().tobytes() == mine.tobytes()
    t = torch.tensor([0 if ok else 1], device=dev); dist.all_reduce(t)
    fails += int(t.item()) != 0
    if rank == 0:
        print(f"sharded preemption with budgets, {what}: {'OK' if int(t.item()) == 0 else 'MISMATCH'} "
              f"({n_pod} pods, {int((ref[3] == P.EVICT).sum())} evicting, {int(ref[7].sum())} violations, {world} ranks)")


rng = np.random.default_rng(5)
forms = {"dense": (None, None),
         "16 random": (rng.integers(0, n_node + 2, n_pod * 16).astype(np.uint32), (np.arange(n_pod + 1) * 16).astype(np.uint32))}
for name, (cn, co) in forms.items():
    for flags, fname in ((0, "first-fit"), (F_EXH, "exhaustive")):
        check(f"{name}, {fname}", cn, co, flags)
dist.barrier()
ctx.close()
t = torch.tensor([fails], device=dev); dist.all_reduce(t)
if rank == 0:
    print("ALL OK" if int(t.item()) == 0 else f"{int(t.item())} FAILURES")
dist.destroy_process_group()
sys.exit(1 if int(t.item()) else 0)
