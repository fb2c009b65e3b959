"""GPU suite: the torchrun multi-GPU checks (tests/multi_gpu_*check.py), one process per GPU with peer buffers mapped
through IPC handles, as part of `pytest -m gpu`; skipped on a box with fewer than 2 GPUs."""
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPTS = ["multi_gpu_check", "multi_gpu_shard_unsuitable_check", "multi_gpu_shard_pods_check", "multi_gpu_shard_sync_check",
           "multi_gpu_shard_dealloc_check", "multi_gpu_shard_place_check", "multi_gpu_shard_preempt_check",
           "multi_gpu_shard_preempt_pdb_check", "multi_gpu_shard_capacity_check", "multi_gpu_shard_preempt_place_check"]


def _free_port():
    """A port no one held a moment ago.  The socket closes before torchrun binds the port, so another process could take
    it in between; that would fail this run's rendezvous, not give it a wrong answer."""
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.parametrize("script", SCRIPTS, ids=SCRIPTS)
def test_multi_process(script):
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = (2 if n < 4 else 4) if script == "multi_gpu_check" else min(n, 4)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
                        os.path.join(ROOT, "tests", script + ".py")],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
