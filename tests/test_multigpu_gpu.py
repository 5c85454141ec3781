"""GPU, real NCCL: spawns one rank per GPU (2 ranks) running tests/dist_worker.py when the box has >= 2 GPUs.
On a single-GPU box the same library entry point (om_index_search_sharded) and the distributed loss are still
exercised through a world-size-1 NCCL group, and the merge of the exchanged lists through logical shards
(tests/test_search_gpu.py::test_sharded_merge_matches_unsharded)."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _torchrun(nproc, script, timeout=900):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), script]
    env = dict(os.environ, NCCL_DEBUG="WARN", OMP_NUM_THREADS="8")
    return subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)


def test_two_rank_nccl_parity():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs (covered at world size 1 below and by bench.py --gpus N's parity check)")
    r = _torchrun(2, os.path.join("tests", "dist_worker.py"))
    assert r.returncode == 0 and "DIST CHECK OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


_WORLD1 = r'''
import os, sys, types
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.getcwd())
import oracle
from openmatch_b200.index import FlatIPIndex, comm_for, sharded_search_device
from openmatch_b200.loss import DistributedContrastiveLoss
torch.cuda.set_device(0)
dist.init_process_group("nccl", device_id=torch.device("cuda", 0))
rng = np.random.default_rng(3)
x = rng.integers(-6, 7, (9000, 64)).astype(np.float32); q = rng.integers(-6, 7, (13, 64)).astype(np.float32)
idx = FlatIPIndex(64); idx.add(x)
comm = comm_for(None)
assert comm.world == 1
D, I = idx.search_sharded_device(comm, torch.from_numpy(q).cuda(), 50, id_offset=1000)
D0, I0 = oracle.flat_ip_search(q, x, 50)
assert (I.cpu().numpy() == I0 + 1000).all() and (D.cpu().numpy() == D0).all()
xq = (torch.randn(4, 64) * 0.5).to(torch.bfloat16); yp = (torch.randn(32, 64) * 0.5).to(torch.bfloat16)
a, b = xq.cuda().requires_grad_(), yp.cuda().requires_grad_()
loss = DistributedContrastiveLoss()(a, b); loss.backward()
want, dx, dy, _ = oracle.contrastive_loss_fwd_bwd(xq.float().numpy(), yp.float().numpy())
assert abs(loss.item() - want) <= 1e-3 * max(1.0, abs(want))
assert np.linalg.norm(a.grad.float().cpu().numpy() - dx) <= 1e-2 * np.linalg.norm(dx)
dist.destroy_process_group()
print("WORLD1 OK")
'''


def test_world_size_one_nccl_paths(tmp_path):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    script = tmp_path / "w1.py"
    script.write_text(_WORLD1)
    r = _torchrun(1, str(script), timeout=600)
    assert r.returncode == 0 and "WORLD1 OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
