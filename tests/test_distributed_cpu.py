"""CPU, world_size 2 over gloo: the global row offsets of a row-sharded index (uneven shards) and the
autograd-aware all-gather used for cross-device negatives."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, tmp):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from openmatch_b200.index import shard_offsets
        bounds = [0, 380, 1000]  # uneven shards
        offset, total = shard_offsets(bounds[rank + 1] - bounds[rank])
        assert (offset, total) == (bounds[rank], 1000)

        # cross-device negatives: gathered tensor is rank-major and only the local slice carries gradient
        from openmatch_b200.modeling.dense_retrieval_model import DRModel
        m = DRModel.__new__(DRModel)
        torch.nn.Module.__init__(m)
        m.world_size, m.process_rank = world, rank
        t = torch.full((2, 3), float(rank + 1), requires_grad=True)
        g = m.dist_gather_tensor(t)
        assert g.shape == (4, 3) and g[:2].eq(1).all() and g[2:].eq(2).all()
        g.sum().backward()
        assert t.grad.eq(1).all()
        with open(os.path.join(tmp, "ok.%d" % rank), "w") as f:
            f.write("ok")
    finally:
        dist.destroy_process_group()


def test_shard_offsets_and_gather_world2(tmp_path):
    port = _free_port()
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    assert all(os.path.exists(tmp_path / ("ok.%d" % r)) for r in range(2))
