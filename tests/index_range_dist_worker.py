"""Sharded range search (one rank per GPU, NCCL).  Launched by tests/test_index_range_gpu.py, or by hand:
  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29523 tests/index_range_dist_worker.py
Every rank holds a contiguous row shard and calls om_index_range_search_sharded with the same queries and radii; the
global (lims, D, I) must equal the range search of ONE unsharded index bit for bit, on every storage, also when a shard
holds no rows, when one shard holds all the results, with re-sweeps, and when the ranks' id offsets do not rise with
rank.  At world size 1 the same entry point runs over a one-rank communicator."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmatch_b200.index import FlatIPIndex, ShardedFlatIPIndex, comm_for  # noqa: E402

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
comm = comm_for(None)

rng = np.random.default_rng(0)  # same data on every rank
n, d = 50000, 96
x = rng.standard_normal((n, d), dtype=np.float32)
q = rng.standard_normal((300, d), dtype=np.float32)
bounds = np.linspace(0, n, world + 1).astype(int)


def same(a, b, what):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    assert a.shape == b.shape, "%s: shape %s vs %s" % (what, a.shape, b.shape)
    if a.dtype == np.float32:
        a, b = a.view(np.uint32), b.view(np.uint32)
    assert np.array_equal(a, b), what


def check(dtype, xs, rho, what, bounds=bounds, offsets=None, **params):
    whole = FlatIPIndex(d, dtype=dtype)
    whole.add(xs)
    qd = torch.from_numpy(q).cuda()
    want = whole.range_search_device(qd, rho)
    local = FlatIPIndex(d, dtype=dtype)
    if bounds[rank + 1] > bounds[rank]:
        local.add(torch.from_numpy(xs[bounds[rank]:bounds[rank + 1]]).cuda())
    for name, v in params.items():
        local.set_param(name, v)
    off = int(bounds[rank]) if offsets is None else int(offsets[rank])
    got = local.range_search_sharded_device(comm, qd, rho, off)
    if offsets is not None:  # compare with the single index's ids mapped to the shards' ids
        ids = want[2].cpu().numpy()
        shard = np.searchsorted(bounds, ids, side="right") - 1
        mapped = ids - bounds[shard] + np.asarray(offsets)[shard]
        want = (want[0], want[1], torch.from_numpy(mapped).cuda())
        # the merge orders equal scores by the ids themselves: re-sort the single index's ties by the mapped ids
        lims, D, I = (t.cpu().numpy() for t in want)
        for i in range(q.shape[0]):
            a, b = lims[i], lims[i + 1]
            o = np.lexsort((I[a:b], -D[a:b].astype(np.float64)))
            D[a:b], I[a:b] = D[a:b][o], I[a:b][o]
        want = tuple(torch.from_numpy(t).cuda() for t in (lims, D, I))
    for a, b, name in zip(got, want, ("lims", "D", "I")):
        same(a, b, "%s %s: %s" % (what, dtype, name))


rho_mix = np.where(np.arange(300) % 3 == 0, 10.0, np.where(np.arange(300) % 3 == 1, 14.0, 20.0)).astype(np.float32)
for dtype in (torch.float32, torch.float16, torch.int8):
    check(dtype, x, rho_mix, "mixed radii")
check(torch.float32, x, rho_mix, "re-sweeps", range_list=256)
check(torch.float32, x, np.float32(-np.inf), "radius -inf")
check(torch.float16, x, np.float32(np.inf), "radius +inf")
check(torch.float32, x, rho_mix, "exact scan", exact_only=1)
if world > 1:
    empty = np.array([0, 0] + list(np.linspace(0, n, world)[1:].astype(int)))[: world + 1]
    check(torch.float32, x, rho_mix, "an empty shard", bounds=empty)
    hot = x.copy()
    hot[bounds[-2]:] *= 3.0  # the last shard holds every result at radius 60
    check(torch.float16, hot, np.float32(60.0), "one shard holds all results")
    rev = [int(n - bounds[r + 1]) for r in range(world)]  # id offsets that fall with rank
    check(torch.float32, x, rho_mix, "falling id offsets", offsets=rev)
sharded = ShardedFlatIPIndex(d)
sharded.add_local(x[bounds[rank]:bounds[rank + 1]])
sharded.finalize_offsets()
lims, D, I = sharded.range_search(q[:5], 12.0)
whole = FlatIPIndex(d)
whole.add(x)
l0, D0, I0 = whole.range_search(q[:5], 12.0)
assert np.array_equal(lims, l0) and np.array_equal(D.view(np.uint32), D0.view(np.uint32)) and np.array_equal(I, I0)
dist.barrier()
if rank == 0:
    print("RANGE DIST OK")
dist.destroy_process_group()
