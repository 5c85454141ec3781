"""Sharded search over int8 index shards (one rank per GPU, NCCL).  Launched by tests/test_index_i8_gpu.py, or by hand:
  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29519 tests/index_i8_dist_worker.py
Every rank holds a contiguous row shard of an int8 index and calls om_index_search_sharded; the global (D, I) must equal
those of ONE unsharded int8 index bit for bit (both are the exact top-k over the same stored rows), on even and on skewed
shards.  A rank that committed a row with a non-finite scale makes the sharded search fail on every rank, and a reset on
that rank clears it.  At world size 1 the same entry point runs over a one-rank communicator."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmatch_b200.index import FlatIPIndex, _wrap_device, comm_for  # noqa: E402

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
comm = comm_for(None)


def shard(x, bounds):
    idx = FlatIPIndex(x.shape[1], dtype=torch.int8)
    idx.add(torch.from_numpy(x[bounds[rank]:bounds[rank + 1]]).cuda())
    return idx


def check(x, q, k, bounds, what):
    whole = FlatIPIndex(x.shape[1], dtype=torch.int8)
    whole.add(x)
    qd = torch.from_numpy(q).cuda()
    D0, I0 = whole.search_device(qd, k)
    local = shard(x, bounds)
    D, I = local.search_sharded_device(comm, qd, k, id_offset=int(bounds[rank]))
    assert torch.equal(I, I0), "%s: ids differ from the unsharded int8 index" % what
    assert torch.equal(D.view(torch.int32), D0.view(torch.int32)), "%s: scores differ from the unsharded int8 index" % what
    print("rank %d %s: uncertified %d / %d (unsharded %d), exact %d" % (rank, what, local.stat("uncertified"), q.shape[0],
                                                                         whole.stat("uncertified"), local.stat("exact_queries")))
    return local


rng = np.random.default_rng(0)  # same data on every rank
n, d = 60000, 96
x = rng.standard_normal((n, d), dtype=np.float32)
q = rng.standard_normal((300, d), dtype=np.float32)
even = np.linspace(0, n, world + 1).astype(int)
for nq in (7, 300):
    for k in (10, 1000):
        check(x, q[:nq], k, even, "even shards nq=%d k=%d" % (nq, k))

# skewed shards: the answer lives on the last rank (rows aligned with the queries' direction)
v = rng.standard_normal(d, dtype=np.float32)
xs = rng.standard_normal((n, d), dtype=np.float32)
xs[even[-2]:n] += 3 * v
qs = (v + 0.3 * rng.standard_normal((129, d), dtype=np.float32)).astype(np.float32)
check(xs, qs, 100, even, "skewed shards")

# near-duplicates colliding after quantisation across shards: the exact level answers
xd = x.copy()
dup = rng.choice(n, 5000, replace=False)
xd[dup] = v + 1e-6 * rng.standard_normal((5000, d), dtype=np.float32)
qd = (v + 0.1 * rng.standard_normal((5, d), dtype=np.float32)).astype(np.float32)
loc = check(xd, qd, 10, even, "int8 collisions")
assert loc.stat("exact_queries") > 0, "premise: the exact level must run"

# a row with a non-finite scale committed on rank 0 fails the search on every rank until rank 0 resets
idx = shard(x, even)
if rank == 0:
    rows = idx.reserve_rows(1)
    pitch = rows.stride(0)
    dpad = (d + 15) // 16 * 16
    full = _wrap_device(rows.data_ptr(), (1, pitch), pitch, torch.int8)
    full.zero_()
    full[0, dpad:dpad + 4] = torch.tensor([float("inf")], device="cuda").view(torch.int8)
    idx.commit_rows(1)
failed = False
try:
    idx.search_sharded_device(comm, torch.from_numpy(q[:3]).cuda(), 5, id_offset=int(even[rank]))
except RuntimeError as e:
    failed = "inf or NaN" in str(e)
assert failed, "rank %d: the sharded search did not refuse the non-finite row" % rank
assert idx.stat("nonfinite_rows") == (1 if rank == 0 else 0)
if rank == 0:
    idx.reset()
    idx.add(x[even[0]:even[1]])
D, I = idx.search_sharded_device(comm, torch.from_numpy(q[:3]).cuda(), 5, id_offset=int(even[rank]))
assert (I >= 0).all()

dist.barrier()
dist.destroy_process_group()
if rank == 0:
    print("I8 DIST OK (world %d)" % world)
