"""Filtered sharded search (one rank per GPU, NCCL).  Launched by tests/test_index_filter_gpu.py, or by hand:
  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29521 tests/index_filter_dist_worker.py
Every rank holds a contiguous row shard and calls om_index_search_sharded_filtered with the same queries, the same
exclusion CSR (global ids) and its slice of one global bitmap; the global (D, I) must equal the filtered search of ONE
unsharded index bit for bit, also when the bitmap empties a shard, when a shard holds no rows, and when one rank passes
a null filter while the others pass bitmaps.  At world size 1 the same entry point runs over a one-rank communicator."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes  # noqa: E402

from openmatch_b200 import _lib  # noqa: E402
from openmatch_b200.index import FlatIPIndex, ShardedFlatIPIndex, comm_for, local_allow, pack_allow  # noqa: E402

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
comm = comm_for(None)

rng = np.random.default_rng(0)  # same data on every rank
n, d = 60000, 96
x = rng.standard_normal((n, d), dtype=np.float32)
q = rng.standard_normal((300, d), dtype=np.float32)
bounds = np.linspace(0, n, world + 1).astype(int)


def check(dtype, nq, k, allow, excl, what, bounds=bounds):
    whole = FlatIPIndex(d, dtype=dtype)
    whole.add(x)
    qd = torch.from_numpy(q[:nq]).cuda()
    ex = excl[:nq] if excl is not None else None
    D0, I0 = whole.search_device(qd, k, allow=allow, exclude=ex)
    local = FlatIPIndex(d, dtype=dtype)
    if bounds[rank + 1] > bounds[rank]:
        local.add(torch.from_numpy(x[bounds[rank]:bounds[rank + 1]]).cuda())
    mine = local_allow(allow, int(bounds[rank]), local.ntotal)  # this rank's slice of the global bitmap
    D, I = local.search_sharded_device(comm, qd, k, int(bounds[rank]), allow=mine, exclude=ex)
    assert torch.equal(I, I0), "%s: ids differ from the unsharded filtered search" % what
    assert torch.equal(D.view(torch.int32), D0.view(torch.int32)), "%s: scores differ" % what
    print("rank %d %s: uncertified %d, exact %d" % (rank, what, local.stat("uncertified"), local.stat("exact_queries")))


unsharded = FlatIPIndex(d)
unsharded.add(x)
_, Itop = unsharded.search(q, 200)
excl = [list(rng.choice(Itop[i, :100], 60, replace=False)) + [n + 5, 3] for i in range(300)]
half = rng.random(n) < 0.5
one_shard = np.zeros(n, bool)
one_shard[rng.choice(bounds[1], 3000, replace=False)] = True  # rows of rank 0 only: every other shard is empty
for dtype in (torch.float32, torch.float16, torch.int8):
    for nq, k in ((7, 10), (300, 100), (129, 1000)):
        check(dtype, nq, k, half, None, "%s half nq=%d k=%d" % (dtype, nq, k))
        check(dtype, nq, k, None, excl, "%s exclusions nq=%d k=%d" % (dtype, nq, k))
    check(dtype, 300, 100, one_shard, excl, "%s one shard allowed + exclusions" % dtype)
    check(dtype, 40, 50, np.zeros(n, bool), None, "%s nothing allowed" % dtype)

# ranks that differ in whether they pass a filter at all: rank 0 passes a null filter pointer (all of its rows are
# eligible), the others their slice of a bitmap; the collective must stay in step and answer the global filter
mixed = half.copy()
mixed[:bounds[1]] = True
for dtype in (torch.float32, torch.int8):
    whole = FlatIPIndex(d, dtype=dtype)
    whole.add(x)
    qd = torch.from_numpy(q[:100]).cuda()
    D0, I0 = whole.search_device(qd, 50, allow=mixed)
    local = FlatIPIndex(d, dtype=dtype)
    local.add(torch.from_numpy(x[bounds[rank]:bounds[rank + 1]]).cuda())
    D = torch.empty_like(D0)
    I = torch.empty_like(I0)
    f, words = None, None
    if rank > 0:
        words = pack_allow(local_allow(mixed, int(bounds[rank]), local.ntotal), local.ntotal, "cuda")
        f = _lib.SearchFilter()
        f.allow_bits, f.allow_words = words.data_ptr(), words.numel()
    rc = local._lib.om_index_search_sharded_filtered(local._h, comm._h, qd.data_ptr(), _lib.OM_DEVICE, 100, 50, D.data_ptr(),
                                                     I.data_ptr(), _lib.OM_DEVICE, int(bounds[rank]),
                                                     ctypes.byref(f) if f is not None else None,
                                                     torch.cuda.current_stream().cuda_stream)
    _lib.check(rc)
    assert torch.equal(I, I0) and torch.equal(D.view(torch.int32), D0.view(torch.int32)), "%s: null filter on rank 0" % dtype

# an empty shard: rank 0 holds no rows (its bitmap slice is empty); at world size 1 the whole index is empty
empty0 = np.concatenate([[0], np.linspace(0, n, world).astype(int)]) if world > 1 else None
for dtype in (torch.float32, torch.float16, torch.int8):
    if empty0 is not None:
        check(dtype, 64, 100, half, excl, "%s rank 0 empty, bitmap + exclusions" % dtype, bounds=empty0)
        check(dtype, 64, 100, half, None, "%s rank 0 empty, bitmap" % dtype, bounds=empty0)
    else:
        local = FlatIPIndex(d, dtype=dtype)
        D, I = local.search_sharded_device(comm, torch.from_numpy(q[:5]).cuda(), 10, 0,
                                           allow=torch.zeros(0, dtype=torch.bool), exclude=excl[:5])
        assert (I == -1).all(), "%s: empty index" % dtype

# the ShardedFlatIPIndex surface: the bitmap over global ids, packed words accepted as well
sh = ShardedFlatIPIndex(d)
sh.add_local(x[bounds[rank]:bounds[rank + 1]])
sh.finalize_offsets()
D, I = sh.search(q[:50], 20, allow=torch.from_numpy(half), exclude=excl[:50])
D0, I0 = unsharded.search(q[:50], 20, allow=half, exclude=excl[:50])
assert (I == I0).all() and (D.view(np.uint32) == D0.view(np.uint32)).all(), "ShardedFlatIPIndex.search"

dist.barrier()
dist.destroy_process_group()
if rank == 0:
    print("FILTER DIST OK (world %d)" % world)
