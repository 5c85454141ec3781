"""Sharded filtered range search (one rank per GPU, NCCL).  Launched by tests/test_index_range_filter_gpu.py, or by hand:
  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29524 tests/index_range_filter_dist_worker.py
Every rank holds a contiguous row shard and calls om_index_range_search_sharded_filtered with the same queries, radii and
exclusions (global ids) and its own slice of a global bitmap; the global (lims, D, I) must equal the filtered range
search of ONE unsharded index bit for bit, on every storage, with re-sweeps and on the exact scan.  One rank may pass a
null filter while the others pass theirs: its rows are then all eligible.  At world size 1 the same entry point runs
over a one-rank communicator."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmatch_b200 import _lib  # noqa: E402
from openmatch_b200.index import FlatIPIndex, ShardedFlatIPIndex, comm_for, sharded_range_search_device  # noqa: E402

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
comm = comm_for(None)

rng = np.random.default_rng(0)  # same data on every rank
n, d, nq = 50000, 96, 300
x = rng.standard_normal((n, d), dtype=np.float32)
q = rng.standard_normal((nq, d), dtype=np.float32)
allow = rng.random(n) < 0.4
excl = [list(rng.choice(n, 100, replace=False)) for _ in range(nq)]
bounds = np.linspace(0, n, world + 1).astype(int)
lo, hi = int(bounds[rank]), int(bounds[rank + 1])
rho_mix = np.where(np.arange(nq) % 3 == 0, 8.0, np.where(np.arange(nq) % 3 == 1, 12.0, 16.0)).astype(np.float32)


def same(a, b, what):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    assert a.shape == b.shape, "%s: shape %s vs %s" % (what, a.shape, b.shape)
    if a.dtype == np.float32:
        a, b = a.view(np.uint32), b.view(np.uint32)
    assert np.array_equal(a, b), what


def null_filter_call(local, qd, rho, off):
    """om_index_range_search_sharded_filtered with a null filter: this rank's rows unfiltered, in step with the others"""
    lib = local._lib
    r = torch.as_tensor(rho, dtype=torch.float32).expand(nq).contiguous().cuda()
    lims = torch.empty(nq + 1, dtype=torch.int64)
    stream = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.om_index_range_search_sharded_filtered(local._h, comm._h, qd.data_ptr(), _lib.OM_DEVICE, nq,
                                                          r.data_ptr(), lims.data_ptr(), _lib.OM_HOST, off, None,
                                                          stream))
    total = int(lims[-1])
    D = torch.empty(total, dtype=torch.float32, device="cuda")
    I = torch.empty(total, dtype=torch.int64, device="cuda")
    _lib.check(lib.om_index_range_results(local._h, D.data_ptr() or None, I.data_ptr() or None, _lib.OM_DEVICE, stream))
    return lims.cuda(), D, I


def check(dtype, rho, what, null_rank=None, **params):
    # the single index: the global bitmap (the null rank's rows all allowed) and the exclusions that fall on ranks
    # with a filter (a null filter excludes nothing)
    g_allow = allow.copy()
    g_excl = excl
    if null_rank is not None:
        a, b = int(bounds[null_rank]), int(bounds[null_rank + 1])
        g_allow[a:b] = True
        g_excl = [[i for i in e if not a <= i < b] for e in excl]
    whole = FlatIPIndex(d, dtype=dtype)
    whole.add(x)
    for name, v in params.items():
        whole.set_param(name, v)
    qd = torch.from_numpy(q).cuda()
    want = whole.range_search_device(qd, rho, allow=g_allow, exclude=g_excl)
    local = FlatIPIndex(d, dtype=dtype)
    if hi > lo:
        local.add(torch.from_numpy(x[lo:hi]).cuda())
    for name, v in params.items():
        local.set_param(name, v)
    if rank == null_rank:
        got = null_filter_call(local, qd, rho, lo)
    else:
        got = local.range_search_sharded_device(comm, qd, rho, lo, allow=allow[lo:hi], exclude=excl)
    for a, b, name in zip(got, want, ("lims", "D", "I")):
        same(a, b, "%s %s: %s" % (what, dtype, name))


for dtype in (torch.float32, torch.float16, torch.int8):
    check(dtype, rho_mix, "mixed radii")
check(torch.float32, rho_mix, "re-sweeps", range_list=256)
check(torch.float32, np.float32(-np.inf), "radius -inf")
check(torch.float32, rho_mix, "exact scan", exact_only=1)
check(torch.float16, rho_mix, "a rank with a null filter", null_rank=world - 1)
# the Python wrappers: the global bitmap sliced per rank
qd = torch.from_numpy(q[:20]).cuda()
whole = FlatIPIndex(d)
whole.add(x)
want = whole.range_search_device(qd, 10.0, allow=allow, exclude=excl[:20])
local = FlatIPIndex(d)
local.add(x[lo:hi])
got = sharded_range_search_device(local, qd, 10.0, lo, allow=allow, exclude=excl[:20])
for a, b, name in zip(got, want, ("lims", "D", "I")):
    same(a, b, "sharded_range_search_device: %s" % name)
sharded = ShardedFlatIPIndex(d)
sharded.add_local(x[lo:hi])
sharded.finalize_offsets()
lims, D, I = sharded.range_search(q[:20], 10.0, allow=allow, exclude=excl[:20])
for a, b, name in zip((lims, D, I), want, ("lims", "D", "I")):
    same(torch.from_numpy(a), b, "ShardedFlatIPIndex.range_search: %s" % name)
dist.barrier()
if rank == 0:
    print("RANGE FILTER DIST OK")
dist.destroy_process_group()
