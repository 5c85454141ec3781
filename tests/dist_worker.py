"""Multi-GPU parity worker (one rank per GPU, NCCL).  Launched by tests/test_multigpu_gpu.py when the box has >= 2
GPUs, or by hand:
  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29517 tests/dist_worker.py
Covers, on real NCCL:
  * om_index_search_sharded (library-side exchange) on integer data (bit-exact vs the CPU oracle), on Gaussian data
    (bit-identical to the same search on ONE unsharded index + eps-check vs float64), on a near-duplicate cluster that
    forces the exact-scan level, and on skewed shards that force the full-width exchange;
  * Retriever.from_embeddings / _search_sharded with more embedding files than ranks (reference :43-58,94-106);
  * DistributedContrastiveLoss (reference loss.py:18-38) and DRModel.forward with negatives_x_device
    (reference dense_retrieval_model.py:104-125,247-258) against the oracle on the gathered batch.
"""
import os
import pickle
import sys
import tempfile
import types

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle  # noqa: E402
from openmatch_b200.index import FlatIPIndex, ShardedFlatIPIndex, comm_for  # noqa: E402
from openmatch_b200.loss import DistributedContrastiveLoss  # noqa: E402

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
report = []


def eps_check(q, x, D, I, k, rel):
    s = q.astype(np.float64) @ x.astype(np.float64).T
    best = -np.sort(-s, axis=1)[:, :k]
    eps = rel * np.linalg.norm(q, axis=1, keepdims=True) * np.linalg.norm(x, axis=1).max()
    got = np.take_along_axis(s, I, axis=1)
    assert (np.abs(got - best) <= eps).all(), "ids are not an eps-valid top-k"
    assert (np.abs(D - got) <= eps).all(), "scores deviate from the float64 scores"


def sharded(x, bounds):
    idx = ShardedFlatIPIndex(x.shape[1])
    idx.add_local(x[bounds[rank]:bounds[rank + 1]])
    idx.finalize_offsets()
    assert idx.ntotal == x.shape[0] and idx.offset == bounds[rank]
    return idx


def uneven(n):
    b = np.linspace(0, n, world + 1).astype(int)
    b[1:-1] += 37
    return b


# ---- 1. integer data: bit-exact vs the oracle, incl. ties ----
rng = np.random.default_rng(0)  # same data on every rank
n, d, nq, k = 40000, 128, 77, 100
x = rng.integers(-6, 7, (n, d)).astype(np.float32)
q = rng.integers(-6, 7, (nq, d)).astype(np.float32)
idx = sharded(x, uneven(n))
D, I = idx.search(q, k)
D0, I0 = oracle.flat_ip_search(q, x, k)
assert (I == I0).all() and (D == D0).all(), "sharded integer search differs from the oracle on rank %d" % rank
report.append("integer exact")

# ---- 2. Gaussian data: identical to the unsharded index, eps-valid vs float64, all ranks agree ----
n, d, nq, k = 200000, 256, 300, 1000  # > 128 queries: the scan runs on 2-CTA clusters
x = rng.standard_normal((n, d), dtype=np.float32)
q = rng.standard_normal((nq, d), dtype=np.float32)
idx = sharded(x, uneven(n))
D, I = idx.search(q, k)
one = FlatIPIndex(d)
one.add(x)
D1, I1 = one.search(q, k)
assert (I == I1).all() and (D == D1).all(), "sharded Gaussian search differs from the single-shard search"
eps_check(q, x, D, I, k, 2e-5)
assert idx.local.stat("exact_queries") == 0 and idx.local.stat("uncertified") <= 2
sums = torch.tensor([float(I.sum()), float(D.astype(np.float64).sum())], dtype=torch.float64, device="cuda")
lo, hi = sums.clone(), sums.clone()
dist.all_reduce(lo, op=dist.ReduceOp.MIN)
dist.all_reduce(hi, op=dist.ReduceOp.MAX)
assert torch.equal(lo, hi), "ranks disagree on the merged result"
report.append("gaussian == unsharded (uncertified %d)" % idx.local.stat("uncertified"))
del one

# ---- 3. near-duplicate cluster spread over the shards: certificate fails, exact scan answers ----
n, d, nq, k = 60000, 128, 5, 1000
x = rng.standard_normal((n, d), dtype=np.float32)
v = rng.standard_normal(d, dtype=np.float32)
dup = rng.choice(n, 9000, replace=False)
x[dup] = v + 1e-4 * rng.standard_normal((9000, d), dtype=np.float32)
q = (v + 0.1 * rng.standard_normal((nq, d), dtype=np.float32)).astype(np.float32)
idx = sharded(x, uneven(n))
D, I = idx.search(q, k)
stats3 = tuple(idx.local.stat(s) for s in ("uncertified", "uncertified_wide", "exact_queries"))
assert stats3[0] == nq, "the first level cannot certify a near-duplicate cluster: %s" % (stats3,)
if 9000 // world > 4096:  # more duplicates per shard than the widest list holds: only the exact scan can answer
    assert stats3[2] == nq, "expected the exact level, stats (uncertified, wide, exact): %s" % (stats3,)
one = FlatIPIndex(d)
one.add(x)
D1, I1 = one.search(q, k)
assert (I == I1).all() and (D == D1).all()
eps_check(q, x, D, I, k, 2e-6)
report.append("near-duplicates exact (uncertified %d, after wide level %d, exact scan %d)" % stats3)
del one

# ---- 4. skewed shards: every relevant row lives on the last rank, whose shard-sized list (kp / W + 6 sigma + 32 < k) cannot
#         hold the answer -> its floor is high, the certificate fails, the 4096-wide level answers ----
n, d, nq, k = 30000, 64, 9, 1000
x = rng.integers(-3, 4, (n, d)).astype(np.float32)
q = rng.integers(1, 4, (nq, d)).astype(np.float32)
hot = n - 3000
x[hot:] = rng.integers(2, 4, (3000, d)).astype(np.float32)  # all positive: dominate every all-positive query
idx = sharded(x, np.linspace(0, n, world + 1).astype(int))
D, I = idx.search(q, k)
D0, I0 = oracle.flat_ip_search(q, x, k)
assert (I == I0).all() and (D == D0).all()
assert (I >= hot).all()
assert idx.local.stat("uncertified") == nq, "stats: uncertified %d wide %d exact %d" % (
    idx.local.stat("uncertified"), idx.local.stat("uncertified_wide"), idx.local.stat("exact_queries"))
report.append("skewed shards -> escalated (still uncertified after the wide level: %d)" % idx.local.stat("uncertified_wide"))

# ---- 5. Retriever.from_embeddings with more files than ranks + _search_sharded ----
from openmatch_b200.retriever import Retriever  # noqa: E402

tmp = [tempfile.mkdtemp() if rank == 0 else None]
dist.broadcast_object_list(tmp, src=0)
out = tmp[0]
n, d, nfiles = 5000, 64, 2 * world + 1
x = rng.integers(-5, 6, (n, d)).astype(np.float32)
qv = rng.integers(-5, 6, (11, d)).astype(np.float32)
cuts = np.linspace(0, n, nfiles + 1).astype(int)
if rank == 0:
    for f in range(nfiles):
        with open(os.path.join(out, "embeddings.corpus.rank.%d" % f), "wb") as fh:
            pickle.dump((x[cuts[f]:cuts[f + 1]], ["d%d" % i for i in range(cuts[f], cuts[f + 1])]), fh, protocol=4)
    for r in range(world):
        sl = slice(r * 11 // world, (r + 1) * 11 // world)
        with open(os.path.join(out, "embeddings.query.rank.%d" % r), "wb") as fh:
            pickle.dump((qv[sl], ["q%d" % i for i in range(sl.start, sl.stop)]), fh, protocol=4)
dist.barrier()
args = types.SimpleNamespace(device=torch.device("cuda"), fp16=False, bf16=False, per_device_eval_batch_size=16,
                             dataloader_num_workers=0, dataloader_pin_memory=False, output_dir=out, process_index=rank,
                             local_process_index=rank, world_size=world, use_gpu=True)
ret = Retriever.from_embeddings(torch.nn.Identity(), args)
assert ret.index.ntotal == len(ret.doc_lookup) > 0, "index rows and doc_lookup out of step (rank %d)" % rank
total = torch.tensor([ret.index.ntotal], device="cuda")
dist.all_reduce(total)
assert int(total.item()) == n
res = ret.search(topk=20)
if rank == 0:
    D0, I0 = oracle.flat_ip_search(qv, x, 20)
    for qi in range(11):
        got = res["q%d" % qi]
        want = ["d%d" % i for i in I0[qi]]
        # equal scores may order differently across shard boundaries by id string; compare as score-sorted multisets
        assert sorted(got.values(), reverse=True) == [float(s) for s in D0[qi]]
        assert set(got) == set(want) or sorted(got.values()) == sorted(float(s) for s in D0[qi])
report.append("Retriever.from_embeddings(%d files) + sharded search" % nfiles)

# ---- 6. cross-device negatives ----
g = torch.Generator().manual_seed(5)
allx = (torch.randn(world * 4, 64, generator=g) * 0.5).to(torch.bfloat16)
ally = (torch.randn(world * 32, 64, generator=g) * 0.5).to(torch.bfloat16)
lx = allx[rank * 4:(rank + 1) * 4].cuda().requires_grad_()
ly = ally[rank * 32:(rank + 1) * 32].cuda().requires_grad_()
loss = DistributedContrastiveLoss()(lx, ly)
loss.backward()
want, dx, dy, _ = oracle.contrastive_loss_fwd_bwd(allx.float().numpy(), ally.float().numpy())
assert abs(loss.item() - want * world) <= 1e-3 * max(1.0, abs(want * world)), (loss.item(), want * world)
gx = lx.grad.float().cpu().numpy() / world
ref = dx[rank * 4:(rank + 1) * 4]
assert np.linalg.norm(gx - ref) <= 1e-2 * np.linalg.norm(ref), "x-device grad mismatch (queries)"
gy = ly.grad.float().cpu().numpy() / world
refy = dy[rank * 32:(rank + 1) * 32]
assert np.linalg.norm(gy - refy) <= 1e-2 * np.linalg.norm(refy), "x-device grad mismatch (passages)"
report.append("DistributedContrastiveLoss")

# DRModel.forward(negatives_x_device): tiny BERT under autograd + gather + fused loss vs the oracle on gathered reps
from transformers import BertConfig, BertModel  # noqa: E402

from openmatch_b200.modeling import DRModel  # noqa: E402

torch.manual_seed(0)
lm = BertModel(BertConfig(vocab_size=300, hidden_size=64, num_hidden_layers=1, num_attention_heads=1, intermediate_size=128,
                          max_position_embeddings=64, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0),
               add_pooling_layer=False).cuda()
model = DRModel(lm, lm, tied=True, pooling="first", data_args=types.SimpleNamespace(train_n_passages=4),
                train_args=types.SimpleNamespace(negatives_x_device=True)).cuda().train()
gi = torch.Generator().manual_seed(100 + rank)
qi = torch.randint(5, 300, (3, 16), generator=gi).cuda()
pi = torch.randint(5, 300, (12, 24), generator=gi).cuda()
qb = {"input_ids": qi, "attention_mask": torch.ones_like(qi), "token_type_ids": torch.zeros_like(qi)}
pb = {"input_ids": pi, "attention_mask": torch.ones_like(pi), "token_type_ids": torch.zeros_like(pi)}
outm = model(qb, pb)
assert outm.q_reps.shape == (3 * world, 64) and outm.p_reps.shape == (12 * world, 64)
want, _, _, _ = oracle.contrastive_loss_fwd_bwd(outm.q_reps.detach().float().cpu().numpy(),
                                                outm.p_reps.detach().float().cpu().numpy())
assert abs(outm.loss.item() - want * world) <= 2e-3 * max(1.0, abs(want * world)), (outm.loss.item(), want, world)
outm.loss.backward()
gnorm = lm.encoder.layer[0].attention.self.query.weight.grad
assert gnorm is not None and torch.isfinite(gnorm).all() and gnorm.abs().sum() > 0
report.append("DRModel.forward negatives_x_device")

dist.barrier()
if rank == 0:
    print("DIST CHECK OK world=%d: %s" % (world, "; ".join(report)))
dist.destroy_process_group()
