"""Oracle: exact (brute-force) maximum-inner-product search, i.e. what ``faiss.IndexFlatIP`` computes for
the reference at ``src/openmatch/retriever/dense_retriever.py:38-41`` (construction), ``:105`` (add),
``:133-137`` (reset) and ``:180`` (``D, I = self.index.search(encoded, topk)``).

faiss is NOT in /root/reference (un-vendored, undeclared in setup.py:23-27, README.md:17-19 says "install
faiss-cpu or faiss-gpu") and is not installed; no version is pinned.  Restated from its published
behaviour (faiss ``IndexFlat.cpp`` / ``utils/distances.cpp`` ``knn_inner_product``):
  * scores are fp32 inner products ``<q, x_i>`` (blocked SGEMM on CPU);
  * each result row holds the k largest scores in descending order, labels are int64 insertion rows;
  * when fewer than k vectors exist the tail is padded with label -1 and score ``lowest(float)`` = -FLT_MAX
    (``CMin<float,int64>::neutral()``);
  * the order among exactly-equal scores is implementation-defined in faiss (heap / reservoir order);
    this oracle, and the CUDA path, fix it to (score descending, row ascending).
Parity for this step is therefore "unpinned" against faiss itself; it is anchored on the reference's call
sites and on exact-arithmetic (integer-valued) inputs where any correct fp32 implementation agrees.
"""
from __future__ import annotations

import numpy as np

NEG_FILL = np.float32(-3.4028234663852886e38)  # std::numeric_limits<float>::lowest()


def _topk_row_exact(s: np.ndarray, kk: int) -> np.ndarray:
    """Column indices of the kk largest entries of one row, ordered by (score desc, column asc)."""
    n = s.shape[0]
    if kk < n:
        part = np.argpartition(-s, kk - 1)[:kk]
        kth = s[part].min()
        gt = np.flatnonzero(s > kth)
        eq = np.flatnonzero(s == kth)[: kk - gt.size]  # ascending column = ascending row id
        idx = np.concatenate([gt, eq])
    else:
        idx = np.arange(n)
    return idx[np.lexsort((idx, -s[idx].astype(np.float64)))]


def _topk_rows(scores: np.ndarray, k: int, row_offset: int = 0):
    """Top-k of every row of ``scores`` ordered by (score desc, column asc).  Returns (D f32, I i64).

    Fast path: multi-threaded ``torch.topk`` for the selection, then a stable re-sort for the tie order; rows
    whose k-th score is tied with an unselected column fall back to the exact per-row routine."""
    import torch
    nq, n = scores.shape
    kk = min(k, n)
    D = np.full((nq, k), NEG_FILL, dtype=np.float32)
    I = np.full((nq, k), -1, dtype=np.int64)
    if kk == 0:
        return D, I
    st = torch.from_numpy(np.ascontiguousarray(scores))
    vals, idx = torch.topk(st, kk, dim=1, sorted=True)
    vals, idx = vals.numpy(), idx.numpy()
    by_col = np.argsort(idx, axis=1, kind="stable")
    idx, vals = np.take_along_axis(idx, by_col, 1), np.take_along_axis(vals, by_col, 1)
    by_score = np.argsort(-vals.astype(np.float64), axis=1, kind="stable")
    idx, vals = np.take_along_axis(idx, by_score, 1), np.take_along_axis(vals, by_score, 1)
    if kk < n:
        n_ge = (st >= torch.from_numpy(vals[:, -1:].copy())).sum(dim=1).numpy()
        for r in np.flatnonzero(n_ge > kk):  # boundary ties: which equal-score columns survive matters
            sel = _topk_row_exact(scores[r], kk)
            idx[r], vals[r] = sel, scores[r][sel]
    D[:, :kk] = vals
    I[:, :kk] = idx + row_offset
    return D, I


def flat_ip_search(q: np.ndarray, x: np.ndarray, k: int, block_rows: int = 262144):
    """``IndexFlatIP.search``: q f32 [nq, d], x f32 [n, d] -> (D f32 [nq, k], I i64 [nq, k]).

    The corpus is scanned in row blocks (like faiss's blocked SGEMM) and per-block top-k are merged, so
    memory stays bounded for million-row slices; the result is independent of ``block_rows``.
    """
    q = np.ascontiguousarray(q, dtype=np.float32)
    x = np.ascontiguousarray(x, dtype=np.float32)
    nq = q.shape[0]
    n = x.shape[0]
    if n == 0 or nq == 0:
        return (np.full((nq, k), NEG_FILL, np.float32), np.full((nq, k), -1, np.int64))
    parts = []
    for lo in range(0, n, block_rows):
        hi = min(n, lo + block_rows)
        s = q @ x[lo:hi].T  # fp32 SGEMM
        parts.append(_topk_rows(s, k, row_offset=lo))
    if len(parts) == 1:
        return parts[0]
    return merge_topk(parts, k)


def merge_topk(parts, k: int):
    """Merge per-shard (D, I) lists into the global top-k by (score desc, id asc); -1 labels are padding.

    This is the exchange step of the sharded search (the role faiss ``IndexShards`` plays behind
    ``index_cpu_to_gpu_multiple(shard=True)``, dense_retriever.py:43-58).
    """
    D = np.concatenate([p[0] for p in parts], axis=1)
    I = np.concatenate([p[1] for p in parts], axis=1)
    nq = D.shape[0]
    outD = np.full((nq, k), NEG_FILL, np.float32)
    outI = np.full((nq, k), -1, np.int64)
    for r in range(nq):
        valid = np.flatnonzero(I[r] >= 0)
        order = np.lexsort((I[r, valid], -D[r, valid].astype(np.float64)))[:k]
        sel = valid[order]
        outD[r, : sel.size] = D[r, sel]
        outI[r, : sel.size] = I[r, sel]
    return outD, outI


class FlatIPIndex:
    """Duck-type of ``faiss.IndexFlatIP`` (the five members the reference touches)."""

    def __init__(self, d: int):
        self.d = int(d)
        self._chunks = []
        self.ntotal = 0

    def add(self, x):
        x = np.ascontiguousarray(x, dtype=np.float32)
        assert x.ndim == 2 and x.shape[1] == self.d
        self._chunks.append(x.copy())
        self.ntotal += x.shape[0]

    def reset(self):
        self._chunks = []
        self.ntotal = 0

    def search(self, q, k: int):
        x = np.concatenate(self._chunks) if self._chunks else np.zeros((0, self.d), np.float32)
        return flat_ip_search(q, x, k)


def merge_retrieval_results_by_score(results, topk: int = 100):
    """Restatement of ``src/openmatch/utils.py:215-229``: union per query id (first-seen score wins for a
    duplicated doc id), stable sort by score descending, keep ``topk``."""
    merged = {}
    for result in results:
        for qid, docs in result.items():
            slot = merged.setdefault(qid, {})
            for doc_id, score in docs.items():
                if doc_id not in slot:
                    slot[doc_id] = score
    out = {}
    for qid, docs in merged.items():
        ranked = sorted(docs.items(), key=lambda kv: kv[1], reverse=True)[:topk]
        out[qid] = dict(ranked)
    return out
