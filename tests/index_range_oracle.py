"""Oracle of the range search: ``IndexFlatIP.range_search`` restated in float64 (faiss keeps, for inner products, every
row whose score is strictly above the radius).  Scores are exact float64 inner products of the fp32 inputs; the order is
(score desc, id asc).  On integer-valued data of small magnitude every fp32 sum is exact, so the library must match it
as a set; elsewhere the GPU tests compare within the re-score error bound.

It lives with the tests, beside ``index_i8_oracle.py``, rather than in ``oracle/flat_index.py``: the ``oracle`` package is
the restatement pinned against golden vectors of the reference (``tests/test_oracle_pinning.py``) and is kept as it
stands, and faiss's range search has no counterpart in the reference to pin it against.  ``RangeFlatIPIndex`` extends the
oracle's ``FlatIPIndex`` duck type with ``range_search`` without changing it."""
from __future__ import annotations

import numpy as np

import oracle


def flat_ip_range_search(q: np.ndarray, x: np.ndarray, radius, block_rows: int = 1 << 16):
    """q [nq, d], x [n, d], radius a number or [nq] -> (lims int64 [nq + 1], D float64, I int64)."""
    q = np.asarray(q, dtype=np.float32).astype(np.float64)
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    nq = q.shape[0]
    rho = np.broadcast_to(np.asarray(radius, dtype=np.float32).astype(np.float64), (nq,))
    Ds, Is = [[] for _ in range(nq)], [[] for _ in range(nq)]
    for lo in range(0, x.shape[0], block_rows):
        s = q @ x[lo:lo + block_rows].T
        for i in range(nq):
            keep = np.flatnonzero(s[i] > rho[i])
            Ds[i].append(s[i, keep])
            Is[i].append(keep + lo)
    lims = np.zeros(nq + 1, np.int64)
    D, I = [], []
    for i in range(nq):
        d = np.concatenate(Ds[i]) if Ds[i] else np.zeros(0)
        ids = np.concatenate(Is[i]).astype(np.int64) if Is[i] else np.zeros(0, np.int64)
        order = np.lexsort((ids, -d))
        D.append(d[order])
        I.append(ids[order])
        lims[i + 1] = lims[i] + order.size
    return lims, np.concatenate(D) if D else np.zeros(0), np.concatenate(I) if I else np.zeros(0, np.int64)


class RangeFlatIPIndex(oracle.FlatIPIndex):
    """The oracle's ``faiss.IndexFlatIP`` duck type with ``range_search``."""

    def range_search(self, q, radius):
        x = np.concatenate(self._chunks) if self._chunks else np.zeros((0, self.d), np.float32)
        return flat_ip_range_search(q, x, radius)
