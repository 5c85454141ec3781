"""Oracle of the filtered range search: ``flat_ip_range_search`` (float64) restricted to the rows the bitmap allows and
the query does not exclude.  A filter only removes rows from each query's ordered list, so the (score desc, id asc)
order of what remains is the order of the eligible rows' own range search."""
from __future__ import annotations

import numpy as np

from index_range_oracle import flat_ip_range_search


def flat_ip_range_search_filtered(q: np.ndarray, x: np.ndarray, radius, allow=None, exclude=None, id_offset: int = 0):
    """q [nq, d], x [n, d], radius a number or [nq]; allow: bool [n] or None; exclude: ``nq`` lists of ids in the
    result id space (``id_offset`` + row; others ignored, duplicates allowed) or None -> (lims int64 [nq + 1], D
    float64, I int64 of ids ``id_offset`` + row)."""
    lims, D, I = flat_ip_range_search(q, x, radius)
    nq = lims.size - 1
    allow = np.ones(np.asarray(x).shape[0], bool) if allow is None else np.asarray(allow, bool)
    out_l = np.zeros(nq + 1, np.int64)
    Ds, Is = [], []
    for i in range(nq):
        rows = I[lims[i]:lims[i + 1]]
        keep = allow[rows]
        if exclude is not None and len(exclude[i]):
            keep &= ~np.isin(rows + id_offset, np.asarray(exclude[i], np.int64))
        Ds.append(D[lims[i]:lims[i + 1]][keep])
        Is.append(rows[keep] + id_offset)
        out_l[i + 1] = out_l[i] + int(keep.sum())
    D = np.concatenate(Ds) if Ds else np.zeros(0)
    I = np.concatenate(Is).astype(np.int64) if Is else np.zeros(0, np.int64)
    return out_l, D, I
