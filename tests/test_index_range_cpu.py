"""CPU: the range search's oracle (strictness, order), the radius argument of ``FlatIPIndex.range_search`` and
``Retriever.range_search`` driven through the oracle index."""
import types

import numpy as np
import pytest
import torch

from index_range_oracle import RangeFlatIPIndex, flat_ip_range_search
from openmatch_b200.index import range_radius
from openmatch_b200.retriever.dense_retriever import Retriever


def test_oracle_is_strict_and_ordered():
    x = np.array([[1, 0], [2, 0], [1, 0], [0, 1], [3, 0], [-1, 0]], np.float32)
    q = np.array([[1, 0], [0, 2]], np.float32)
    lims, D, I = flat_ip_range_search(q, x, np.array([1.0, -0.5], np.float32))
    assert lims.tolist() == [0, 2, 8]
    assert I[:2].tolist() == [4, 1] and D[:2].tolist() == [3.0, 2.0]  # rows 0 and 2 score 1 == radius: excluded
    # row 3 (score 2), then the rows of score 0 > -0.5 by ascending id
    assert I[2:].tolist() == [3, 0, 1, 2, 4, 5] and D[2:].tolist() == [2.0, 0.0, 0.0, 0.0, 0.0, 0.0]
    assert flat_ip_range_search(q, x, -np.inf)[0].tolist() == [0, 6, 12]
    assert flat_ip_range_search(q, x, np.inf)[0].tolist() == [0, 0, 0]
    assert flat_ip_range_search(q[:0], x, 0.0)[0].tolist() == [0]
    assert flat_ip_range_search(q, x[:0], 0.0)[0].tolist() == [0, 0, 0]


def test_oracle_matches_a_thresholded_top_k():
    rng = np.random.default_rng(3)
    x = rng.integers(-4, 5, size=(300, 24)).astype(np.float32)
    q = rng.integers(-4, 5, size=(9, 24)).astype(np.float32)
    import oracle
    Dk, Ik = oracle.flat_ip_search(q, x, 300)
    rho = Dk[:, 40]
    lims, D, I = flat_ip_range_search(q, x, rho)
    for i in range(9):
        n = int((Dk[i] > rho[i]).sum())
        assert lims[i + 1] - lims[i] == n
        assert I[lims[i]:lims[i + 1]].tolist() == Ik[i, :n].tolist(), "the prefix of the top-k, tie order included"


def test_range_radius_broadcasts_and_checks_shape():
    assert range_radius(0.5, 3).tolist() == [0.5, 0.5, 0.5]
    assert range_radius(np.float32(2), 2).dtype == torch.float32
    assert range_radius([1, 2], 2).tolist() == [1.0, 2.0]
    assert range_radius(np.array([1.5, 2.5], np.float64), 2).dtype == torch.float32
    assert range_radius(torch.tensor(3.0), 2).tolist() == [3.0, 3.0]
    assert range_radius(np.array([-np.inf, np.inf]), 2).tolist() == [-np.inf, np.inf]
    assert range_radius(0.0, 0).numel() == 0
    with pytest.raises(ValueError, match=r"one value per query \(\[3\]\)"):
        range_radius([1.0, 2.0], 3)
    with pytest.raises(ValueError, match="one value per query"):
        range_radius(np.zeros((2, 1), np.float32), 2)
    with pytest.raises(TypeError):
        range_radius("0.5", 1)


def _retriever(x, q, docs, queries):
    idx = RangeFlatIPIndex(x.shape[1])
    idx.add(x)
    r = Retriever.__new__(Retriever)
    r.index = idx
    r.args = types.SimpleNamespace(world_size=1)
    r.doc_lookup = list(docs)
    r.query_lookup = list(queries)
    r._load_queries = lambda: q
    return r


def test_retriever_range_search_against_the_oracle():
    rng = np.random.default_rng(7)
    x = rng.integers(-3, 4, size=(50, 8)).astype(np.float32)
    q = rng.integers(-3, 4, size=(5, 8)).astype(np.float32)
    docs = ["doc%03d" % i for i in range(50)]
    queries = ["q%d" % i for i in range(5)]
    r = _retriever(x, q, docs, queries)
    radius = np.array([0, 5, -100, 1000, 3], np.float32)
    out = r.range_search(radius)
    lims, D, I = flat_ip_range_search(q, x, radius)
    assert list(out) == queries
    for i, qid in enumerate(queries):
        assert list(out[qid]) == [docs[j] for j in I[lims[i]:lims[i + 1]]], "rank order"
        assert list(out[qid].values()) == D[lims[i]:lims[i + 1]].tolist()
    assert len(out["q2"]) == 50 and out["q3"] == {}
    # a single radius is broadcast over the queries
    assert r.range_search(5.0)["q1"] == out["q1"]
    r.index = None
    with pytest.raises(ValueError, match="not initialized"):
        r.range_search(0.0)


def _merge_places(runs, nq):
    """The placement rule of the sharded range search's merge (range_merge_parts_kernel), restated: entry j of part p's
    run for query q goes to glims[q] + j + the entries of the other parts' runs for q that precede it (higher score, or
    equal score and lower id, or equal id and lower part), each count a binary search of a sorted run.  runs[p] =
    (lims, D, I) of part p."""
    W = len(runs)
    glims = np.zeros(nq + 1, np.int64)
    glims[1:] = np.cumsum(sum(np.diff(r[0]) for r in runs))
    D = np.full(glims[-1], np.nan, np.float32)
    I = np.full(glims[-1], -1, np.int64)
    filled = np.zeros(glims[-1], bool)
    for p, (lp, Dp, Ip) in enumerate(runs):
        for q in range(nq):
            for e in range(lp[q], lp[q + 1]):
                s, i = Dp[e], Ip[e]
                pos = glims[q] + (e - lp[q])
                for p2 in range(W):
                    if p2 == p:
                        continue
                    l2, D2, I2 = runs[p2]
                    a, b = l2[q], l2[q + 1]
                    while a < b:
                        mid = (a + b) // 2
                        if D2[mid] > s or (D2[mid] == s and (I2[mid] < i or (I2[mid] == i and p2 < p))):
                            a = mid + 1
                        else:
                            b = mid
                    pos += a - l2[q]
                assert not filled[pos], "two entries placed at %d" % pos
                filled[pos] = True
                D[pos], I[pos] = s, i
    assert filled.all()
    return glims, D, I


def test_merge_placement_rule_is_the_global_sort():
    rng = np.random.default_rng(13)
    nq, W = 6, 3
    x = rng.integers(-3, 4, size=(90, 4)).astype(np.float32)  # integer scores: many ties across parts
    q = rng.integers(-3, 4, size=(nq, 4)).astype(np.float32)
    radius = np.array([-np.inf, 0, 2, 5, 100, -3], np.float32)
    whole = flat_ip_range_search(q, x, radius)
    for bounds, offsets in (([0, 30, 60, 90], [0, 30, 60]), ([0, 0, 45, 90], [0, 0, 45]),  # an empty part
                            ([0, 30, 60, 90], [60, 30, 0]),  # id offsets that fall with the part
                            ([0, 90, 90, 90], [0, 90, 90])):  # one part holds every result
        runs = []
        for p in range(W):
            lims, D, I = flat_ip_range_search(q, x[bounds[p]:bounds[p + 1]], radius)
            runs.append((lims, D.astype(np.float32), I + offsets[p]))
        glims, D, I = _merge_places(runs, nq)
        assert glims.tolist() == whole[0].tolist()
        for i in range(nq):  # the single index's result with its ids mapped to the parts' ids, re-sorted by (score, id)
            a, b = whole[0][i], whole[0][i + 1]
            part = np.searchsorted(bounds, whole[2][a:b], side="right") - 1
            part = np.minimum(part, W - 1)
            ids = whole[2][a:b] - np.asarray(bounds)[part] + np.asarray(offsets)[part]
            o = np.lexsort((ids, -whole[1][a:b]))
            assert D[a:b].tolist() == whole[1][a:b][o].astype(np.float32).tolist()
            assert I[a:b].tolist() == ids[o].tolist()
    # equal ids in two parts (overlapping id offsets): the lower part first, still one place each
    r = (np.array([0, 2]), np.array([3.0, 1.0], np.float32), np.array([7, 8]))
    glims, D, I = _merge_places([r, r], 1)
    assert I.tolist() == [7, 7, 8, 8] and D.tolist() == [3.0, 3.0, 1.0, 1.0]
