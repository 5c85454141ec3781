"""CPU: the filtered range search without a GPU: the filter-restricted oracle, the routing of ``FlatIPIndex.range_search``
(an unfiltered call never takes a ``_filtered`` entry, a filtered one passes the packed filter) and
``Retriever.range_search(allowed_docs=, exclude=)`` driven through the oracle index."""
import ctypes
import types

import numpy as np
import pytest
import torch

from index_range_filter_oracle import flat_ip_range_search_filtered
from index_range_oracle import RangeFlatIPIndex, flat_ip_range_search
from openmatch_b200 import index as om_index
from openmatch_b200.retriever.dense_retriever import Retriever


def _data(seed, n=300, d=16, nq=7):
    rng = np.random.default_rng(seed)
    return (rng.integers(-4, 5, size=(n, d)).astype(np.float32), rng.integers(-4, 5, size=(nq, d)).astype(np.float32),
            rng)


def test_oracle_bitmap_is_the_sub_index_with_ids_mapped_back():
    x, q, rng = _data(1)
    allow = rng.random(x.shape[0]) < 0.3
    rho = np.array([-100, 0, 3, 5, 8, 1000, -2], np.float32)
    lims, D, I = flat_ip_range_search_filtered(q, x, rho, allow=allow)
    rows = np.flatnonzero(allow)
    l0, D0, I0 = flat_ip_range_search(q, x[rows], rho)
    assert lims.tolist() == l0.tolist()
    assert I.tolist() == rows[I0].tolist(), "order, ties by ascending id, survives the id mapping"
    np.testing.assert_array_equal(D, D0)
    assert lims[1] - lims[0] == allow.sum(), "radius -100: every allowed row"
    none = flat_ip_range_search_filtered(q, x, rho, allow=np.zeros(x.shape[0], bool))
    assert none[0].tolist() == [0] * 8 and none[1].size == 0


def test_oracle_exclusions_duplicates_offsets_and_other_shards():
    x, q, _ = _data(2, nq=3)
    off = 1000
    l0, D0, I0 = flat_ip_range_search(q, x, 0.0)
    first = [int(I0[l0[i]]) + off for i in range(3)]
    excl = [[first[0], first[0], 5, off + 10 ** 6], [], [first[2], off + x.shape[0]]]  # dups, ids outside the shard
    lims, D, I = flat_ip_range_search_filtered(q, x, 0.0, exclude=excl, id_offset=off)
    for i in range(3):
        want = [int(r) + off for r in I0[l0[i]:l0[i + 1]] if int(r) + off not in excl[i]]
        assert I[lims[i]:lims[i + 1]].tolist() == want
    assert lims[2] - lims[1] == l0[2] - l0[1], "no exclusions: the unfiltered list"
    assert lims[1] - lims[0] == l0[1] - l0[0] - 1, "a duplicated id drops one row; ids outside the shard none"


def test_oracle_prefix_is_the_filtered_top_k():
    import oracle
    x, q, rng = _data(3)
    allow = rng.random(x.shape[0]) < 0.5
    rows = np.flatnonzero(allow)
    Dk, Ik = oracle.flat_ip_search(q, x[rows], rows.size)
    rho = Dk[:, 20]
    lims, _, I = flat_ip_range_search_filtered(q, x, rho, allow=allow)
    for i in range(q.shape[0]):
        n = int((Dk[i] > rho[i]).sum())
        assert I[lims[i]:lims[i + 1]].tolist() == rows[Ik[i, :n]].tolist()


class _FakeLib:
    """Records which range search entry a FlatIPIndex call takes, and the filter it passes; writes lims = 0."""

    def __init__(self):
        self.calls = []

    def _entry(self, name):
        def fn(*args):
            filt = None
            if name.endswith("_filtered"):
                filt = args[-2]._obj  # ctypes.byref(om_search_filter)
                filt = (filt.allow_bits, filt.allow_words, filt.exclude_offsets, filt.exclude_ids)
            nq = args[3] if "sharded" not in name else args[4]
            lims_ptr = args[5] if "sharded" not in name else args[6]
            ctypes.memset(lims_ptr, 0, (nq + 1) * 8)
            self.calls.append((name, filt))
            return 0
        return fn

    def __getattr__(self, name):
        if name.startswith("om_index_range_search"):
            return self._entry(name)
        if name == "om_index_range_results":
            return lambda *a: 0
        if name == "om_index_ntotal":
            return lambda h: 100
        raise AttributeError(name)


@pytest.fixture
def fake_index(monkeypatch):
    monkeypatch.setattr(om_index, "_stream", lambda: 0)
    idx = om_index.FlatIPIndex.__new__(om_index.FlatIPIndex)
    idx._lib, idx._h, idx.d, idx.dtype = _FakeLib(), ctypes.c_void_p(1), 8, torch.float32
    yield idx
    idx._h = None


def test_unfiltered_calls_never_take_a_filtered_entry(fake_index):
    q = torch.zeros(3, 8)
    comm = types.SimpleNamespace(_h=ctypes.c_void_p(2))
    fake_index.range_search_device(q, 0.5)
    fake_index.range_search_sharded_device(comm, q, 0.5, 7)
    fake_index.range_search_device(q, 0.5, allow=None, exclude=None)
    assert [c[0] for c in fake_index._lib.calls] == ["om_index_range_search", "om_index_range_search_sharded",
                                                     "om_index_range_search"]


def test_filtered_calls_pass_the_packed_filter(fake_index):
    q = torch.zeros(3, 8)
    comm = types.SimpleNamespace(_h=ctypes.c_void_p(2))
    allow = np.zeros(100, bool)
    allow[[0, 33, 99]] = True
    lims, D, I = fake_index.range_search_device(q, [0.0, 1.0, 2.0], allow=allow)
    name, (bits, words, off, ids) = fake_index._lib.calls[-1]
    assert name == "om_index_range_search_filtered" and bits and words == 4 and off is None and ids is None
    assert lims.tolist() == [0, 0, 0, 0] and D.numel() == I.numel() == 0
    fake_index.range_search_sharded_device(comm, q, 0.5, 7, exclude=[[7], [], [8, 8]])
    name, (bits, words, off, ids) = fake_index._lib.calls[-1]
    assert name == "om_index_range_search_sharded_filtered" and bits is None and off and ids
    # exclusions that are all empty still take the filtered entry (a null id pointer, offsets given)
    fake_index.range_search_device(q, 0.5, exclude=[[], [], []])
    name, (bits, words, off, ids) = fake_index._lib.calls[-1]
    assert name == "om_index_range_search_filtered" and off and ids is None


def test_filter_argument_errors_are_raised_before_the_library(fake_index):
    q = torch.zeros(2, 8)
    with pytest.raises(ValueError, match="entries"):
        fake_index.range_search_device(q, 0.0, allow=np.ones(99, bool))
    with pytest.raises(ValueError, match="packed words"):
        fake_index.range_search_device(q, 0.0, allow=torch.zeros(3, dtype=torch.int32))
    with pytest.raises(ValueError, match="3 id lists for 2 queries"):
        fake_index.range_search_device(q, 0.0, exclude=[[1], [2], [3]])
    with pytest.raises(ValueError, match="one value per query"):
        fake_index.range_search_device(q, [1.0, 2.0, 3.0], allow=np.ones(100, bool))
    assert fake_index._lib.calls == []


class _FilteredOracleIndex(RangeFlatIPIndex):
    """The oracle index with the filter arguments of FlatIPIndex.range_search."""

    def range_search(self, q, radius, allow=None, exclude=None):
        x = np.concatenate(self._chunks) if self._chunks else np.zeros((0, self.d), np.float32)
        return flat_ip_range_search_filtered(q, x, radius, allow=allow, exclude=exclude)


def _retriever(x, q, docs, queries):
    idx = _FilteredOracleIndex(x.shape[1])
    idx.add(x)
    r = Retriever.__new__(Retriever)
    r.index = idx
    r.args = types.SimpleNamespace(world_size=1)
    r.doc_lookup = list(docs)
    r.query_lookup = list(queries)
    r._load_queries = lambda: q
    return r


def test_retriever_filtered_range_search_against_the_oracle():
    x, q, rng = _data(7, n=60, d=8, nq=4)
    docs = ["doc%03d" % i for i in range(60)]
    queries = ["q%d" % i for i in range(4)]
    r = _retriever(x, q, docs, queries)
    radius = np.array([0, 2, -100, 1000], np.float32)
    allowed = [docs[i] for i in range(0, 60, 3)] + ["not-a-doc"]
    exclude = {"q0": ["doc003", "doc003", "unknown"], "q2": [docs[i] for i in range(0, 30, 3)]}
    out = r.range_search(radius, allowed_docs=allowed, exclude=exclude)
    allow = np.zeros(60, bool)
    allow[::3] = True
    excl = [[3], [], list(range(0, 30, 3)), []]
    lims, D, I = flat_ip_range_search_filtered(q, x, radius, allow=allow, exclude=excl)
    assert list(out) == queries
    for i, qid in enumerate(queries):
        assert list(out[qid]) == [docs[j] for j in I[lims[i]:lims[i + 1]]], "rank order"
        assert list(out[qid].values()) == D[lims[i]:lims[i + 1]].tolist()
    assert len(out["q2"]) == 10 and "doc003" not in out["q0"] and out["q3"] == {}
    # no filter: the unfiltered range search
    assert r.range_search(radius) == r.range_search(radius, allowed_docs=None, exclude=None)
    assert len(r.range_search(radius)["q2"]) == 60
