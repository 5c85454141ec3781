"""CPU: which C entry each search and range search call of ``openmatch_b200.index`` takes, and what it passes, without a
GPU.  A recording fake library stands in for the eight search entries; every call records the entry's name, the
communicator, the query and output memkinds, ``k`` or the radii, ``id_offset`` and the filter it points to (the packed
bitmap words, the exclusion offsets and ids).  The table is pinned: an unfiltered call never takes a ``_filtered``
entry, a filter with every exclusion list empty still does, and the module helpers slice the global bitmap to the
shard and pick the single-shard or the sharded entry from the world size.

``python tests/test_search_routing_cpu.py`` prints the table."""
import ctypes
import os
import sys
import types

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmatch_b200 import index as om_index  # noqa: E402

NQ, D, NTOTAL = 3, 8, 100
KIND = {0: "host", 1: "device"}


def _read(ctype, ptr, n):
    return list((ctype * n).from_address(ptr)) if ptr and n else None


class _FakeLib:
    """The eight search entries, recording; ``om_index_range_search*`` write lims = 0, so there are no results to read."""

    def __init__(self):
        self.calls = []

    def _entry(self, name):
        def fn(*args):
            sharded, filtered, rng = "_sharded" in name, name.endswith("_filtered"), "range" in name
            body = args[2 if sharded else 1:-2 if filtered else -1]
            comm = args[1].value if sharded else None
            if rng:
                q, q_kind, nq, radius, lims, out_kind, id_offset = body
                arg = tuple(_read(ctypes.c_float, radius, nq) or ())
                ctypes.memset(lims, 0, (nq + 1) * 8)
            else:
                q, q_kind, nq, k, _D, _I, out_kind, id_offset = body
                arg = k
            filt = None
            if filtered:
                f = args[-2]._obj  # ctypes.byref(om_search_filter)
                off = _read(ctypes.c_int64, f.exclude_offsets, nq + 1)
                filt = (f.allow_words, _read(ctypes.c_int32, f.allow_bits, f.allow_words), off,
                        _read(ctypes.c_int64, f.exclude_ids, off[-1] if off else 0))
            self.calls.append((name, comm, KIND[q_kind], nq, arg, KIND[out_kind], id_offset, filt))
            return 0
        return fn

    def __getattr__(self, name):
        if name.startswith(("om_index_search", "om_index_range_search")):
            return self._entry(name)
        if name == "om_index_range_results":
            return lambda *a: 0
        if name == "om_index_ntotal":
            return lambda h: NTOTAL
        raise AttributeError(name)


def _fake_index():
    idx = om_index.FlatIPIndex.__new__(om_index.FlatIPIndex)
    idx._lib, idx._h, idx.d, idx.dtype = _FakeLib(), ctypes.c_void_p(1), D, torch.float32
    return idx


_ALLOW = np.zeros(130, bool)  # over global ids; a shard at id_offset 7 takes [7, 107)
_ALLOW[[0, 7, 8, 40, 106, 107, 129]] = True
FILTERS = {
    "none": (None, None),
    "bitmap": (_ALLOW, None),
    "exclusions": (None, [[7, 9], [], [8, 8, 200]]),
    "empty exclusions": (None, [[], [], []]),
}
RADII = [0.25, -1.0, 3.5]


def _calls():
    """(label, call(index, allow, exclude)) of the index's own calls, and of the module helpers"""
    q = torch.arange(NQ * D, dtype=torch.float32).view(NQ, D)
    comm = types.SimpleNamespace(_h=ctypes.c_void_p(2))

    def local(allow):
        return None if allow is None else allow[:NTOTAL]

    def outputs(k):
        return torch.empty(NQ, k), torch.empty(NQ, k, dtype=torch.int64)

    methods = [
        ("search_pinned", lambda ix, a, e: ix.search_pinned(q, 6, *outputs(6), id_offset=11)),
        ("search_sharded_pinned", lambda ix, a, e: ix.search_sharded_pinned(comm, q, 6, *outputs(6), 13)),
        ("search (numpy)", lambda ix, a, e: ix.search(q.numpy(), 2, id_offset=5)),
        ("search_device", lambda ix, a, e: ix.search_device(q, 5, 3, allow=local(a), exclude=e)),
        ("search_sharded_device", lambda ix, a, e: ix.search_sharded_device(comm, q, 5, 7, allow=local(a), exclude=e)),
        ("range_search_device", lambda ix, a, e: ix.range_search_device(q, RADII, 3, allow=local(a), exclude=e)),
        ("range_search_sharded_device",
         lambda ix, a, e: ix.range_search_sharded_device(comm, q, 0.5, 7, allow=local(a), exclude=e)),
    ]
    helpers = [
        ("sharded_search_device", lambda ix, a, e: om_index.sharded_search_device(ix, q, 4, 7, allow=a, exclude=e)),
        ("sharded_range_search_device",
         lambda ix, a, e: om_index.sharded_range_search_device(ix, q, RADII, 7, allow=a, exclude=e)),
    ]
    return methods, helpers


def _fake_world(monkeypatch, world):
    """No process group at world size 1; at 2, torch.distributed reports an initialised group of two ranks and
    ``comm_for`` hands out a fake communicator (handle 3)."""
    import torch.distributed as dist
    monkeypatch.setattr(om_index, "_stream", lambda: 0)
    if world > 1:
        monkeypatch.setattr(dist, "is_initialized", lambda: True)
        monkeypatch.setattr(dist, "get_world_size", lambda group=None: world)
        monkeypatch.setattr(om_index, "comm_for", lambda group=None: types.SimpleNamespace(_h=ctypes.c_void_p(3)))


def table(monkeypatch):
    rows = []
    methods, helpers = _calls()
    for world, calls in ((1, methods + helpers), (2, helpers)):
        _fake_world(monkeypatch, world)
        for label, call in calls:
            unfilterable = label in ("search_pinned", "search_sharded_pinned", "search (numpy)")
            for fname, (allow, exclude) in FILTERS.items():
                if unfilterable and fname != "none":
                    continue
                ix = _fake_index()
                try:
                    call(ix, allow, exclude)
                finally:
                    ix._h = None  # nothing to destroy
                for c in ix._lib.calls:
                    rows.append((world, label, fname) + c)
    return rows


# (world, call, filter, entry, comm, q_kind, nq, k or radii, out_kind, id_offset,
#  filter: (allow_words, bitmap words, exclusion offsets, excluded ids))
EXPECTED = [
    (1, 'search_pinned', 'none', 'om_index_search', None, 'host', 3, 6, 'host', 11, None),
    (1, 'search_sharded_pinned', 'none', 'om_index_search_sharded', 2, 'host', 3, 6, 'host', 13, None),
    (1, 'search (numpy)', 'none', 'om_index_search', None, 'host', 3, 2, 'host', 5, None),
    (1, 'search_device', 'none', 'om_index_search', None, 'device', 3, 5, 'device', 3, None),
    (1, 'search_device', 'bitmap', 'om_index_search_filtered', None, 'device', 3, 5, 'device', 3, (4, [385, 256, 0, 0], None, None)),
    (1, 'search_device', 'exclusions', 'om_index_search_filtered', None, 'device', 3, 5, 'device', 3, (0, None, [0, 2, 2, 5], [7, 9, 8, 8, 200])),
    (1, 'search_device', 'empty exclusions', 'om_index_search_filtered', None, 'device', 3, 5, 'device', 3, (0, None, [0, 0, 0, 0], None)),
    (1, 'search_sharded_device', 'none', 'om_index_search_sharded', 2, 'device', 3, 5, 'device', 7, None),
    (1, 'search_sharded_device', 'bitmap', 'om_index_search_sharded_filtered', 2, 'device', 3, 5, 'device', 7, (4, [385, 256, 0, 0], None, None)),
    (1, 'search_sharded_device', 'exclusions', 'om_index_search_sharded_filtered', 2, 'device', 3, 5, 'device', 7, (0, None, [0, 2, 2, 5], [7, 9, 8, 8, 200])),
    (1, 'search_sharded_device', 'empty exclusions', 'om_index_search_sharded_filtered', 2, 'device', 3, 5, 'device', 7, (0, None, [0, 0, 0, 0], None)),
    (1, 'range_search_device', 'none', 'om_index_range_search', None, 'device', 3, (0.25, -1.0, 3.5), 'host', 3, None),
    (1, 'range_search_device', 'bitmap', 'om_index_range_search_filtered', None, 'device', 3, (0.25, -1.0, 3.5), 'host', 3, (4, [385, 256, 0, 0], None, None)),
    (1, 'range_search_device', 'exclusions', 'om_index_range_search_filtered', None, 'device', 3, (0.25, -1.0, 3.5), 'host', 3, (0, None, [0, 2, 2, 5], [7, 9, 8, 8, 200])),
    (1, 'range_search_device', 'empty exclusions', 'om_index_range_search_filtered', None, 'device', 3, (0.25, -1.0, 3.5), 'host', 3, (0, None, [0, 0, 0, 0], None)),
    (1, 'range_search_sharded_device', 'none', 'om_index_range_search_sharded', 2, 'device', 3, (0.5, 0.5, 0.5), 'host', 7, None),
    (1, 'range_search_sharded_device', 'bitmap', 'om_index_range_search_sharded_filtered', 2, 'device', 3, (0.5, 0.5, 0.5), 'host', 7, (4, [385, 256, 0, 0], None, None)),
    (1, 'range_search_sharded_device', 'exclusions', 'om_index_range_search_sharded_filtered', 2, 'device', 3, (0.5, 0.5, 0.5), 'host', 7, (0, None, [0, 2, 2, 5], [7, 9, 8, 8, 200])),
    (1, 'range_search_sharded_device', 'empty exclusions', 'om_index_range_search_sharded_filtered', 2, 'device', 3, (0.5, 0.5, 0.5), 'host', 7, (0, None, [0, 0, 0, 0], None)),
    (1, 'sharded_search_device', 'none', 'om_index_search', None, 'device', 3, 4, 'device', 7, None),
    (1, 'sharded_search_device', 'bitmap', 'om_index_search_filtered', None, 'device', 3, 4, 'device', 7, (4, [3, 2, 0, 8], None, None)),
    (1, 'sharded_search_device', 'exclusions', 'om_index_search_filtered', None, 'device', 3, 4, 'device', 7, (0, None, [0, 2, 2, 5], [7, 9, 8, 8, 200])),
    (1, 'sharded_search_device', 'empty exclusions', 'om_index_search_filtered', None, 'device', 3, 4, 'device', 7, (0, None, [0, 0, 0, 0], None)),
    (1, 'sharded_range_search_device', 'none', 'om_index_range_search', None, 'device', 3, (0.25, -1.0, 3.5), 'host', 7, None),
    (1, 'sharded_range_search_device', 'bitmap', 'om_index_range_search_filtered', None, 'device', 3, (0.25, -1.0, 3.5), 'host', 7, (4, [3, 2, 0, 8], None, None)),
    (1, 'sharded_range_search_device', 'exclusions', 'om_index_range_search_filtered', None, 'device', 3, (0.25, -1.0, 3.5), 'host', 7, (0, None, [0, 2, 2, 5], [7, 9, 8, 8, 200])),
    (1, 'sharded_range_search_device', 'empty exclusions', 'om_index_range_search_filtered', None, 'device', 3, (0.25, -1.0, 3.5), 'host', 7, (0, None, [0, 0, 0, 0], None)),
    (2, 'sharded_search_device', 'none', 'om_index_search_sharded', 3, 'device', 3, 4, 'device', 7, None),
    (2, 'sharded_search_device', 'bitmap', 'om_index_search_sharded_filtered', 3, 'device', 3, 4, 'device', 7, (4, [3, 2, 0, 8], None, None)),
    (2, 'sharded_search_device', 'exclusions', 'om_index_search_sharded_filtered', 3, 'device', 3, 4, 'device', 7, (0, None, [0, 2, 2, 5], [7, 9, 8, 8, 200])),
    (2, 'sharded_search_device', 'empty exclusions', 'om_index_search_sharded_filtered', 3, 'device', 3, 4, 'device', 7, (0, None, [0, 0, 0, 0], None)),
    (2, 'sharded_range_search_device', 'none', 'om_index_range_search_sharded', 3, 'device', 3, (0.25, -1.0, 3.5), 'host', 7, None),
    (2, 'sharded_range_search_device', 'bitmap', 'om_index_range_search_sharded_filtered', 3, 'device', 3, (0.25, -1.0, 3.5), 'host', 7, (4, [3, 2, 0, 8], None, None)),
    (2, 'sharded_range_search_device', 'exclusions', 'om_index_range_search_sharded_filtered', 3, 'device', 3, (0.25, -1.0, 3.5), 'host', 7, (0, None, [0, 2, 2, 5], [7, 9, 8, 8, 200])),
    (2, 'sharded_range_search_device', 'empty exclusions', 'om_index_range_search_sharded_filtered', 3, 'device', 3, (0.25, -1.0, 3.5), 'host', 7, (0, None, [0, 0, 0, 0], None)),
]


def test_routing_table(monkeypatch):
    assert table(monkeypatch) == EXPECTED


if __name__ == "__main__":
    mp = pytest.MonkeyPatch()
    try:
        for row in table(mp):
            print("    %r," % (row,))
    finally:
        mp.undo()
