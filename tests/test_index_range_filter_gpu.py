"""GPU: filtered range search (``om_index_range_search_filtered``, ``FlatIPIndex.range_search(..., allow=, exclude=)``).

Contract under test: for query i the result is every row that the bitmap allows and the query does not exclude, and
whose fp32 score is strictly greater than radius[i], ordered by (score desc, id asc).  So lims, D and I must be bitwise
the unfiltered range search of an index built from the eligible rows only, with ids mapped back, on every storage; the
first j results of a query are ``search(q, j, allow=, exclude=)``'s for every j <= min(count, 4096).  Exclusions are
checked against the unfiltered range result with the excluded ids removed; integer data against a float64 oracle."""
import ctypes
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from index_range_filter_oracle import flat_ip_range_search_filtered

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.float32, torch.float16, torch.int8]
IDS = ["f32", "f16", "i8"]


@pytest.fixture(scope="module")
def om():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import index as om_index
    return om_index


def _same(a, b, what):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = b.cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
    assert a.shape == b.shape, "%s: shape %s vs %s" % (what, a.shape, b.shape)
    if a.dtype.kind == "f":
        np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32), err_msg=what)
    else:
        np.testing.assert_array_equal(a, b, err_msg=what)


def _same3(got, want, what):
    for a, b, name in zip(got, want, ("lims", "D", "I")):
        _same(a, b, "%s: %s" % (what, name))


def _index(om, x, dtype, **params):
    idx = om.FlatIPIndex(x.shape[1], dtype=dtype)
    if x.shape[0]:
        idx.add(torch.from_numpy(x).cuda())
    for name, v in params.items():
        idx.set_param(name, v)
    return idx


def _data(seed, n, d, nq):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((n, d), dtype=np.float32), rng.standard_normal((nq, d), dtype=np.float32), rng


def _sub_range(om, x, eligible, q, rho, dtype, **params):
    """Unfiltered range search of an index of x[eligible] only, ids mapped back to rows of x."""
    rows = np.flatnonzero(eligible)
    lims, D, I = _index(om, x[rows], dtype, **params).range_search(q, rho)
    return lims, D, rows[I] if I.size else I


def _sub_radii(om, x, eligible, q, kth, dtype):
    """per query the kth score of the sub-index of the eligible rows (its last score when it holds fewer)"""
    rows = np.flatnonzero(eligible)
    if rows.size == 0:
        return np.zeros(q.shape[0], np.float32)
    k = min(kth, rows.size)
    D, _ = _index(om, x[rows], dtype).search(q, k)
    return D[:, k - 1].astype(np.float32)


def _minus(lims, D, I, excl, id_offset=0):
    """the range result with each query's excluded ids removed"""
    out_l, Ds, Is = [0], [], []
    for i in range(lims.size - 1):
        d, ids = D[lims[i]:lims[i + 1]], I[lims[i]:lims[i + 1]]
        keep = ~np.isin(ids, np.asarray(excl[i], np.int64))
        Ds.append(d[keep])
        Is.append(ids[keep])
        out_l.append(out_l[-1] + int(keep.sum()))
    return np.array(out_l, np.int64), np.concatenate(Ds), np.concatenate(Is)


def _bitmaps(n, rng):
    out = {"all": np.ones(n, bool), "none": np.zeros(n, bool), "50%": rng.random(n) < 0.5, "1%": rng.random(n) < 0.01}
    s = np.zeros(n, bool)
    s[n // 3:n // 3 + n // 100] = True
    out["1% range"] = s
    s = np.zeros(n, bool)
    s[:n // 5] = True
    out["sub-collection at the start"] = s
    return out


# ---------------------------------------------------------------------------------------------------------------------
# bitmap: bitwise the sub-index
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("nq", [1, 64, 129, 1500])
def test_bitmap_equals_sub_index(om, dtype, nq):
    n = 40000
    x, q, rng = _data(nq * 3 + 1, n, 128, nq)
    idx = _index(om, x, dtype)
    for name, allow in _bitmaps(n, rng).items():
        for kth in (10, 1000):
            rho = _sub_radii(om, x, allow, q, kth, dtype)
            got = idx.range_search(q, rho, allow=allow)
            want = _sub_range(om, x, allow, q, rho, dtype)
            _same3(got, want, "%s nq=%d %s kth=%d" % (dtype, nq, name, kth))
            if name == "none":
                assert not got[0].any(), "allow-none: lims all zero"
            if name == "all":
                _same3(got, idx.range_search(q, rho), "allow-all vs unfiltered")


# ---------------------------------------------------------------------------------------------------------------------
# exclusions
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("with_bitmap", [False, True], ids=["excl", "excl+bitmap"])
def test_exclusions_from_the_queries_own_results(om, dtype, with_bitmap):
    n, nq, off = 30000, 150, 5000
    x, q, rng = _data(31 + with_bitmap, n, 96, nq)
    idx = _index(om, x, dtype)
    allow = rng.random(n) < 0.5 if with_bitmap else None
    rho = _sub_radii(om, x, allow if with_bitmap else np.ones(n, bool), q, 600, dtype)
    lims, D, I = idx.range_search(q, rho, id_offset=off, allow=allow)
    excl = []
    for i in range(nq):
        own = I[lims[i]:lims[i + 1]]
        e = list(rng.choice(own, min(120, own.size), replace=False)) if own.size else []
        e += e[:4]  # duplicates
        e += [off - 1, 3, off + n, off + n + 12345]  # ids outside the shard
        excl.append(e[:128])
    got = idx.range_search(q, rho, id_offset=off, allow=allow, exclude=excl)
    _same3(got, _minus(lims, D, I, excl), "%s bitmap=%s: minus the excluded ids" % (dtype, with_bitmap))
    # the same exclusions given as one CSR pair
    offs = torch.tensor(np.concatenate([[0], np.cumsum([len(e) for e in excl])]), dtype=torch.int64)
    ids = torch.tensor([v for e in excl for v in e], dtype=torch.int64)
    _same3(idx.range_search(q, rho, id_offset=off, allow=allow, exclude=(offs, ids)), got, "CSR pair")


# ---------------------------------------------------------------------------------------------------------------------
# prefix rule
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_prefix_rule_against_filtered_search(om, dtype):
    n, nq = 60000, 40
    x, q, rng = _data(41, n, 128, nq)
    idx = _index(om, x, dtype)
    allow = rng.random(n) < 0.3
    D4, _ = idx.search(q, 4096, allow=allow)
    ks = np.array([1, 10, 700, 4096, 3000])[np.arange(nq) % 5]
    rho = D4[np.arange(nq), ks - 1].astype(np.float32)
    rho[7] = D4[7, -1] - 1.0  # more than 4096 results: the prefix is the whole top-4096
    excl = [list(rng.choice(n, 30, replace=False)) for _ in range(nq)]
    for exclude in (None, excl):
        lims, D, I = idx.range_search(q, rho, allow=allow, exclude=exclude)
        counts = np.diff(lims)
        assert counts[7] > 4096
        k = int(min(max(counts.max(), 1), 4096))
        Ds, Is = idx.search(q, k, allow=allow, exclude=exclude)
        for i in range(nq):
            j = int(min(counts[i], k))
            _same(D[lims[i]:lims[i] + j], Ds[i, :j], "%s: D prefix of query %d" % (dtype, i))
            _same(I[lims[i]:lims[i] + j], Is[i, :j], "%s: I prefix of query %d" % (dtype, i))
            if counts[i] < k and Is[i, counts[i]] >= 0:
                assert Ds[i, counts[i]] <= rho[i], "query %d stops above its radius" % i


# ---------------------------------------------------------------------------------------------------------------------
# every scan shape
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["f32", "f16"])
@pytest.mark.parametrize("pair,cq,cx", [(0, 0, 0), (1, 0, 0), (1, 2, 2), (1, 4, 1), (1, 4, 2)])
def test_every_scan_shape(om, dtype, pair, cq, cx):
    n = 30000
    x, q, rng = _data(10 * cq + cx + pair, n, 256, 300)
    allow = rng.random(n) < 0.3
    rho = _sub_radii(om, x, allow, q, 500, dtype)
    excl = [list(rng.choice(n, 20, replace=False)) for _ in range(300)]
    idx = _index(om, x, dtype, pair_scan=pair, scan_cluster_q=cq, scan_cluster_x=cx)
    got = idx.range_search(q, rho, allow=allow, exclude=excl)
    if pair:
        assert idx.stat("scan_cluster") == 10 * (cq or 2) + (cx or 1)
    sub = _sub_range(om, x, allow, q, rho, dtype)
    _same3(got, _minus(*sub, excl), "shape %d %dx%d" % (pair, cq, cx))


def test_int8_scan(om):
    n = 30000
    x, q, rng = _data(53, n, 200, 300)
    allow = rng.random(n) < 0.3
    rho = _sub_radii(om, x, allow, q, 500, torch.int8)
    excl = [list(rng.choice(n, 20, replace=False)) for _ in range(300)]
    got = _index(om, x, torch.int8).range_search(q, rho, allow=allow, exclude=excl)
    _same3(got, _minus(*_sub_range(om, x, allow, q, rho, torch.int8), excl), "int8 scan")


# ---------------------------------------------------------------------------------------------------------------------
# exact paths
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_exact_only_and_non_finite_bounds(om, dtype):
    n, nq = 20000, 80
    x, q, rng = _data(61, n, 64, nq)
    allow = rng.random(n) < 0.4
    excl = [list(rng.choice(n, 64, replace=False)) for _ in range(nq)]
    rho = _sub_radii(om, x, allow, q, 300, dtype)
    idx = _index(om, x, dtype)
    want = idx.range_search(q, rho, allow=allow, exclude=excl)
    _same3(want, _minus(*_sub_range(om, x, allow, q, rho, dtype), excl), "%s sweep" % dtype)
    idx.set_param("exact_only", 1)
    _same3(idx.range_search(q, rho, allow=allow, exclude=excl), want, "%s exact_only" % dtype)
    assert idx.stat("exact_queries") == nq
    idx.set_param("exact_only", 0)
    # queries whose certificate bound is not finite (overflowing norms) take the exact scan with the filter
    bad = q[:6].copy()
    bad[1] *= 1e30
    bad[4] *= 1e30
    rb = np.array([rho[0], 0.0, rho[2], rho[3], 1e31, rho[5]], np.float32)
    got = idx.range_search(bad, rb, allow=allow, exclude=excl[:6])
    assert idx.stat("exact_queries") == 2
    assert np.diff(got[0])[1] > 0 and np.diff(got[0])[4] > 0, "premise: the exact queries have results"
    _same3(got, _minus(*_sub_range(om, x, allow, bad, rb, dtype), excl[:6]), "%s non-finite bound" % dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_integer_data_equals_the_oracle(om, dtype):
    rng = np.random.default_rng(2)
    n, nq = 30000, 100
    x = rng.integers(-8, 9, size=(n, 96)).astype(np.float32)
    q = rng.integers(-8, 9, size=(nq, 96)).astype(np.float32)
    x[:, 0], q[:, 0] = 127, 0  # int8 rows: scale 1, so every storage holds x exactly
    idx = _index(om, x, dtype)
    allow = rng.random(n) < 0.2
    excl = [list(rng.choice(n, 100, replace=False)) for _ in range(nq)]
    rho = np.quantile(q @ x[:2000].T, 0.97, axis=1, method="lower").astype(np.float32)
    for exact in (0, 1):
        idx.set_param("exact_only", exact)
        lims, D, I = idx.range_search(q, rho, allow=allow, exclude=excl)
        l0, D0, I0 = flat_ip_range_search_filtered(q, x, rho, allow=allow, exclude=excl)
        _same(lims, l0, "lims exact_only=%d" % exact)
        _same(I, I0, "I exact_only=%d" % exact)
        np.testing.assert_array_equal(D.astype(np.float64), D0)


# ---------------------------------------------------------------------------------------------------------------------
# re-sweeps
# ---------------------------------------------------------------------------------------------------------------------
def test_resweeps_and_long_lists(om):
    n, nq = 60000, 40
    x, q, rng = _data(5, n, 128, nq)
    allow = rng.random(n) < 0.6
    rho = _sub_radii(om, x, allow, q, 700, torch.float32)
    rho[3] = -np.inf  # 36000 results: lists longer than one shared-memory sort
    rho[5] = np.float32(-1.0)
    excl = [list(rng.choice(n, 128, replace=False)) for _ in range(nq)]
    want = _minus(*_sub_range(om, x, allow, q, rho, torch.float32), excl)
    assert np.diff(want[0])[3] > 16384
    idx = _index(om, x, torch.float32, range_list=256)
    got = idx.range_search(q, rho, allow=allow, exclude=excl)
    assert idx.stat("range_resweeps") > 2
    _same3(got, want, "range_list 256")
    idx.set_param("exact_only", 1)
    _same3(idx.range_search(q, rho, allow=allow, exclude=excl), want, "range_list 256, exact_only")


def test_a_bitmap_keeps_a_query_within_its_list(om):
    # every row passes radius -inf: 60000 candidates unfiltered, 600 under a 1 % bitmap, which fit range_list = 4096
    n = 60000
    x, q, rng = _data(7, n, 64, 3)
    allow = np.zeros(n, bool)
    allow[rng.choice(n, 600, replace=False)] = True
    idx = _index(om, x, torch.float32)
    rho = np.full(3, -np.inf, np.float32)
    idx.range_search(q, rho)
    assert idx.stat("range_resweeps") == 3, "premise: the whole corpus overflows the list"
    got = idx.range_search(q, rho, allow=allow)
    assert idx.stat("range_resweeps") == 0 and idx.stat("range_candidates") == 3 * 600
    _same3(got, _sub_range(om, x, allow, q, rho, torch.float32), "1 % bitmap at radius -inf")


# ---------------------------------------------------------------------------------------------------------------------
# near-duplicate detection
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_near_duplicates_of_stored_rows(om, dtype):
    rng = np.random.default_rng(71)
    n, d, nq = 40000, 64, 50
    x = rng.integers(-8, 9, size=(n, d)).astype(np.float32)
    x[:, 0] = 127  # int8: scale 1, every storage holds x exactly
    qrows = rng.choice(n, nq, replace=False)
    # 5 near-duplicates of each query row (one coordinate moved by 1) planted at random rows
    for r in qrows:
        for dst in rng.choice(n, 5, replace=False):
            if dst in qrows:
                continue
            x[dst] = x[r]
            x[dst, 1 + rng.integers(d - 1)] += rng.choice([-1.0, 1.0])
    q = x[qrows].copy()
    allow = np.zeros(n, bool)
    allow[: n // 2] = True  # a sub-collection
    allow[qrows] = True  # the queries themselves are in it, and each excludes itself
    rho = (np.einsum("ij,ij->i", q, q) - 20).astype(np.float32)
    excl = [[int(r)] for r in qrows]
    idx = _index(om, x, dtype)
    lims, D, I = idx.range_search(q, rho, allow=allow, exclude=excl)
    l0, D0, I0 = flat_ip_range_search_filtered(q, x, rho, allow=allow, exclude=excl)
    _same(lims, l0, "lims")
    _same(I, I0, "I")
    np.testing.assert_array_equal(D.astype(np.float64), D0)
    assert all(int(qrows[i]) not in I[lims[i]:lims[i + 1]] for i in range(nq)), "a query excludes itself"
    assert lims[-1] > 0, "premise: near-duplicates found"


# ---------------------------------------------------------------------------------------------------------------------
# contract edges
# ---------------------------------------------------------------------------------------------------------------------
def _raw(idx, q, rho, f, lims, id_offset=0):
    """om_index_range_search_filtered on device queries and radii, host lims; returns the code"""
    from openmatch_b200 import _lib
    return idx._lib.om_index_range_search_filtered(idx._h, q.data_ptr(), _lib.OM_DEVICE, q.shape[0], rho.data_ptr(),
                                                   lims.ctypes.data, _lib.OM_HOST, id_offset,
                                                   ctypes.byref(f) if f is not None else None,
                                                   torch.cuda.current_stream().cuda_stream)


def test_argument_rules_leave_lims_untouched(om):
    from openmatch_b200 import _lib
    n, nq = 5000, 6
    x, q, _ = _data(19, n, 64, nq)
    idx = _index(om, x, torch.float32)
    qd = torch.from_numpy(q).cuda()
    rho = torch.zeros(nq, device="cuda")
    words = om.pack_allow(torch.ones(n, dtype=torch.bool), n, "cuda")
    offs = torch.tensor([0, 1, 2, 3, 4, 5, 6], dtype=torch.int64, device="cuda")
    ids = torch.arange(6, dtype=torch.int64, device="cuda")
    alive = []

    def filt(allow_words=None, off=offs, ex=ids):
        alive.extend([off, ex])
        f = _lib.SearchFilter()
        if allow_words is not None:
            f.allow_bits, f.allow_words = words.data_ptr(), allow_words
        f.exclude_offsets = off.data_ptr() if off is not None else None
        f.exclude_ids = ex.data_ptr() if ex is not None else None
        return f

    too_many = torch.tensor([0, 129, 129, 129, 129, 129, 129], dtype=torch.int64, device="cuda")
    cases = {"allow_words too short": (filt(allow_words=(n + 31) // 32 - 1), "search filter"),
             "129 ids for one query": (filt(off=too_many, ex=torch.arange(129, dtype=torch.int64, device="cuda")),
                                       "search filter"),
             "offsets not monotone": (filt(off=torch.tensor([0, 2, 1, 3, 4, 5, 6], dtype=torch.int64, device="cuda")),
                                      "search filter"),
             "negative id": (filt(ex=torch.tensor([0, 1, -2, 3, 4, 5], dtype=torch.int64, device="cuda")),
                             "search filter")}
    for name, (f, msg) in cases.items():
        lims = np.full(nq + 1, -7, np.int64)
        assert _raw(idx, qd, rho, f, lims) == -1, name
        assert msg.encode() in idx._lib.om_last_error(), name
        assert (lims == -7).all(), "%s: lims written" % name
    lims = np.full(nq + 1, -7, np.int64)
    nan = torch.tensor([0, float("nan"), 0, 0, 0, 0], device="cuda")
    assert _raw(idx, qd, nan, filt(allow_words=(n + 31) // 32), lims) == -1
    assert b"NaN" in idx._lib.om_last_error() and (lims == -7).all(), "a NaN radius writes nothing"
    # the accepted edge: exactly 128 ids
    idx.range_search(q, 0.0, exclude=[list(range(128))] * nq)
    with pytest.raises(RuntimeError, match="more than 128"):
        idx.range_search(q, 0.0, exclude=[list(range(129))] + [[]] * (nq - 1))
    # non-finite stored rows are refused as by the unfiltered call
    s = _index(om, x, torch.float16)
    s.reserve_rows(1).fill_(float("inf"))
    s.commit_rows(1)
    with pytest.raises(RuntimeError, match="inf or NaN"):
        s.range_search(q, 0.0, allow=np.ones(n + 1, bool))


def test_null_and_empty_filters_are_the_unfiltered_call(om):
    from openmatch_b200 import _lib
    n, nq = 20000, 200
    x, q, _ = _data(23, n, 128, nq)
    idx = _index(om, x, torch.float16)
    qd = torch.from_numpy(q).cuda()
    rho = torch.full((nq,), 8.0, device="cuda")
    want = idx.range_search_device(qd, rho)
    launches = idx.stat("launches")
    for name, f in (("null", None), ("empty", _lib.SearchFilter())):
        lims = np.empty(nq + 1, np.int64)
        assert _raw(idx, qd, rho, f, lims) == 0, name
        assert idx.stat("launches") == launches, "%s filter: the unfiltered path's work" % name
        D = torch.empty(int(lims[-1]), device="cuda")
        I = torch.empty(int(lims[-1]), dtype=torch.int64, device="cuda")
        assert idx._lib.om_index_range_results(idx._h, D.data_ptr(), I.data_ptr(), _lib.OM_DEVICE,
                                               torch.cuda.current_stream().cuda_stream) == 0
        _same3((lims, D, I), want, "%s filter" % name)
    got = idx.range_search_device(qd, rho, allow=torch.ones(n, dtype=torch.bool, device="cuda"), exclude=[[]] * nq)
    _same3(got, want, "allow-all bitmap, empty exclusions")


def test_host_resident_index_is_refused(om):
    x, q, _ = _data(3, 3000, 32, 4)
    idx = om.FlatIPIndex(32, memory="host", window_rows=1024)
    idx.add(x)
    with pytest.raises(RuntimeError, match="host-resident"):
        idx.range_search(q, 0.0, allow=np.ones(3000, bool))
    with pytest.raises(RuntimeError, match="om_index_range_search_filtered.*host-resident"):
        idx.range_search(q, 0.0, exclude=[[1]] * 4)


def _busy(stream, seconds=0.2):
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(seconds * 1.5e9))


def _sequence(om, x, q, allow, excl, stream=None):
    out = []
    ctx = torch.cuda.stream(stream) if stream is not None else torch.cuda.stream(torch.cuda.current_stream())
    with ctx:
        if stream is not None:
            _busy(torch.cuda.default_stream())
        for dtype in DTYPES:
            idx = _index(om, x, dtype, range_list=256)
            qd = torch.from_numpy(q).cuda()
            allow_d = torch.from_numpy(allow).cuda()  # filter buffers made on the range search's stream
            for nq in (1, 129, 300):
                got = idx.range_search_device(qd[:nq], 9.0, allow=allow_d, exclude=excl[:nq])
                out.append(tuple(t.clone() for t in got))
                idx.search_device(qd[:nq], 10, allow=allow_d)
    torch.cuda.synchronize()
    return out


def test_side_stream_and_poisoned_allocations(om):
    x, q, rng = _data(29, 20000, 128, 300)
    allow = rng.random(20000) < 0.5
    excl = [list(rng.integers(0, 20000, 50)) for _ in range(300)]
    want = _sequence(om, x, q, allow, excl)
    os.environ["OPENMATCH_B200_POISON_ALLOC"] = "1"
    try:
        for what, got in (("side stream", _sequence(om, x, q, allow, excl, torch.cuda.Stream())),
                          ("poisoned", _sequence(om, x, q, allow, excl)),
                          ("poisoned, side stream", _sequence(om, x, q, allow, excl, torch.cuda.Stream()))):
            for i, (g, w) in enumerate(zip(got, want)):
                _same3(g, w, "%s step %d" % (what, i))
    finally:
        del os.environ["OPENMATCH_B200_POISON_ALLOC"]


# ---------------------------------------------------------------------------------------------------------------------
# sharded
# ---------------------------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _torchrun(nproc, timeout=900):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join("tests", "index_range_filter_dist_worker.py")]
    env = dict(os.environ, NCCL_DEBUG="WARN", OMP_NUM_THREADS="8")
    return subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)


def test_sharded_filtered_range_search_at_world_size_one(om):
    r = _torchrun(1, timeout=600)
    assert r.returncode == 0 and "RANGE FILTER DIST OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_sharded_filtered_range_search_on_two_gpus(om):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    r = _torchrun(2)
    assert r.returncode == 0 and "RANGE FILTER DIST OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
