"""GPU: filtered search (``om_index_search_filtered``, ``FlatIPIndex.search(..., allow=, exclude=)``).

Contract under test: a filtered search returns the exact top-k, by fp32 inner product over the stored rows, among the
rows the bitmap allows and the query does not exclude, ties by ascending id.  So its D and I must be bitwise what an
unfiltered search returns on an index built from the eligible rows only, with ids mapped back, for every storage (a
row's stored values and its re-score order do not depend on the other rows); fewer than k eligible rows leave id -1 /
-FLT_MAX slots.  Exclusions are checked against an unfiltered top-(k + 128) with the excluded ids removed."""
import ctypes
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import search_bound as sb

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATS = ("uncertified", "uncertified_wide", "exact_queries")
DEFAULTS = {"round_growth": 0, "certify": 1, "exact_only": 0, "force_safe_rounds": 0, "pair_scan": 1,
            "scan_cluster_q": 0, "scan_cluster_x": 0}
DTYPES = [torch.float32, torch.float16, torch.int8]
NEG = np.float32(-np.finfo(np.float32).max)


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


def _index(om, x, dtype, **params):
    idx = om.FlatIPIndex(x.shape[1], dtype=dtype)
    idx.add(torch.from_numpy(x).cuda())
    for name, v in {**DEFAULTS, **params}.items():
        idx.set_param(name, v)
    return idx


def _sub_search(om, x, eligible, q, k, dtype, **params):
    """Unfiltered search of an index of x[eligible] only, ids mapped back to rows of x."""
    rows = np.flatnonzero(eligible)
    if rows.size == 0:
        return np.full((q.shape[0], k), NEG, np.float32), np.full((q.shape[0], k), -1, np.int64)
    D, I = _index(om, x[rows], dtype, **params).search(q, k)
    return D, np.where(I >= 0, rows[np.maximum(I, 0)], -1)


def _check_sub(om, x, allow, q, k, dtype, what, idx=None, **params):
    idx = idx if idx is not None else _index(om, x, dtype, **params)
    for name, v in {**DEFAULTS, **params}.items():
        idx.set_param(name, v)
    D, I = idx.search(q, k, allow=allow)
    D0, I0 = _sub_search(om, x, allow, q, k, dtype, **params)
    _same(I, I0, "%s: I" % what)
    _same(D, D0, "%s: D" % what)
    return idx, D, I


def _data(seed, n, d, nq):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((n, d), dtype=np.float32), rng.standard_normal((nq, d), dtype=np.float32), rng


# ---------------------------------------------------------------------------------------------------------------------
# bitwise against a sub-index
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "i8"])
@pytest.mark.parametrize("nq", [1, 64, 128, 129, 1500])
@pytest.mark.parametrize("k", [10, 1000])
def test_bitmap_equals_sub_index(om, dtype, nq, k):
    x, q, rng = _data(nq * 7 + k, 30000, 768, nq)
    allow = rng.random(30000) < 0.5
    _check_sub(om, x, allow, q, k, dtype, "nq=%d k=%d" % (nq, k))


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "i8"])
@pytest.mark.parametrize("k,d", [(1, 64), (4096, 64), (100, 1000), (4096, 768)])
def test_bitmap_k_and_d(om, dtype, k, d):
    x, q, rng = _data(k + d, 20000, d, 130)
    allow = rng.random(20000) < 0.4
    _check_sub(om, x, allow, q, k, dtype, "k=%d d=%d" % (k, d))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["f32", "f16"])
@pytest.mark.parametrize("pair,cq,cx", [(0, 0, 0), (1, 2, 1), (1, 4, 1), (1, 2, 2), (1, 4, 2)])
def test_bitmap_on_every_scan_shape(om, dtype, pair, cq, cx):
    x, q, rng = _data(10 * cq + cx + pair, 40000, 256, 1500)
    allow = rng.random(40000) < 0.3
    idx, _, _ = _check_sub(om, x, allow, q, 100, dtype, "pair_scan=%d %dx%d" % (pair, cq, cx), pair_scan=pair,
                           scan_cluster_q=cq, scan_cluster_x=cx)
    if pair:
        assert idx.stat("scan_cluster") == 10 * cq + cx


# ---------------------------------------------------------------------------------------------------------------------
# selectivity
# ---------------------------------------------------------------------------------------------------------------------
def _selections(n, k, rng):
    """name -> bool [n].  The first round of a k = 100 search of <= 256 queries scans C = 4096 rows."""
    first = 4096
    out = {"all": np.ones(n, bool), "half": rng.random(n) < 0.5, "1%": rng.random(n) < 0.01,
           "1e-4": rng.random(n) < 1e-4, "none": np.zeros(n, bool)}
    s = np.zeros(n, bool)
    s[rng.choice(n, k - 1, replace=False)] = True
    out["k-1 rows"] = s
    s = np.zeros(n, bool)
    s[2 * first + rng.choice(n - 2 * first, 3 * k, replace=False)] = True
    out["past the first round"] = s
    s = np.zeros(n, bool)
    s[rng.choice(first, k // 2, replace=False)] = True
    out["inside the first round"] = s
    s = np.zeros(n, bool)
    s[n // 3:n // 3 + n // 100] = True
    out["one range"] = s
    return out


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "i8"])
@pytest.mark.parametrize("nq", [1, 129])
def test_selectivity(om, dtype, nq):
    n, k = 50000, 100
    x, q, rng = _data(nq, n, 128, nq)
    idx = _index(om, x, dtype)
    for name, allow in _selections(n, k, rng).items():
        for exact_only in (0, 1):
            _, D, I = _check_sub(om, x, allow, q, k, dtype, "%s exact_only=%d" % (name, exact_only), idx=idx,
                                 exact_only=exact_only)
            m = int(allow.sum())
            if m < k:  # padding past the eligible rows
                assert (I[:, m:] == -1).all() and (D[:, m:].view(np.uint32) == NEG.view(np.uint32)).all(), name
                assert (I[:, :m] >= 0).all(), name
            assert np.isin(I[I >= 0], np.flatnonzero(allow)).all(), name


def test_dense_round_with_few_allowed_rows(om):
    """Fewer than kp = k + slack allowed rows in the first round's C rows, and none at all there: the list must count
    allowed rows only, and the later rounds must keep every allowed row that beats the threshold."""
    n, k = 30000, 1000
    x, q, rng = _data(5, n, 64, 300)
    for dtype in DTYPES:
        idx = _index(om, x, dtype)
        for name, lo in (("few in the first round", 1000), ("none in the first round", 8192)):
            allow = np.zeros(n, bool)
            allow[rng.choice(lo, 50, replace=False)] = lo == 1000
            allow[lo + rng.choice(n - lo, 2 * k, replace=False)] = True
            for safe in (0, 1):
                _check_sub(om, x, allow, q, k, dtype, "%s %s safe=%d" % (dtype, name, safe), idx=idx,
                           force_safe_rounds=safe)


# ---------------------------------------------------------------------------------------------------------------------
# adversarial: the disallowed rows are each query's near-duplicates, so the max test fires on every tile
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "i8"])
@pytest.mark.parametrize("nq", [64, 300])
def test_disallowed_near_duplicates(om, dtype, nq):
    n, d, k = 40000, 256, 50
    x, q, rng = _data(nq + 1, n, d, nq)
    dup = rng.choice(n, n // 2, replace=False)
    x[dup] = 4 * q[rng.integers(0, nq, dup.size)] + 1e-3 * rng.standard_normal((dup.size, d), dtype=np.float32)
    allow = np.ones(n, bool)
    allow[dup] = False
    idx, D, I = _check_sub(om, x, allow, q, k, dtype, "near-duplicates disallowed")
    stats = {s: idx.stat(s) for s in STATS}
    print("[filter adversarial] %s nq=%d: %s" % (dtype, nq, stats))
    assert all(v >= 0 for v in stats.values())


# ---------------------------------------------------------------------------------------------------------------------
# exclusions
# ---------------------------------------------------------------------------------------------------------------------
def _minus(D, I, excl, k):
    """top-k of the (D, I) lists after removing each query's excluded ids"""
    Dk = np.full((D.shape[0], k), NEG, np.float32)
    Ik = np.full((D.shape[0], k), -1, np.int64)
    for i in range(D.shape[0]):
        keep = (I[i] >= 0) & ~np.isin(I[i], np.asarray(list(excl[i]), np.int64))
        m = min(k, int(keep.sum()))
        Dk[i, :m], Ik[i, :m] = D[i][keep][:m], I[i][keep][:m]
    return Dk, Ik


def _check_excl(idx, q, k, excl, what, id_offset=0, allow=None, ref=None):
    D, I = idx.search(q, k, id_offset=id_offset, allow=allow, exclude=excl)
    if ref is None:
        D0, I0 = idx.search(q, min(k + 128, 4096), id_offset=id_offset, allow=allow)
    else:
        D0, I0 = ref
    Dk, Ik = _minus(D0, I0, excl, k)
    _same(I, Ik, "%s: I" % what)
    _same(D, Dk, "%s: D" % what)
    return D, I


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "i8"])
@pytest.mark.parametrize("nq,k", [(1, 10), (64, 100), (300, 1000), (129, 3968)])
def test_exclude_128_of_the_top_k(om, dtype, nq, k):
    x, q, rng = _data(nq + k, 30000, 128, nq)
    idx = _index(om, x, dtype)
    _, I = idx.search(q, k + 128 if k + 128 <= 4096 else k)
    excl = [list(rng.choice(I[i, :k], min(128, k), replace=False)) for i in range(nq)]
    _check_excl(idx, q, k, excl, "128 of the top-k")
    # the float64 oracle over the eligible stored rows of each query
    stored = torch.cat(list(idx.rows_f32())).cpu().numpy()
    for i in range(min(nq, 4)):
        keep = np.setdiff1d(np.arange(x.shape[0]), excl[i])
        xs = stored[keep]
        D, I = idx.search(q[i:i + 1], k, exclude=[excl[i]])
        Is = np.searchsorted(keep, I)  # row of the eligible sub-matrix
        sb.check_topk(q[i:i + 1], xs, D, Is, k)


def test_k_4096_with_exclusions_answers_exactly(om):
    x, q, rng = _data(9, 20000, 64, 20)
    idx = _index(om, x, torch.float32)
    _, I = idx.search(q, 4096)
    excl = [list(rng.choice(I[i], 128, replace=False)) for i in range(20)]
    D, I2 = idx.search(q, 4096, exclude=excl)
    keep = [np.setdiff1d(np.arange(20000), e) for e in excl]
    for i in range(20):
        D0, I0 = _index(om, x[keep[i]], torch.float32).search(q[i:i + 1], 4096)
        _same(I2[i:i + 1], keep[i][I0], "k=4096 query %d: I" % i)
        _same(D[i:i + 1], D0, "k=4096 query %d: D" % i)


def test_exclusion_duplicates_and_other_shards(om):
    n, k, off = 20000, 100, 1 << 33
    x, q, rng = _data(11, n, 96, 70)
    idx = _index(om, x, torch.float32)
    D0, I0 = idx.search(q, k + 128, id_offset=off)
    excl = []
    for i in range(70):
        mine = list(rng.choice(I0[i, :k], 20, replace=False))
        other = list(rng.integers(0, off, 40)) + list(off + n + rng.integers(0, 10 ** 6, 40))  # ids of other shards
        excl.append(mine + mine[:8] + other[:108 - 28 - 8])
        assert len(excl[-1]) <= 128
    _check_excl(idx, q, k, excl, "duplicates and other shards", id_offset=off, ref=(D0, I0))
    # as an (offsets, ids) CSR of device tensors
    offs = torch.tensor(np.concatenate([[0], np.cumsum([len(e) for e in excl])]), device="cuda")
    ids = torch.tensor([i for e in excl for i in e], dtype=torch.int64, device="cuda")
    D1, I1 = idx.search(q, k, id_offset=off, exclude=(offs, ids))
    D2, I2 = idx.search(q, k, id_offset=off, exclude=excl)
    _same(I1, I2, "CSR input: I")
    _same(D1, D2, "CSR input: D")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "i8"])
def test_exclusions_with_a_bitmap(om, dtype):
    n, k, nq = 30000, 200, 150
    x, q, rng = _data(13, n, 128, nq)
    allow = rng.random(n) < 0.3
    rows = np.flatnonzero(allow)
    sub = _index(om, x[rows], dtype)
    D0, I0 = sub.search(q, k + 128)
    excl_sub = [list(rng.choice(I0[i, :k], 100, replace=False)) for i in range(nq)]
    excl = [list(rows[e]) + list(rng.choice(np.flatnonzero(~allow), 20)) for e in excl_sub]  # + disallowed ids
    Dk, Ik = _minus(D0, I0, excl_sub, k)
    D, I = _index(om, x, dtype).search(q, k, allow=allow, exclude=excl)
    _same(I, np.where(Ik >= 0, rows[np.maximum(Ik, 0)], -1), "bitmap + exclusions: I")
    _same(D, Dk, "bitmap + exclusions: D")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "i8"])
def test_exclusions_on_the_exact_and_safe_paths(om, dtype):
    n, k, nq = 20000, 50, 40
    x, q, rng = _data(17, n, 64, nq)
    idx = _index(om, x, dtype)
    ref = idx.search(q, k + 128)
    excl = [list(rng.choice(ref[1][i, :k], 30, replace=False)) for i in range(nq)]
    for params in ({"exact_only": 1}, {"force_safe_rounds": 1}):
        for name, v in {**DEFAULTS, **params}.items():
            idx.set_param(name, v)
        _check_excl(idx, q, k, excl, str(params), ref=ref)
    # escalation forced by near-duplicate rows: thousands of rows that collide at the scan's precision
    xd = x.copy()
    dup = rng.choice(n, 5000, replace=False)
    v = rng.standard_normal(64, dtype=np.float32)
    xd[dup] = v + 1e-6 * rng.standard_normal((5000, 64), dtype=np.float32)
    qd = (v + 0.05 * rng.standard_normal((nq, 64), dtype=np.float32)).astype(np.float32)
    idx = _index(om, xd, dtype)
    ref = idx.search(qd, k + 128)
    excl = [list(rng.choice(ref[1][i, :k], 40, replace=False)) for i in range(nq)]
    _check_excl(idx, qd, k, excl, "near-duplicates", ref=ref)
    print("[filter escalation] %s: %s" % (dtype, {s: idx.stat(s) for s in STATS}))
    assert idx.stat("exact_queries") > 0, "premise: the exact level must run"
    _check_sub(om, xd, ~np.isin(np.arange(n), dup[:2500]), qd, k, dtype, "near-duplicates, half disallowed", idx=idx)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "i8"])
def test_exclusions_on_an_escalated_subset(om, dtype):
    """Only the odd queries meet thousands of near-duplicate rows, so the 4096-wide level and the exact level each answer
    a proper subset of the batch: every escalated query must keep its own excluded ids there."""
    n, k, nq = 20000, 50, 40
    x, q, rng = _data(19, n, 64, nq)
    dup = rng.choice(n, 5000, replace=False)
    v = rng.standard_normal(64, dtype=np.float32)
    x[dup] = v + 1e-6 * rng.standard_normal((5000, 64), dtype=np.float32)
    q[1::2] = v + 0.05 * rng.standard_normal((nq // 2, 64), dtype=np.float32)
    idx = _index(om, x, dtype)
    ref = idx.search(q, k + 128)
    excl = [list(rng.choice(ref[1][i, :k], 40, replace=False)) for i in range(nq)]
    _check_excl(idx, q, k, excl, "escalated subset", ref=ref)
    stats = {s: idx.stat(s) for s in STATS}
    print("[filter escalated subset] %s: %s" % (dtype, stats))
    assert stats["uncertified"] < nq and stats["exact_queries"] > 0, "premise: a proper subset reaches both levels"


# ---------------------------------------------------------------------------------------------------------------------
# contract edges
# ---------------------------------------------------------------------------------------------------------------------
def _raw(idx, q, k, f, D, I, id_offset=0):
    """om_index_search_filtered on device tensors; returns the code"""
    from openmatch_b200 import _lib
    return idx._lib.om_index_search_filtered(idx._h, q.data_ptr(), _lib.OM_DEVICE, q.shape[0], k, D.data_ptr(),
                                             I.data_ptr(), _lib.OM_DEVICE, id_offset,
                                             ctypes.byref(f) if f is not None else None,
                                             torch.cuda.current_stream().cuda_stream)


def test_argument_rules_leave_outputs_untouched(om):
    from openmatch_b200 import _lib
    n, k, nq = 5000, 10, 6
    x, q, _ = _data(19, n, 64, nq)
    idx = _index(om, x, torch.float32)
    qd = torch.from_numpy(q).cuda()
    words = om.pack_allow(torch.ones(n, dtype=torch.bool), n, "cuda")
    offs = torch.tensor([0, 1, 2, 3, 4, 5, 6], dtype=torch.int64, device="cuda")
    ids = torch.arange(6, dtype=torch.int64, device="cuda")

    alive = []  # the filter holds raw pointers: its tensors must outlive the calls

    def filt(allow_words=None, off=offs, ex=ids):
        alive.extend([off, ex])
        f = _lib.SearchFilter()
        if allow_words is not None:
            f.allow_bits, f.allow_words = words.data_ptr(), allow_words
        f.exclude_offsets = off.data_ptr() if off is not None else None
        f.exclude_ids = ex.data_ptr() if ex is not None else None
        return f

    too_many = torch.tensor([0, 129, 129, 129, 129, 129, 129], dtype=torch.int64, device="cuda")
    cases = {"allow_words too short": filt(allow_words=(n + 31) // 32 - 1),
             "129 ids for one query": filt(off=too_many, ex=torch.arange(129, dtype=torch.int64, device="cuda")),
             "offsets not monotone": filt(off=torch.tensor([0, 2, 1, 3, 4, 5, 6], dtype=torch.int64, device="cuda")),
             "negative id": filt(ex=torch.tensor([0, 1, -2, 3, 4, 5], dtype=torch.int64, device="cuda"))}
    for name, f in cases.items():
        D = torch.full((nq, k), 7.0, device="cuda")
        I = torch.full((nq, k), 7, dtype=torch.int64, device="cuda")
        rc = _raw(idx, qd, k, f, D, I)
        assert rc < 0, name
        assert b"search filter" in idx._lib.om_last_error(), name
        assert (D == 7.0).all() and (I == 7).all(), "%s: outputs written" % name
    with pytest.raises(RuntimeError, match="more than 128"):
        idx.search(q, k, exclude=[list(range(129))] + [[]] * (nq - 1))
    # the accepted edge: exactly 128 ids
    idx.search(q, k, exclude=[list(range(128))] * nq)


def test_null_and_empty_filters_are_the_unfiltered_search(om):
    from openmatch_b200 import _lib
    n, k, nq = 20000, 100, 200
    x, q, _ = _data(23, n, 128, nq)
    idx = _index(om, x, torch.float32)
    qd = torch.from_numpy(q).cuda()
    D0, I0 = idx.search_device(qd, k)
    for name, f in (("null", None), ("empty", _lib.SearchFilter())):
        D = torch.empty_like(D0)
        I = torch.empty_like(I0)
        assert _raw(idx, qd, k, f, D, I) == 0, name
        _same(I, I0, "%s filter: I" % name)
        _same(D, D0, "%s filter: D" % name)
    # an allow-all bitmap and exclusion lists that are all empty
    D, I = idx.search_device(qd, k, allow=torch.ones(n, dtype=torch.bool, device="cuda"), exclude=[[]] * nq)
    _same(I, I0, "allow-all: I")
    _same(D, D0, "allow-all: D")


def _busy(stream, seconds=0.2):
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(seconds * 1.5e9))


def _filtered_sequence(om, x, q, allow, excl, stream=None):
    out = []
    ctx = torch.cuda.stream(stream) if stream is not None else torch.cuda.stream(torch.cuda.current_stream())
    with ctx:
        if stream is not None:
            _busy(torch.cuda.default_stream())
        for dtype in DTYPES:
            idx = om.FlatIPIndex(x.shape[1], dtype=dtype)
            idx.add(torch.from_numpy(x).cuda())
            qd = torch.from_numpy(q).cuda()
            allow_d = torch.from_numpy(allow).cuda()  # filter buffers made on the search's stream
            for nq in (1, 129, 300):
                D, I = idx.search_device(qd[:nq], 20, allow=allow_d, exclude=excl[:nq])
                out.append((D.clone(), I.clone()))
    torch.cuda.synchronize()
    return out


def test_side_stream_and_poisoned_allocations(om):
    x, q, rng = _data(29, 8000, 96, 300)
    allow = rng.random(8000) < 0.5
    excl = [list(rng.integers(0, 8000, 50)) for _ in range(300)]
    want = _filtered_sequence(om, x, q, allow, excl)
    os.environ["OPENMATCH_B200_POISON_ALLOC"] = "1"
    try:
        for what, got in (("side stream", _filtered_sequence(om, x, q, allow, excl, torch.cuda.Stream())),
                          ("poisoned", _filtered_sequence(om, x, q, allow, excl)),
                          ("poisoned, side stream", _filtered_sequence(om, x, q, allow, excl, torch.cuda.Stream()))):
            for i, ((D, I), (D0, I0)) in enumerate(zip(got, want)):
                _same(I, I0, "%s step %d: I" % (what, i))
                _same(D, D0, "%s step %d: D" % (what, i))
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
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join("tests", "index_filter_dist_worker.py")]
    env = dict(os.environ, NCCL_DEBUG="WARN", OMP_NUM_THREADS="8")
    return subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)


def test_sharded_filtered_search_at_world_size_one(om):
    r = _torchrun(1, timeout=600)
    assert r.returncode == 0 and "FILTER DIST OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_sharded_filtered_search_on_two_gpus(om):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    r = _torchrun(2)
    assert r.returncode == 0 and "FILTER DIST OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
