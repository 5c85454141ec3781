"""GPU: range search (``om_index_range_search``, ``FlatIPIndex.range_search``).

Contract under test: for query i the result is every row whose fp32 score (as search computes it, over the stored rows)
is strictly greater than radius[i], ordered by (score desc, id asc); the first j results of a query are bitwise
``search(q, j)``'s D and I for every j <= min(count, 4096), on every storage and scan path, and equal to the exact scan's
(``exact_only``) bit for bit.  Float64 oracles: set equality on integer data, the re-score bound on Gaussian data."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from index_range_oracle import flat_ip_range_search
from oracle import search_bound as sb

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.float32, torch.float16, torch.int8]


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
    if x.shape[0]:
        idx.add(torch.from_numpy(x).cuda())
    for name, v in params.items():
        idx.set_param(name, v)
    return idx


def _stored(idx):
    return torch.cat(list(idx.rows_f32())).cpu().numpy() if idx.ntotal else np.zeros((0, idx.d), np.float32)


def _check_prefix(idx, q, rho, lims, D, I, what):
    """The first j results of every query are search(q, j)'s, j <= min(count, 4096)."""
    counts = np.diff(lims)
    k = int(min(max(int(counts.max()) if counts.size else 0, 1), 4096, max(idx.ntotal, 1)))
    Ds, Is = idx.search(q, k)
    for i in range(q.shape[0]):
        j = int(min(counts[i], k))
        _same(D[lims[i]:lims[i] + j], Ds[i, :j], "%s: D prefix of query %d" % (what, i))
        _same(I[lims[i]:lims[i] + j], Is[i, :j], "%s: I prefix of query %d" % (what, i))
        if counts[i] < k and Is[i, counts[i]] >= 0:
            assert Ds[i, counts[i]] <= rho[i], "%s: query %d stops above its radius" % (what, i)


def _radii(idx, q, kth):
    """radius per query: the kth score of search (a mix of k), so that counts differ between queries"""
    ks = np.minimum(np.array([kth, kth // 3 + 1, 1, 2 * kth])[np.arange(q.shape[0]) % 4], max(idx.ntotal, 1))
    D, _ = idx.search(q, int(ks.max()))
    return D[np.arange(q.shape[0]), ks - 1].astype(np.float32)


CASES = [(1, 64), (64, 768), (128, 1000), (129, 768), (1500, 64), (64, 30), (129, 1001)]  # d % 4 != 0: element path


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("nq,d", CASES)
def test_prefix_rule_and_exact_scan(om, dtype, nq, d):
    rng = np.random.default_rng(nq * 7 + d)
    x = rng.standard_normal((12000, d), dtype=np.float32)
    q = rng.standard_normal((nq, d), dtype=np.float32)
    idx = _index(om, x, dtype)
    rho = _radii(idx, q, 300)
    lims, D, I = idx.range_search(q, rho)
    _check_prefix(idx, q, rho, lims, D, I, "%s nq=%d d=%d" % (dtype, nq, d))
    idx.set_param("exact_only", 1)
    l2, D2, I2 = idx.range_search(q, rho)
    assert idx.stat("exact_queries") == nq
    _same(l2, lims, "lims vs exact_only")
    _same(D2, D, "D vs exact_only")
    _same(I2, I, "I vs exact_only")
    if nq <= 64:  # float64 oracle within the re-score bound
        xs = _stored(idx)
        s, beta = sb.score64(q, xs), sb.rescore_bound(q, xs)
        for i in range(nq):
            got = set(I[lims[i]:lims[i + 1]].tolist())
            must = set(np.flatnonzero(s[i] > rho[i] + beta[i]).tolist())
            may = set(np.flatnonzero(s[i] > rho[i] - beta[i]).tolist())
            assert must <= got <= may, "query %d" % i


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("pair,cq,cx", [(0, 0, 0), (1, 2, 2), (1, 4, 1), (1, 4, 2)])
def test_every_scan_shape(om, dtype, pair, cq, cx):
    rng = np.random.default_rng(11)
    x = rng.standard_normal((20000, 256), dtype=np.float32)
    q = rng.standard_normal((300, 256), dtype=np.float32)
    ref = _index(om, x, dtype)
    rho = _radii(ref, q, 500)
    l0, D0, I0 = ref.range_search(q, rho)
    idx = _index(om, x, dtype, pair_scan=pair, scan_cluster_q=cq, scan_cluster_x=cx)
    l1, D1, I1 = idx.range_search(q, rho)
    _same(l1, l0, "lims")
    _same(D1, D0, "D")
    _same(I1, I0, "I")
    _check_prefix(idx, q, rho, l1, D1, I1, "shape %d %d %d" % (pair, cq, cx))


@pytest.mark.parametrize("dtype", DTYPES)
def test_integer_data_equals_the_oracle(om, dtype):
    rng = np.random.default_rng(2)
    x = rng.integers(-8, 9, size=(30000, 96)).astype(np.float32)
    q = rng.integers(-8, 9, size=(200, 96)).astype(np.float32)
    x[:, 0], q[:, 0] = 127, 0  # int8 rows: scale 127 / 127 = 1, codes = values, so every storage holds x exactly
    idx = _index(om, x, dtype)
    np.testing.assert_array_equal(_stored(idx), x)
    xs = _stored(idx)
    rho = np.quantile(q @ xs[:2000].T, 0.97, axis=1, method="lower").astype(np.float32)  # radii equal to existing scores
    lims, D, I = idx.range_search(q, rho)
    l0, D0, I0 = flat_ip_range_search(q, xs, rho)
    _same(lims, l0, "lims")
    _same(I, I0, "I")
    np.testing.assert_array_equal(D.astype(np.float64), D0)
    # a radius equal to a row's score excludes that row
    s = D[lims[0]]
    lims2, _, I2 = idx.range_search(q[:1], float(s))
    assert I[lims[0]] not in I2.tolist() and lims2[1] == int((D0[l0[0]:l0[1]] > s).sum())


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_rows_below_the_radius_on_the_stage_are_returned(om, dtype):
    # 2000 copies of one fp16 row whose fp32 score sits above the radius while its fp16 stage score does not
    rng = np.random.default_rng(4)
    d = 256
    x = rng.standard_normal((20000, d)).astype(np.float16).astype(np.float32)
    q = rng.standard_normal((1, d), dtype=np.float32)
    for _ in range(5000):
        row = rng.standard_normal(d).astype(np.float16).astype(np.float32)
        s, B = sb.score64(q, row[None])[0, 0], sb.stage_exact(q, row[None])[0, 0]
        beta = sb.rescore_bound(q, row[None])[0, 0]
        rho = np.float32((s + B) / 2)
        if B <= rho and s - rho > beta:  # the fp32 re-score is above the radius for sure
            break
    else:
        pytest.fail("no row with a stage score below the radius found")
    dup = rng.choice(x.shape[0], 2000, replace=False)
    x[dup] = row
    assert (sb.stage_exact(q, x[dup]) <= rho).all() and (sb.score64(q, x[dup]) > rho).all(), "premise"
    idx = _index(om, x, dtype)
    lims, D, I = idx.range_search(q, rho)
    assert set(dup.tolist()) <= set(I.tolist()), "rows above the radius whose stage score is below it"
    idx.set_param("exact_only", 1)
    l2, D2, I2 = idx.range_search(q, rho)
    _same(I2, I, "I vs exact_only")
    _same(D2, D, "D vs exact_only")


def test_int8_rows_below_the_radius_on_the_stage_are_returned(om):
    # int8 storage: the stage is the scan of the two-level int8 query split (stage_i8), with its own E.  Rows of integer
    # codes with a +-127 and scale 2^-7, which the index stores exactly; 2000 copies of one whose fp32 score sits above the
    # radius while its stage score does not.
    import index_i8_oracle as io
    rng = np.random.default_rng(12)
    d = 256

    def rows(n):
        c = rng.integers(-100, 101, size=(n, d))
        c[:, 0] = 127
        return (c * 2.0 ** -7).astype(np.float32)

    x = rows(20000)
    q = rng.standard_normal((1, d), dtype=np.float32)
    for _ in range(5000):
        row = rows(1)
        codes, scales = io.quantize_i8(row)
        s, B = sb.score64(q, row)[0, 0], io.stage_i8(q, codes, scales)[0, 0]
        beta = sb.rescore_bound(q, row)[0, 0]
        rho = np.float32((s + B) / 2)
        if B <= rho and s - rho > beta:  # the fp32 re-score is above the radius for sure
            break
    else:
        pytest.fail("no row with a stage score below the radius found")
    dup = rng.choice(x.shape[0], 2000, replace=False)
    x[dup] = row[0]
    codes, scales = io.quantize_i8(x[dup])
    assert (io.stage_i8(q, codes, scales) <= rho).all() and (sb.score64(q, x[dup]) > rho).all(), "premise"
    idx = _index(om, x, torch.int8)
    np.testing.assert_array_equal(_stored(idx), x)
    lims, D, I = idx.range_search(q, rho)
    assert set(dup.tolist()) <= set(I.tolist()), "rows above the radius whose stage score is below it"
    idx.set_param("exact_only", 1)
    l2, D2, I2 = idx.range_search(q, rho)
    _same(I2, I, "I vs exact_only")
    _same(D2, D, "D vs exact_only")


def test_resweeps_and_long_lists(om):
    rng = np.random.default_rng(5)
    x = rng.standard_normal((60000, 128), dtype=np.float32)
    q = rng.standard_normal((40, 128), dtype=np.float32)
    ref = _index(om, x, torch.float32)
    rho = _radii(ref, q, 700)
    rho[3] = -np.inf  # 60000 results: lists longer than one shared-memory sort
    rho[5] = np.float32(-1.0)  # about 46000
    l0, D0, I0 = ref.range_search(q, rho)
    assert ref.stat("range_resweeps") >= 2 and np.diff(l0)[3] == 60000
    idx = _index(om, x, torch.float32, range_list=256)
    l1, D1, I1 = idx.range_search(q, rho)
    assert idx.stat("range_resweeps") > 2
    _same(l1, l0, "lims")
    _same(D1, D0, "D")
    _same(I1, I0, "I")
    _check_prefix(idx, q, rho, l1, D1, I1, "range_list 256")
    i3 = I0[l0[3]:l0[4]]
    assert np.array_equal(np.sort(i3), np.arange(60000))
    d3 = D0[l0[3]:l0[4]]
    assert (np.diff(d3) <= 0).all() and all(i3[j] < i3[j + 1] for j in np.flatnonzero(np.diff(d3) == 0))
    idx.set_param("exact_only", 1)
    l2, D2, I2 = idx.range_search(q, rho)
    _same(I2, I0, "I vs exact_only")
    _same(D2, D0, "D vs exact_only")


def test_a_query_with_two_million_results(om):
    rng = np.random.default_rng(6)
    x = torch.randn(2_000_000, 64, device="cuda", generator=torch.Generator("cuda").manual_seed(6)).half()
    idx = om.FlatIPIndex(64, dtype=torch.float16)
    idx.add(x)
    q = rng.standard_normal((2, 64), dtype=np.float32)
    lims, D, I = idx.range_search_device(torch.from_numpy(q).cuda(), torch.tensor([-np.inf, np.inf]))
    assert lims.tolist() == [0, 2_000_000, 2_000_000]
    assert torch.equal(torch.sort(I).values, torch.arange(2_000_000, device="cuda"))
    assert bool((D[1:] <= D[:-1]).all())
    tie = (D[1:] == D[:-1])
    assert bool((I[1:][tie] > I[:-1][tie]).all())
    Ds, Is = idx.search(q[:1], 4096)
    _same(D[:4096], Ds[0], "D prefix")
    _same(I[:4096], Is[0], "I prefix")


def test_edge_radii_empty_index_and_no_queries(om):
    rng = np.random.default_rng(8)
    x = rng.standard_normal((5000, 32), dtype=np.float32)
    q = rng.standard_normal((3, 32), dtype=np.float32)
    for dtype in DTYPES:
        idx = _index(om, x, dtype)
        lims, D, I = idx.range_search(q, [np.inf, -np.inf, np.inf])
        assert lims.tolist() == [0, 0, 5000, 5000] and D.size == I.size == 5000
        lims, D, I = idx.range_search(q[:0], 0.0)
        assert lims.tolist() == [0] and D.size == 0
        empty = om.FlatIPIndex(32, dtype=dtype)
        lims, D, I = empty.range_search(q, -np.inf)
        assert lims.tolist() == [0, 0, 0, 0] and D.size == 0


def _abi_call(om, idx, q, radius, lims):
    lib = idx._lib
    return lib.om_index_range_search(idx._h, q.ctypes.data, 0, q.shape[0], radius.ctypes.data, lims.ctypes.data, 0, 0,
                                     None)


def test_errors_and_state(om):
    from openmatch_b200 import _lib
    rng = np.random.default_rng(9)
    x = rng.standard_normal((3000, 48), dtype=np.float32)
    q = rng.standard_normal((4, 48), dtype=np.float32)
    idx = _index(om, x, torch.float32)
    D = np.full(8, 7.0, np.float32)
    I = np.full(8, 7, np.int64)
    assert idx._lib.om_index_range_results(idx._h, D.ctypes.data, I.ctypes.data, 0, None) == -5, "before any range search"
    lims = np.full(5, -7, np.int64)
    assert _abi_call(om, idx, q, np.array([0, np.nan, 0, 0], np.float32), lims) == -1
    assert (lims == -7).all(), "a NaN radius writes nothing"
    assert _abi_call(om, idx, q, np.full(4, 5.0, np.float32), lims) == 0 and lims[0] == 0
    total = int(lims[-1])
    Dr, Ir = np.empty(total, np.float32), np.empty(total, np.int64)
    assert idx._lib.om_index_range_results(idx._h, Dr.ctypes.data, Ir.ctypes.data, 0, None) == 0
    l2, D2, I2 = idx.range_search(q, 5.0)
    _same(l2, lims, "lims")
    _same(D2, Dr, "D")
    _same(I2, Ir, "I")
    idx.search(q, 3)
    assert idx._lib.om_index_range_results(idx._h, D.ctypes.data, I.ctypes.data, 0, None) == -5, "after a search"
    # queries holding inf / NaN, or overflowing norms, take the exact scan
    bad = q.copy()
    bad[1, 3] = np.inf
    bad[2, 0] = np.nan
    bad[3] *= 1e30
    lims, Db, Ib = idx.range_search(bad, 0.0)
    assert idx.stat("exact_queries") == 3
    idx.set_param("exact_only", 1)
    l2, D2, I2 = idx.range_search(bad, 0.0)
    _same(l2, lims, "lims, non-finite queries")
    _same(D2, Db, "D, non-finite queries")
    _same(I2, Ib, "I, non-finite queries")
    idx.set_param("exact_only", 0)
    with pytest.raises(ValueError, match="one value per query"):
        idx.range_search(q, [1.0, 2.0])
    # non-finite stored rows are refused as search refuses them
    for dtype in (torch.float16, torch.int8):
        s = _index(om, x, dtype)
        if dtype == torch.int8:  # a row of zero codes and an infinite scale
            p, pitch = s._rows_at(1)
            row = om._wrap_device(p, (1, pitch), pitch, torch.int8)
            row.zero_()
            dpad = (s.d + 15) // 16 * 16
            row[0, dpad:dpad + 4] = torch.tensor([np.inf], dtype=torch.float32).view(torch.int8).cuda()
        else:
            s.reserve_rows(1).fill_(float("inf"))
        s.commit_rows(1)
        with pytest.raises(RuntimeError, match="inf or NaN"):
            s.range_search(q, 0.0)
        assert s.stat("nonfinite_rows") == 1


def test_side_stream_and_poisoned_allocations(om):
    rng = np.random.default_rng(10)
    x = rng.standard_normal((20000, 128), dtype=np.float32)
    q = torch.from_numpy(rng.standard_normal((200, 128), dtype=np.float32)).cuda()
    ref = _index(om, x, torch.float16)
    l0, D0, I0 = ref.range_search_device(q, 9.0)
    os.environ["OPENMATCH_B200_POISON_ALLOC"] = "1"
    try:
        for dtype in DTYPES:
            want = _index(om, x, dtype).range_search_device(q, 9.0) if dtype != torch.float16 else (l0, D0, I0)
            idx = _index(om, x, dtype, range_list=256)
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                got = idx.range_search_device(q, 9.0)
                idx.search_device(q, 10)
                got2 = idx.range_search_device(q, 9.0)
            s.synchronize()
            for a, b, what in zip(got + got2, want + want, ("lims", "D", "I") * 2):
                _same(a, b, "%s, side stream, poisoned: %s" % (dtype, what))
    finally:
        del os.environ["OPENMATCH_B200_POISON_ALLOC"]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _torchrun(nproc, timeout=900):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join("tests", "index_range_dist_worker.py")]
    env = dict(os.environ, NCCL_DEBUG="WARN", OMP_NUM_THREADS="8")
    return subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)


def test_sharded_range_search_at_world_size_one(om):
    r = _torchrun(1, timeout=600)
    assert r.returncode == 0 and "RANGE DIST OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_sharded_range_search_on_two_gpus(om):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    r = _torchrun(2)
    assert r.returncode == 0 and "RANGE DIST OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
