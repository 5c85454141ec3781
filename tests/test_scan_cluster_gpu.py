"""GPU: the wide search scan on every cluster shape CQ x CX (CQ CTAs along the queries, CX along the corpus; each CTA
owns 128 queries x 256 corpus rows and multicasts its slices of the query box and the corpus tile to the CTAs that
share them).

Integer data => every fp16 product and fp32 partial sum is exact, so ids AND scores must match the oracle bit for bit.
The shapes sit on the cluster's edges: query counts around multiples of 512 (a 4 x 1 or 4 x 2 cluster tile that is
partly padding, whole CTAs of padding at nq = 200), last rounds whose last 512-row cluster tile holds 1, 255, 256, 257 or
511 valid rows (with CX = 2 the second CTA's corpus tile then lies wholly past the round for <= 256 rows), and a partial
k block (d = 72).  On Gaussian data the candidate-stage scores must be bitwise equal across shapes: every score comes
from the same wgmma sequence whichever CTA computes it."""
import numpy as np
import pytest
import torch

import oracle

pytestmark = pytest.mark.gpu

SHAPES = [(2, 1), (4, 1), (2, 2), (4, 2)]
_IDS = ["%dx%d" % s for s in SHAPES]

# Every round schedule these tests run at (k = 10 or 100, growth 2 or 8) starts its last round at row 2048, 4096 or 8192
# and every later round covers a multiple of 512 rows, so with N = _N0 + r the last cluster tile holds r valid rows.
_N0 = 256 * 60


@pytest.fixture(scope="module")
def om():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import index as om_index
    return om_index


def _int_data(rng, n, d, lo=-5, hi=5):
    return rng.integers(lo, hi + 1, size=(n, d)).astype(np.float32)


def _index(om, x, shape):
    idx = om.FlatIPIndex(x.shape[1])
    idx.add(x)
    if shape is not None:
        idx.set_param("scan_cluster_q", shape[0])
        idx.set_param("scan_cluster_x", shape[1])
    return idx


def _exact(om, x, q, k, shape):
    idx = _index(om, x, shape)
    D, I = idx.search(q, k)
    assert idx.stat("scan_cluster") == 10 * shape[0] + shape[1]
    assert idx.stat("scan_max_clusters") >= 1
    D0, I0 = oracle.flat_ip_search(q, x, k)
    np.testing.assert_array_equal(I, I0)
    np.testing.assert_array_equal(D, D0)
    return idx


@pytest.mark.parametrize("shape", SHAPES, ids=_IDS)
@pytest.mark.parametrize("nq", [129, 200, 511, 512, 513, 640])
def test_query_edges(om, nq, shape):
    rng = np.random.default_rng(nq)
    _exact(om, _int_data(rng, _N0 + 257, 72), _int_data(rng, nq, 72), 10, shape)


@pytest.mark.parametrize("shape", SHAPES, ids=_IDS)
@pytest.mark.parametrize("r", [1, 255, 256, 257, 511])
def test_last_cluster_tile_edges(om, r, shape):
    rng = np.random.default_rng(1000 + r)
    _exact(om, _int_data(rng, _N0 + r, 72), _int_data(rng, 513, 72), 10, shape)


@pytest.mark.parametrize("shape", SHAPES, ids=_IDS)
@pytest.mark.parametrize("d,r", [(768, 1), (1024, 257)])
def test_wide_rows(om, d, r, shape):
    rng = np.random.default_rng(d + r)
    _exact(om, _int_data(rng, _N0 + r, d), _int_data(rng, 600, d), 100, shape)


@pytest.mark.parametrize("k", [100, 1000])
@pytest.mark.parametrize("d", [768, 1024])
def test_stage_scores_bitwise_equal_across_shapes(om, d, k):
    rng = np.random.default_rng(d + k)
    x = rng.standard_normal((40000, d), dtype=np.float32)
    q = rng.standard_normal((600, d), dtype=np.float32)
    ref = None
    for shape in SHAPES:
        idx = _index(om, x, shape)
        idx.set_param("debug_stage_scores", 1)
        D, I = idx.search(q, k)
        assert idx.stat("scan_cluster") == 10 * shape[0] + shape[1]
        assert idx.stat("rounds") > 1
        if ref is None:
            ref = (D, I)
        else:
            np.testing.assert_array_equal(I, ref[1])
            np.testing.assert_array_equal(D.view(np.uint32), ref[0].view(np.uint32))


@pytest.mark.parametrize("shape", SHAPES, ids=_IDS)
def test_sorted_corpus_forces_overflow_retry(om, shape):
    # every later row beats every earlier row for every query: the doubling schedule overflows the candidate lists
    # inside the cluster scan, and the overflow-proof schedule must take over
    n, d, nq = 60000, 64, 600
    v = np.arange(n) // 4  # ascending scores with 4-way ties
    x = np.zeros((n, d), np.float32)
    x[:, 0], x[:, 1] = v // 128, v % 128
    a = np.arange(1, nq + 1, dtype=np.float32) / 4
    q = np.zeros((nq, d), np.float32)
    q[:, 0], q[:, 1] = 128 * a, a  # score = a * v: exact in fp16 operands and fp32 sums
    idx = _exact(om, x, q, 100, shape)
    assert idx.stat("overflow_retries") >= 1


@pytest.mark.parametrize("shape", SHAPES, ids=_IDS)
def test_massive_ties_overflow_the_stash(om, shape):
    # 0/1 data: scores take 65 values, so the early rounds let a large share of every tile through the threshold, far
    # more than the per-thread stash holds; the excess takes the synchronous path
    rng = np.random.default_rng(7)
    _exact(om, _int_data(rng, 30000, 64, 0, 1), _int_data(rng, 513, 64, 0, 1), 1000, shape)


def test_auto_shape_is_run_to_run_identical_and_equals_4x2(om):
    rng = np.random.default_rng(5)
    x = rng.standard_normal((40000, 768), dtype=np.float32)
    q = rng.standard_normal((4100, 768), dtype=np.float32)
    idx = _index(om, x, None)
    D1, I1 = idx.search(q, 100)
    assert idx.stat("scan_cluster") == 21  # the automatic shape
    D2, I2 = idx.search(q, 100)
    assert idx.stat("scan_cluster") == 21
    np.testing.assert_array_equal(I1, I2)
    np.testing.assert_array_equal(D1, D2)
    idx.set_param("scan_cluster_q", 4)
    idx.set_param("scan_cluster_x", 2)
    D3, I3 = idx.search(q, 100)
    assert idx.stat("scan_cluster") == 42
    np.testing.assert_array_equal(I1, I3)
    np.testing.assert_array_equal(D1, D3)


def test_small_chunks_keep_their_kernels(om):
    rng = np.random.default_rng(11)
    x = _int_data(rng, 20000, 64)
    idx = _index(om, x, None)
    idx.search(_int_data(rng, 128, 64), 10)
    assert idx.stat("scan_cluster") == 0  # <= 128 queries: the single-CTA kernel
    idx.search(_int_data(rng, 300, 64), 10)
    assert idx.stat("scan_cluster") == 21
    idx.set_param("pair_scan", 0)
    idx.search(_int_data(rng, 300, 64), 10)
    assert idx.stat("scan_cluster") == 0


@pytest.mark.parametrize("name,value", [("scan_cluster_q", 1), ("scan_cluster_q", 3), ("scan_cluster_q", 8),
                                        ("scan_cluster_q", -2), ("scan_cluster_x", 3), ("scan_cluster_x", 4),
                                        ("scan_cluster_x", -1)])
def test_invalid_shape_parameters(om, name, value):
    idx = om.FlatIPIndex(16)
    with pytest.raises(RuntimeError, match=r"\(code -1\)"):
        idx.set_param(name, value)
