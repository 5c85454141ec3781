"""GPU: the wide search scan (2-CTA clusters, 128 queries x 256 corpus rows per CTA, top-k filter on the wgmma
accumulator registers), which runs every round after the first for chunks of more than 128 queries.

Integer data => every fp16 product and fp32 partial sum is exact, so ids AND scores must match the oracle bit for bit.
The shapes sit on the kernel's edges: a pair row that is partly or entirely padding (nq around multiples of 256), a last
corpus tile with 255, 256 or 1 valid rows (the last round starts at a multiple of 256), and a partial k block (d = 72)."""
import numpy as np
import pytest
import torch

import oracle

pytestmark = pytest.mark.gpu

# the first round covers C = 1024 (k = 10) or 2048 (k = 100) rows and every later round doubles the rows seen, so the
# last round starts at row 8192 and its last corpus tile holds 255, 256 or 1 rows
_N = 256 * 60


@pytest.fixture(scope="module")
def om():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import index as om_index
    return om_index


def _int_data(rng, n, d, lo=-5, hi=5):
    return rng.integers(lo, hi + 1, size=(n, d)).astype(np.float32)


def _exact(om, x, q, k):
    idx = om.FlatIPIndex(x.shape[1])
    idx.add(x)
    D, I = idx.search(q, k)
    D0, I0 = oracle.flat_ip_search(q, x, k)
    np.testing.assert_array_equal(I, I0)
    np.testing.assert_array_equal(D, D0)
    return idx


@pytest.mark.parametrize("dn", [-1, 0, 1])
@pytest.mark.parametrize("nq", [129, 255, 256, 257, 383])
def test_shape_edges_partial_k_block(om, nq, dn):
    rng = np.random.default_rng(nq * 3 + dn)
    _exact(om, _int_data(rng, _N + dn, 72), _int_data(rng, nq, 72), 10)


@pytest.mark.parametrize("nq,dn", [(129, -1), (256, 0), (383, 1)])
@pytest.mark.parametrize("d", [768, 1024])
def test_shape_edges_wide_rows(om, d, nq, dn):
    rng = np.random.default_rng(d + nq)
    _exact(om, _int_data(rng, _N + dn, d), _int_data(rng, nq, d), 100)


def test_sorted_corpus_forces_overflow_retry_wide(om):
    # every later row beats every earlier row for every one of 300 queries: the doubling schedule overflows the
    # candidate lists inside the wide scan, and the overflow-proof schedule must take over
    n, d, nq = 60000, 64, 300
    v = np.arange(n) // 4  # ascending scores with 4-way ties
    x = np.zeros((n, d), np.float32)
    x[:, 0], x[:, 1] = v // 128, v % 128
    a = np.arange(1, nq + 1, dtype=np.float32)
    q = np.zeros((nq, d), np.float32)
    q[:, 0], q[:, 1] = 128 * a, a  # score = a * v: exact in fp16 operands and fp32 sums
    idx = _exact(om, x, q, 100)
    assert idx.stat("overflow_retries") >= 1


@pytest.mark.parametrize("k", [64, 1000])
def test_massive_ties_overflow_the_stash(om, k):
    # 0/1 data: scores take 65 values, so the early rounds let a large share of every tile through the threshold, far
    # more than the per-thread stash holds; the excess takes the synchronous path
    rng = np.random.default_rng(k)
    _exact(om, _int_data(rng, 30000, 64, 0, 1), _int_data(rng, 257, 64, 0, 1), k)


@pytest.mark.parametrize("d", [768, 1024])
def test_stage_error_model_holds_wide(om, d):
    # the certificate's accumulation term, |stage - exact sum of the half-rounded products| <= d 2^-22 |q_h||x_h|, on the
    # scores the wide scan produced (debug_stage_scores: D is the candidate-stage score)
    rng = np.random.default_rng(d + 1)
    n, nq, k = 50000, 192, 256
    x = rng.standard_normal((n, d), dtype=np.float32)
    q = rng.standard_normal((nq, d), dtype=np.float32)
    idx = om.FlatIPIndex(d)
    idx.add(x)
    idx.set_param("debug_stage_scores", 1)
    Ds, Is = idx.search(q, k)
    xh, qh = x.astype(np.float16).astype(np.float64), q.astype(np.float16).astype(np.float64)
    worst = 0.0
    for r in range(nq):
        B = xh[Is[r]] @ qh[r]
        bound = d * 2.0 ** -22 * np.linalg.norm(qh[r]) * np.linalg.norm(xh[Is[r]], axis=1)
        worst = max(worst, float(np.max(np.abs(Ds[r] - B) / bound)))
    assert worst < 0.25, "tensor-core accumulation error reaches %.3f of the modelled bound" % worst


def test_run_to_run_identical(om):
    rng = np.random.default_rng(5)
    x = rng.standard_normal((40000, 768), dtype=np.float32)
    q = rng.standard_normal((300, 768), dtype=np.float32)
    idx = om.FlatIPIndex(768)
    idx.add(x)
    D1, I1 = idx.search(q, 100)
    D2, I2 = idx.search(q, 100)
    np.testing.assert_array_equal(I1, I2)
    np.testing.assert_array_equal(D1, D2)
