"""GPU parity: libopenmatch_b200 index (through the C ABI) vs the CPU oracle (oracle/flat_index.py).

Integer-valued data => every product/partial sum is exact in bf16 x bf16 -> fp32 and in fp32, so ids AND
scores must match the oracle bit for bit, including the (score desc, row asc) tie order.  Gaussian data =>
eps-tie-aware comparison against float64 scores (tolerance stated at each assert)."""
import numpy as np
import pytest
import torch

import oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def om():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import index as om_index
    return om_index


def _int_data(rng, n, d, lo=-8, hi=8):
    return rng.integers(lo, hi + 1, size=(n, d)).astype(np.float32)


@pytest.mark.parametrize("n,d,nq,k", [(20000, 64, 37, 1), (20000, 64, 37, 10), (20000, 64, 37, 100),
                                       (20000, 64, 37, 1000), (5000, 768, 130, 100), (3000, 100, 5, 7),
                                       (257, 72, 3, 50)])
def test_integer_data_exact(om, n, d, nq, k):
    rng = np.random.default_rng(n + d + k)
    x, q = _int_data(rng, n, d), _int_data(rng, nq, d)
    idx = om.FlatIPIndex(d)
    idx.add(x)
    D, I = idx.search(q, k)
    D0, I0 = oracle.flat_ip_search(q, x, k)
    np.testing.assert_array_equal(I, I0)
    np.testing.assert_array_equal(D, D0)


def test_massive_ties(om):
    # scores take only a handful of distinct values: tie order (row ascending) decides almost every rank
    rng = np.random.default_rng(7)
    x, q = _int_data(rng, 30000, 64, 0, 1), _int_data(rng, 9, 64, 0, 1)
    idx = om.FlatIPIndex(64)
    idx.add(x)
    for k in (1, 64, 1000):
        D, I = idx.search(q, k)
        D0, I0 = oracle.flat_ip_search(q, x, k)
        np.testing.assert_array_equal(I, I0)
        np.testing.assert_array_equal(D, D0)


def test_incremental_add_reset_and_padding(om):
    rng = np.random.default_rng(3)
    x, q = _int_data(rng, 700, 64), _int_data(rng, 4, 64)
    idx = om.FlatIPIndex(64)
    assert idx.ntotal == 0
    D, I = idx.search(q, 5)  # empty index: all padding
    assert (I == -1).all() and (D == oracle.flat_index.NEG_FILL).all()
    idx.add(x[:100]); idx.add(x[100:101]); idx.add(torch.from_numpy(x[101:]).cuda())
    assert idx.ntotal == 700
    D, I = idx.search(q, 20)
    D0, I0 = oracle.flat_ip_search(q, x, 20)
    np.testing.assert_array_equal(I, I0)
    idx.reset()
    assert idx.ntotal == 0
    idx.add(x[:6])
    D, I = idx.search(q, 10)  # k > ntotal: tail padded with -1 / lowest(float) like faiss
    D0, I0 = oracle.flat_ip_search(q, x[:6], 10)
    np.testing.assert_array_equal(I, I0)
    np.testing.assert_array_equal(D, D0)


def test_sorted_corpus_forces_overflow_retry(om):
    # adversarial order: every later row beats every earlier row for every query -> the doubling schedule
    # overflows its candidate lists and the overflow-proof schedule must take over; result still exact
    # (values are split over two columns so that every stored number is bf16-exact: the bf16 candidate
    # stage is then exact and the only difficulty is the ordering)
    n, d = 60000, 64
    v = np.arange(n) // 4  # ascending scores with 4-way ties
    base = np.zeros((n, d), np.float32)
    base[:, 0], base[:, 1] = v // 128, v % 128
    q = np.zeros((3, d), np.float32)
    q[:, 0], q[:, 1] = [128, 256, 384], [1, 2, 3]
    idx = om.FlatIPIndex(d)
    idx.add(base)
    D, I = idx.search(q, 100)
    assert idx.stat("overflow_retries") >= 1
    D0, I0 = oracle.flat_ip_search(q, base, 100)
    np.testing.assert_array_equal(I, I0)
    np.testing.assert_array_equal(D, D0)
    idx.set_param("force_safe_rounds", 1)
    D, I = idx.search(q, 100)
    np.testing.assert_array_equal(I, I0)


def test_descending_corpus_needs_no_retry(om):
    # the opposite order: after the first round no later row ever beats the threshold (rounds without survivors);
    # the threshold must survive such rounds, otherwise the next round accepts every row and overflows
    n, d = 60000, 64
    v = (n - 1 - np.arange(n)) // 4
    base = np.zeros((n, d), np.float32)
    base[:, 0], base[:, 1] = v // 128, v % 128
    q = np.zeros((3, d), np.float32)
    q[:, 0], q[:, 1] = [128, 256, 384], [1, 2, 3]
    idx = om.FlatIPIndex(d)
    idx.add(base)
    D, I = idx.search(q, 100)
    assert idx.stat("overflow_retries") == 0
    D0, I0 = oracle.flat_ip_search(q, base, 100)
    np.testing.assert_array_equal(I, I0)
    np.testing.assert_array_equal(D, D0)


def _eps_check(q, x, D, I, k, rel=2e-5):
    """Every returned (id, score) must be a valid top-k answer up to eps-ties: the float64 score of the
    r-th returned id equals the r-th best float64 score within eps, and the returned fp32 score equals the
    float64 score of that id within eps.  eps = rel * |q| * |x|_max (fp32 summation-order noise)."""
    s = q.astype(np.float64) @ x.astype(np.float64).T
    best = -np.sort(-s, axis=1)[:, :k]
    eps = rel * np.linalg.norm(q, axis=1, keepdims=True) * np.linalg.norm(x, axis=1).max()
    got = np.take_along_axis(s, I, axis=1)
    assert (np.abs(got - best) <= eps).all(), "returned ids are not an eps-valid top-k"
    assert (np.abs(D - got) <= eps).all(), "returned scores deviate from exact scores"
    assert (np.diff(D, axis=1) <= 0).all(), "scores not sorted descending"
    for r in range(I.shape[0]):
        assert len(set(I[r].tolist())) == k, "duplicate ids"


@pytest.mark.parametrize("n,d,nq,k", [(40000, 768, 150, 100), (100000, 768, 64, 1000), (30000, 1024, 33, 10)])
def test_gaussian_eps_aware(om, n, d, nq, k):
    rng = np.random.default_rng(11)
    x = rng.standard_normal((n, d), dtype=np.float32)
    q = rng.standard_normal((nq, d), dtype=np.float32)
    idx = om.FlatIPIndex(d)
    idx.add(x)
    D, I = idx.search(q, k)
    _eps_check(q, x, D, I, k)
    # device-resident entry point gives the same answer
    Dd, Id = idx.search_device(torch.from_numpy(q).cuda(), k)
    np.testing.assert_array_equal(Id.cpu().numpy(), I)


def test_normalized_embeddings(om):
    rng = np.random.default_rng(5)
    x = rng.standard_normal((50000, 768), dtype=np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    q = rng.standard_normal((40, 768), dtype=np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    idx = om.FlatIPIndex(768)
    idx.add(x)
    D, I = idx.search(q, 100)
    _eps_check(q, x, D, I, 100)


def test_sharded_merge_matches_unsharded(om):
    # single-GPU "logical shards": 4 indexes over contiguous row ranges, merged through om_topk_merge_n.  This is the
    # single-GPU check of merge_kernel, the merge step of the row-sharded search: a world-size-1 group never merges.
    rng = np.random.default_rng(2)
    x, q = _int_data(rng, 8000, 64, -3, 3), _int_data(rng, 21, 64, -3, 3)
    k = 50
    Dp, Ip = [], []
    for s in range(4):
        idx = om.FlatIPIndex(64)
        idx.add(x[s * 2000:(s + 1) * 2000])
        D, I = idx.search_device(torch.from_numpy(q).cuda(), k, id_offset=s * 2000)
        Dp.append(D); Ip.append(I)
    D, I = om.merge_topk_device(torch.stack(Dp), torch.stack(Ip), k)
    D0, I0 = oracle.flat_ip_search(q, x, k)
    np.testing.assert_array_equal(I.cpu().numpy(), I0)
    np.testing.assert_array_equal(D.cpu().numpy(), D0)
    # and against the oracle's own merge
    D1, I1 = oracle.merge_topk([(a.cpu().numpy(), b.cpu().numpy()) for a, b in zip(Dp, Ip)], k)
    np.testing.assert_array_equal(I.cpu().numpy(), I1)


def test_zero_copy_ingest(om):
    rng = np.random.default_rng(9)
    x, q = _int_data(rng, 1500, 128), _int_data(rng, 6, 128)
    idx = om.FlatIPIndex(128)
    rows = idx.reserve_rows(1500)
    rows.copy_(torch.from_numpy(x).cuda())
    idx.commit_rows(1500)
    D, I = idx.search(q, 30)
    D0, I0 = oracle.flat_ip_search(q, x, 30)
    np.testing.assert_array_equal(I, I0)


# ---------------------------------------------------------------------------------------------------------------------
# exactness certificate (csrc/search.cu certify_kernel) and its escalation levels
# ---------------------------------------------------------------------------------------------------------------------
def _recall(I, q, x, k):
    s = q.astype(np.float64) @ x.astype(np.float64).T
    truth = np.argsort(-s, axis=1, kind="stable")[:, :k]
    return np.mean([len(set(I[r].tolist()) & set(truth[r].tolist())) / k for r in range(I.shape[0])])


def _near_duplicate_corpus(rng, n, d, n_dup, eps):
    """n rows of which n_dup are copies of one vector perturbed by eps * N(0, 1): they collide in half precision
    (spacing 2^-10 relative) but stay distinct in fp32; the queries point at the cluster."""
    x = rng.standard_normal((n, d), dtype=np.float32)
    v = rng.standard_normal(d, dtype=np.float32)
    dup = rng.choice(n, n_dup, replace=False)
    x[dup] = v + eps * rng.standard_normal((n_dup, d), dtype=np.float32)
    q = (v + 0.1 * rng.standard_normal((5, d), dtype=np.float32)).astype(np.float32)
    return x, q, dup


def test_near_duplicate_cluster_is_exact(om):
    # 6000 near-duplicates, k = 1000: no candidate list of <= 4096 half-precision scores can contain the fp32 top-k
    # (the stage keeps the lowest row ids among colliding scores).  The certificate must notice and the exact fp32 scan
    # must answer; without the certificate (legacy mode) the answer is demonstrably wrong.
    rng = np.random.default_rng(2024)
    n, d, k = 40000, 128, 1000
    x, q, dup = _near_duplicate_corpus(rng, n, d, 6000, 1e-4)
    idx = om.FlatIPIndex(d)
    idx.add(x)
    D, I = idx.search(q, k)
    assert idx.stat("uncertified") == q.shape[0]
    assert idx.stat("exact_queries") == q.shape[0], "near-duplicate queries must fall through to the exact scan"
    _eps_check(q, x, D, I, k, rel=2e-6)  # d = 128: fp32 summation noise is ~1e-6 |q||x|, the cluster's score spread 1e-4
    assert _recall(I, q, x, k) > 0.99   # vs float64: only fp32 near-ties at the k-th rank may differ
    assert np.isin(I, dup).all(), "the top-k must lie inside the duplicate cluster"
    # the exact scan and the re-score share one summation order: exact_only reproduces the answer bit for bit
    idx.set_param("exact_only", 1)
    De, Ie = idx.search(q, k)
    np.testing.assert_array_equal(Ie, I)
    np.testing.assert_array_equal(De, D)
    idx.set_param("exact_only", 0)
    # teeth: the uncertified legacy path (top-k of the candidate stage) loses most of the true top-k here
    idx.set_param("certify", 0)
    _, Il = idx.search(q, k)
    assert _recall(Il, q, x, k) < 0.9
    idx.set_param("certify", 1)


def test_small_duplicate_cluster_resolved_by_wide_level(om):
    # 2500 near-duplicates: level 0 (k + 200 candidates) cannot be certified, the 4096-wide level holds the whole
    # cluster and can
    rng = np.random.default_rng(77)
    n, d, k = 60000, 128, 1000
    x, q, dup = _near_duplicate_corpus(rng, n, d, 2500, 1e-4)
    idx = om.FlatIPIndex(d)
    idx.add(x)
    D, I = idx.search(q, k)
    assert idx.stat("uncertified") == q.shape[0]
    assert idx.stat("exact_queries") == 0 and idx.stat("uncertified_wide") == 0
    _eps_check(q, x, D, I, k, rel=2e-6)
    idx.set_param("exact_only", 1)
    De, Ie = idx.search(q, k)
    np.testing.assert_array_equal(Ie, I)
    np.testing.assert_array_equal(De, D)


@pytest.mark.parametrize("normalise", [False, True])
def test_dense_scores_certified_at_first_level(om, normalise):
    # i.i.d. Gaussian rows (optionally L2-normalised: the densest realistic score distribution per unit of |q||x|):
    # the default slack must certify (nearly) every query at the first level, and the answer must equal the exact scan
    rng = np.random.default_rng(31)
    n, d, nq, k = 300000, 768, 96, 1000
    x = rng.standard_normal((n, d), dtype=np.float32)
    q = rng.standard_normal((nq, d), dtype=np.float32)
    if normalise:
        x /= np.linalg.norm(x, axis=1, keepdims=True)
        q /= np.linalg.norm(q, axis=1, keepdims=True)
    idx = om.FlatIPIndex(d)
    idx.add(torch.from_numpy(x).cuda())
    D, I = idx.search(q, k)
    assert idx.stat("uncertified") <= 2, "%d of %d queries uncertified at the default slack" % (idx.stat("uncertified"), nq)
    assert idx.stat("exact_queries") == 0
    _eps_check(q, x, D, I, k)
    idx.set_param("exact_only", 1)
    De, Ie = idx.search(q, k)
    np.testing.assert_array_equal(Ie, I)
    np.testing.assert_array_equal(De, D)


def test_slack_sweep_never_changes_the_answer(om):
    # the slack only moves work between the levels: whatever it is, the certified answer is the exact one
    rng = np.random.default_rng(8)
    n, d, nq, k = 120000, 256, 40, 100
    x = rng.standard_normal((n, d), dtype=np.float32)
    q = rng.standard_normal((nq, d), dtype=np.float32)
    idx = om.FlatIPIndex(d)
    idx.add(x)
    idx.set_param("exact_only", 1)
    De, Ie = idx.search(q, k)
    idx.set_param("exact_only", 0)
    _eps_check(q, x, De, Ie, k)
    seen = {}
    for slack in (0, 4, 32, 128, 1024):
        idx.set_param("rescore_slack", slack)
        D, I = idx.search(q, k)
        np.testing.assert_array_equal(I, Ie)
        np.testing.assert_array_equal(D, De)
        seen[slack] = idx.stat("uncertified")
    assert seen[0] == nq, "with no slack the k-th candidate is the floor itself: nothing can be certified"
    assert seen[1024] == 0 and seen[0] >= seen[32] >= seen[1024]


def test_nonfinite_and_out_of_range_values_fall_back(om):
    # values beyond the half range saturate in the scan copy; the measured error norm makes the certificate fail and the
    # exact scan answers (fail-safe, not fail-silent)
    rng = np.random.default_rng(4)
    x = rng.standard_normal((20000, 64), dtype=np.float32)
    x[123] *= 1.0e6
    q = rng.standard_normal((6, 64), dtype=np.float32)
    idx = om.FlatIPIndex(64)
    idx.add(x)
    D, I = idx.search(q, 50)
    assert idx.stat("exact_queries") == 6
    _eps_check(q, x, D, I, 50, rel=1e-4)


@pytest.mark.parametrize("d", [768, 1024])
def test_stage_error_model_holds_on_hardware(om, d):
    # The certificate's accumulation term assumes |stage - exact product sum of the half-rounded operands| <=
    # d * 2^-22 * |q_h||x_h|.  Measure it: debug_stage_scores makes D the candidate-stage (tensor-core) score.
    rng = np.random.default_rng(d)
    n, nq, k = 50000, 64, 256
    x = rng.standard_normal((n, d), dtype=np.float32)
    q = rng.standard_normal((nq, d), dtype=np.float32)
    idx = om.FlatIPIndex(d)
    idx.add(x)
    idx.set_param("debug_stage_scores", 1)
    Ds, Is = idx.search(q, k)
    idx.set_param("debug_stage_scores", 0)
    xh, qh = x.astype(np.float16).astype(np.float64), q.astype(np.float16).astype(np.float64)
    worst = 0.0
    for r in range(nq):
        B = xh[Is[r]] @ qh[r]
        bound = d * 2.0 ** -22 * np.linalg.norm(qh[r]) * np.linalg.norm(xh[Is[r]], axis=1)
        worst = max(worst, float(np.max(np.abs(Ds[r] - B) / bound)))
    assert worst < 0.25, "tensor-core accumulation error reaches %.3f of the modelled bound" % worst
    # and the full bound E(q) really covers |stage - fp32 score| for the rows we can see
    D, I = idx.search(q, k)
    xn = np.linalg.norm(x, axis=1).max()
    ex = np.linalg.norm(x - x.astype(np.float16).astype(np.float32), axis=1).max()
    for r in range(nq):
        hn, en = np.linalg.norm(qh[r]), np.linalg.norm(q[r] - q[r].astype(np.float16).astype(np.float32))
        E = hn * ex + en * xn + (d + 16) * 2.0 ** -22 * (hn + en) * (xn + ex)
        stage = dict(zip(Is[r].tolist(), Ds[r].tolist()))
        diff = [abs(stage[i] - s) for i, s in zip(I[r].tolist(), D[r].tolist()) if i in stage]
        assert max(diff) < E


def test_round_growth_settings_agree(om):
    # the round schedule (auto: x8 for small query batches, x2 for large ones) only changes how the corpus is swept
    rng = np.random.default_rng(44)
    x, q = _int_data(rng, 150000, 64, -6, 6), _int_data(rng, 19, 64, -6, 6)
    D0, I0 = oracle.flat_ip_search(q, x, 300)
    idx = om.FlatIPIndex(64)
    idx.add(x)
    rounds = {}
    for g in (0, 2, 3, 8):
        idx.set_param("round_growth", g)
        D, I = idx.search(q, 300)
        np.testing.assert_array_equal(I, I0)
        np.testing.assert_array_equal(D, D0)
        rounds[g] = idx.stat("rounds")
    assert rounds[0] == rounds[8] < rounds[3] < rounds[2]
    with pytest.raises(RuntimeError):
        idx.set_param("round_growth", 9)


def test_more_queries_than_one_chunk(om):
    # 20 000 queries: two query chunks (16 384 + 3 616) through scan / select / re-score / certificate, host and device paths
    rng = np.random.default_rng(99)
    x, q = _int_data(rng, 3000, 64, -7, 7), _int_data(rng, 20000, 64, -7, 7)
    idx = om.FlatIPIndex(64)
    idx.add(x)
    D, I = idx.search(q, 7)
    D0, I0 = oracle.flat_ip_search(q, x, 7)
    np.testing.assert_array_equal(I, I0)
    np.testing.assert_array_equal(D, D0)
    Dd, Id = idx.search_device(torch.from_numpy(q).cuda(), 7)
    np.testing.assert_array_equal(Id.cpu().numpy(), I0)
    # caller-owned output tensors
    out = (torch.empty((20000, 7), dtype=torch.float32, device="cuda"), torch.empty((20000, 7), dtype=torch.int64, device="cuda"))
    Do, Io = idx.search_device(torch.from_numpy(q).cuda(), 7, out=out)
    assert Do.data_ptr() == out[0].data_ptr() and torch.equal(Io, Id) and torch.equal(Do, Dd)
    with pytest.raises(ValueError):
        idx.search_device(torch.from_numpy(q).cuda(), 7, out=(out[0][:5], out[1][:5]))


@pytest.mark.parametrize("n,d,nq,k", [(70001, 72, 300, 50), (40000, 768, 129, 1000), (9000, 64, 257, 10),
                                       (300000, 128, 513, 100)])
def test_pair_scan_and_single_cta_scan_agree(om, n, d, nq, k):
    # > 128 queries: the scan GEMM runs on 2-CTA clusters (2 x 128 query rows per tile, corpus tile multicast to both);
    # "pair_scan" = 0 selects the single-CTA core.  Same candidates, same answer, bit for bit, and equal to the oracle.
    rng = np.random.default_rng(n + nq)
    x, q = _int_data(rng, n, d, -5, 5), _int_data(rng, nq, d, -5, 5)
    D0, I0 = oracle.flat_ip_search(q, x, k)
    idx = om.FlatIPIndex(d)
    idx.add(x)
    for pair in (1, 0, 1):
        idx.set_param("pair_scan", pair)
        D, I = idx.search(q, k)
        np.testing.assert_array_equal(I, I0)
        np.testing.assert_array_equal(D, D0)
    # Gaussian data: both cores accumulate the same fp16 products in the same order
    xg = rng.standard_normal((n, d)).astype(np.float32)
    qg = rng.standard_normal((nq, d)).astype(np.float32)
    idx = om.FlatIPIndex(d)
    idx.add(xg)
    Dp, Ip = idx.search(qg, k)
    idx.set_param("pair_scan", 0)
    Ds, Is = idx.search(qg, k)
    np.testing.assert_array_equal(Ip, Is)
    np.testing.assert_array_equal(Dp, Ds)
