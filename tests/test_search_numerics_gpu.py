"""GPU: the search's exactness certificate and re-score against the float64 oracle (oracle/search_bound.py) at adversarial
data, on every scan path, and at the search limits.

Regimes (oracle.search_bound.make_regime; each asserts its premise in float64 first): Gaussian; anisotropic
retrieval-like embeddings (median cosine >= 0.6); coherent fp16-exact data in [1, 2) (E is only the accumulation term and
the accumulation grows monotonically); query-quantisation dominated (fp16-subnormal query components); a corpus
quantisation borderline (copies within half an fp16 ulp of a cluster centre); range edges (outlier rows, values at and
beyond the half range, fp32 subnormals, zero rows, exact duplicates at rank k); a batch with NaN / inf / 1e5 queries.
In every regime and on every scan path:
  * the default search equals the exact_only search bit for bit (what the certificate promises), on data where the
    regime's modelled certificate bugs would certify a wrong answer by more than the accumulation term;
  * check_topk accepts the answer (each score within the fp32 re-score bound of its float64 score, no unreturned row
    provably better than the k-th, tie order, ids, padding);
  * over the visible candidates (debug_stage_scores): |stage - B| <= (d + 16) 2^-22 |q_h||x_h|, the assumption behind
    the accumulation term, and |stage - fp32| <= E.
Each case prints one ``[numerics]`` line with the worst ratios and the escalation counts."""
import numpy as np
import pytest
import torch

import oracle
from oracle import search_bound as sb

pytestmark = pytest.mark.gpu

K = 10
NQ = 300
# (name, queries, index parameters): the single-CTA scan with growth 8, the wide scan under two cluster shapes, and
# query batches on the single-CTA scan
PATHS = [("single_g8", 64, {"round_growth": 8}),
         ("wide_2x1", NQ, {"scan_cluster_q": 2, "scan_cluster_x": 1}),
         ("wide_4x2", NQ, {"scan_cluster_q": 4, "scan_cluster_x": 2}),
         ("pair_off", NQ, {"pair_scan": 0})]
DEFAULTS = {"round_growth": 0, "pair_scan": 1, "scan_cluster_q": 0, "scan_cluster_x": 0, "certify": 1, "exact_only": 0,
            "debug_stage_scores": 0}
KP = K + sb.default_slack(K)
# modelled certificate bugs (oracle.search_bound.BUGS) that must certify a wrong answer on the very data each regime runs,
# beyond the accumulation term: the bit-equality with exact_only would then fail on hardware
NAMED_BUGS = {"query_quant": ("B1", "B5"), "corpus_quant": ("B2", "B4"), "range_edges": ("B3",)}
# (regime, d, n)
CASES = [("gaussian", 768, 20000),
         ("anisotropic", 384, 20000), ("anisotropic", 768, 20000), ("anisotropic", 4096, 6000),
         ("coherent", 768, 20000), ("coherent", 4096, 6000), ("coherent", 16384, 2500),
         ("query_quant", 768, 20000), ("corpus_quant", 64, 20000), ("range_edges", 768, 20000)]


@pytest.fixture(scope="module")
def om():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import index as om_index
    return om_index


def _set(idx, **params):
    for name, v in {**DEFAULTS, **params}.items():
        idx.set_param(name, v)


def _search(idx, q, k, **params):
    _set(idx, **params)
    D, I = idx.search(q, k)
    st = {s: idx.stat(s) for s in ("uncertified", "uncertified_wide", "exact_queries", "scan_cluster")}
    return D, I, st


def _bitwise_equal(a, b):
    np.testing.assert_array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


def _stage_ratios(q, x, Ds, Is, s, beta, E):
    """(max |stage - B| / ((d + 16) 2^-22 |q_h||x_h|), max (|stage - s64| + beta) / E) over the visible candidates."""
    d = q.shape[1]
    qh, xh = sb.f16_operand(q), sb.f16_operand(x[Is.ravel()]).reshape(Is.shape + (d,))
    B = np.einsum("qd,qkd->qk", qh, xh)
    Babs = np.einsum("qd,qkd->qk", np.abs(qh), np.abs(xh))
    bound = sb.acc_coef(d) * np.linalg.norm(qh, axis=1)[:, None] * np.linalg.norm(xh, axis=2) + 2 * d * 2.0 ** -53 * Babs
    err = np.abs(Ds.astype(np.float64) - B)
    r_acc = np.where(bound > 0, err / np.where(bound > 0, bound, 1), np.where(err == 0, 0.0, np.inf))
    s_rows = np.take_along_axis(s, Is, 1)
    b_rows = np.take_along_axis(beta, Is, 1)
    r_E = (np.abs(Ds.astype(np.float64) - s_rows) + b_rows) / E[:, None]
    return float(r_acc.max()), float(r_E.max())


@pytest.mark.parametrize("regime,d,n", CASES, ids=["%s-%d" % (r, d) for r, d, _ in CASES])
def test_regime_on_every_path(om, regime, d, n):
    x, q, premise, info = sb.make_regime(regime, NQ, n, d, k=K, seed=d)
    premise()
    s = sb.score64(q, x)
    beta = sb.rescore_bound(q, x)
    E = sb.cert_E(q, x)
    idx = om.FlatIPIndex(d)
    idx.add(x)
    stages, worst = {}, []
    caught = {}
    for path, nq, params in PATHS:
        qq = q[:nq]
        for bug in NAMED_BUGS.get(regime, ()):
            if (bug, nq) not in caught:
                caught[bug, nq] = [w for w in sb.certified_wrong(qq, x, K, KP, bug) if w[1] > w[2]]
            assert caught[bug, nq], "%s: modelled bug %s (%s) certifies no wrong answer on the first %d queries" % (
                regime, bug, sb.BUGS[bug], nq)
        D, I, st = _search(idx, qq, K, **params)
        if path.startswith("wide"):
            assert st["scan_cluster"] == 10 * params["scan_cluster_q"] + params["scan_cluster_x"]
        else:
            assert st["scan_cluster"] == 0
        De, Ie, _ = _search(idx, qq, K, exact_only=1, **params)
        np.testing.assert_array_equal(I, Ie)
        _bitwise_equal(D, De)
        rs = sb.check_topk(qq, x, D, I, K, s=s[:nq], beta=beta[:nq])
        Ds, Is, _ = _search(idx, qq, K, debug_stage_scores=1, **params)
        r_acc, r_E = _stage_ratios(qq, x, Ds, Is, s[:nq], beta[:nq], E[:nq])
        stages[path] = (Ds[:64], Is[:64])
        print("[numerics] regime=%s d=%d n=%d path=%s nq=%d |stage-B|/acc=%.4f |stage-fp32|/E=%.4f |D-s64|/beta=%.3f "
              "uncertified=%d uncertified_wide=%d exact_queries=%d" % (regime, d, n, path, nq, r_acc, r_E,
                                                                        rs["rescore_ratio"], st["uncertified"],
                                                                        st["uncertified_wide"], st["exact_queries"]))
        assert r_acc <= 1.0, "%s %s: tensor-core accumulation error %.3f x the modelled bound" % (regime, path, r_acc)
        assert r_E <= 1.0, "%s %s: |stage - fp32| reaches %.3f x E" % (regime, path, r_E)
        worst.append(r_acc)
        if regime == "query_quant":
            Dl, Il, _ = _search(idx, qq, K, certify=0, **params)
            assert (Il != Ie).any(), "query_quant: the uncertified stage answer equals the exact one"
        if regime == "corpus_quant":
            frac = st["uncertified"] / nq
            assert 0.1 <= frac <= 0.9, "corpus_quant: %.2f of the queries uncertified" % frac
    if regime in ("anisotropic", "coherent", "gaussian"):
        ref = stages["single_g8"]
        for path, (Ds, Is) in stages.items():
            np.testing.assert_array_equal(Is, ref[1], err_msg=path)
            _bitwise_equal(Ds, ref[0])


def test_poisoned_batch(om):
    n, d = 20000, 768
    x, q, _, info = sb.make_regime("poisoned", NQ, n, d, seed=7)
    bad = info["poisoned"]
    good = np.setdiff1d(np.arange(q.shape[0]), bad)
    idx = om.FlatIPIndex(d)
    idx.add(x)
    D, I, st = _search(idx, q, K)
    D0, I0, st0 = _search(idx, q[good], K)
    np.testing.assert_array_equal(I[good], I0)
    _bitwise_equal(D[good], D0)
    assert st["uncertified"] == st0["uncertified"] + 3
    De, Ie, _ = _search(idx, q, K, exact_only=1)
    np.testing.assert_array_equal(I[bad], Ie[bad])
    np.testing.assert_array_equal(D[bad], De[bad])  # NaN-aware: NaN equals NaN
    np.testing.assert_array_equal(I[good], Ie[good])
    _bitwise_equal(D[good], De[good])
    rs = sb.check_topk(q[good], x, D0, I0, K)
    print("[numerics] regime=poisoned d=%d n=%d path=auto nq=%d |D-s64|/beta=%.3f uncertified=%d uncertified_wide=%d "
          "exact_queries=%d (clean batch: uncertified=%d)" % (d, n, q.shape[0], rs["rescore_ratio"], st["uncertified"],
                                                              st["uncertified_wide"], st["exact_queries"],
                                                              st0["uncertified"]))


# ---------------------------------------------------------------------------------------------------------------------
# limits (integer data: every product and partial sum is exact, so ids and scores must equal the oracle bit for bit)
# ---------------------------------------------------------------------------------------------------------------------
def _int_data(rng, n, d, lo=-5, hi=5):
    return rng.integers(lo, hi + 1, size=(n, d)).astype(np.float32)


def _exact_vs_oracle(om, x, q, k, id_offset=0):
    idx = om.FlatIPIndex(x.shape[1])
    idx.add(x)
    D0, I0 = oracle.flat_ip_search(q, x, k)
    I0 = np.where(I0 >= 0, I0 + id_offset, -1)
    for exact_only in (0, 1):
        idx.set_param("exact_only", exact_only)
        D, I = idx.search(q, k, id_offset=id_offset)
        np.testing.assert_array_equal(I, I0)
        _bitwise_equal(D, D0)
    return idx


@pytest.mark.parametrize("nq", [5, 300])
@pytest.mark.parametrize("d", [1, 2, 3, 5, 7, 8, 9, 15, 16, 17])
def test_small_dims(om, d, nq):
    # dpad = 8 or 16: one partial k block; d % 4 != 0 takes finalize_kernel's scalar path
    rng = np.random.default_rng(d * 1000 + nq)
    _exact_vs_oracle(om, _int_data(rng, 5000, d), _int_data(rng, nq, d), K)


def test_max_dim(om):
    rng = np.random.default_rng(16384)
    _exact_vs_oracle(om, _int_data(rng, 700, 16384, -2, 2), _int_data(rng, 5, 16384, -2, 2), K)
    idx = om.FlatIPIndex(16385)
    idx.add(np.ones((10, 16385), np.float32))
    with pytest.raises(RuntimeError, match="16384"):
        idx.search(np.ones((2, 16385), np.float32), 5)


@pytest.mark.parametrize("nq", [7, 300])
@pytest.mark.parametrize("n", [4095, 4096, 4097, 30000])
@pytest.mark.parametrize("k", [4095, 4096])
def test_largest_k(om, k, n, nq):
    # k = 4096 leaves no room for slack: level 1 is skipped and an uncertified query goes straight to the exact scan
    rng = np.random.default_rng(k + n + nq)
    _exact_vs_oracle(om, _int_data(rng, n, 16, -3, 3), _int_data(rng, nq, 16, -3, 3), k)


def test_k_4096_near_duplicates(om):
    rng = np.random.default_rng(4096)
    n, d, k = 20000, 128, 4096
    x = rng.standard_normal((n, d), dtype=np.float32)
    v = rng.standard_normal(d, dtype=np.float32)
    dup = rng.choice(n, 6000, replace=False)
    x[dup] = v + 1e-4 * rng.standard_normal((6000, d), dtype=np.float32)
    q = (v + 0.1 * rng.standard_normal((5, d), dtype=np.float32)).astype(np.float32)
    idx = om.FlatIPIndex(d)
    idx.add(x)
    D, I = idx.search(q, k)
    assert idx.stat("uncertified") > 0
    assert idx.stat("exact_queries") == idx.stat("uncertified_wide") == idx.stat("uncertified")
    sb.check_topk(q, x, D, I, k)
    with pytest.raises(RuntimeError, match="4097"):
        idx.search(q, k + 1)


@pytest.mark.parametrize("nq", [5, 300])
def test_corpus_of_exactly_k_plus_slack_rows(om, nq):
    # the list holds every row, yet tau stays finite (the kp-th stage score)
    k = 100
    rng = np.random.default_rng(nq)
    _exact_vs_oracle(om, _int_data(rng, k + sb.default_slack(k), 64), _int_data(rng, nq, 64), k)
    xg = rng.standard_normal((k + sb.default_slack(k), 64), dtype=np.float32)
    qg = rng.standard_normal((nq, 64), dtype=np.float32)
    idx = om.FlatIPIndex(64)
    idx.add(xg)
    D, I = idx.search(qg, k)
    sb.check_topk(qg, xg, D, I, k)
    idx.set_param("exact_only", 1)
    De, Ie = idx.search(qg, k)
    np.testing.assert_array_equal(I, Ie)
    _bitwise_equal(D, De)


def test_k_above_n_in_a_query_batch(om):
    rng = np.random.default_rng(50)
    _exact_vs_oracle(om, _int_data(rng, 50, 72), _int_data(rng, 300, 72), 100)


def test_id_offset_beyond_32_bits(om):
    rng = np.random.default_rng(33)
    _exact_vs_oracle(om, _int_data(rng, 9000, 64), _int_data(rng, 300, 64), 50, id_offset=2 ** 33 + 5)


# ---------------------------------------------------------------------------------------------------------------------
# merge (om_topk_merge_n): bit-equal to oracle.merge_topk
# ---------------------------------------------------------------------------------------------------------------------
def _parts(rng, nparts, nq, k_in):
    """Per-part lists sorted (score desc, id asc) over disjoint increasing id ranges; small integer scores tie within
    and across parts; some parts end in -1 / -FLT_MAX padding."""
    span = 3 * k_in
    D = np.full((nparts, nq, k_in), sb.NEG_FILL, np.float32)
    I = np.full((nparts, nq, k_in), -1, np.int64)
    for p in range(nparts):
        for r in range(nq):
            m = k_in - (rng.integers(1, k_in // 3 + 2) if (p + r) % 3 == 0 else 0)
            ids = p * span + rng.choice(span, m, replace=False)
            sc = rng.integers(-40, 40, m).astype(np.float32)
            o = np.lexsort((ids, -sc.astype(np.float64)))
            D[p, r, :m], I[p, r, :m] = sc[o], ids[o]
    return D, I


@pytest.mark.parametrize("nparts,k_in,k_out", [(3, 4096, 4096), (8, 4096, 4096), (8, 2000, 2000), (17, 1000, 1000),
                                               (30, 300, 4000), (5, 300, 100), (4, 1000, 3000), (1, 8192, 8192)])
def test_merge_accepted(om, nparts, k_in, k_out):
    rng = np.random.default_rng(nparts * k_in + k_out)
    D, I = _parts(rng, nparts, 3, k_in)
    Dm, Im = om.merge_topk_device(torch.from_numpy(D).cuda(), torch.from_numpy(I).cuda(), k_out)
    D0, I0 = oracle.merge_topk([(D[p], I[p]) for p in range(nparts)], k_out)
    np.testing.assert_array_equal(Im.cpu().numpy(), I0)
    _bitwise_equal(Dm.cpu().numpy(), D0)


@pytest.mark.parametrize("nparts,k_in,k_out", [(2, 5000, 5000), (2, 8192, 100), (3, 4096, 8192)])
def test_merge_that_cannot_shrink_is_refused(om, nparts, k_in, k_out):
    # more than 8192 entries per query with k_in or k_out above 4096: a hierarchical level could not reduce the part count
    D = torch.zeros((nparts, 2, k_in), dtype=torch.float32, device="cuda")
    I = torch.arange(nparts * 2 * k_in, device="cuda").reshape(nparts, 2, k_in)
    with pytest.raises(RuntimeError, match="4096"):
        om.merge_topk_device(D, I, k_out)
