"""CPU checks of the search certificate's float64 model (oracle/search_bound.py), which
tests/test_search_numerics_gpu.py judges the kernels by: the model of the search levels agrees with the plain oracle;
check_topk admits a numpy emulation of the re-score's summation order (it does not fail on honest rounding) and rejects
broken answers (it is not vacuous); the correct certificate never certifies a wrong answer on any regime, and every
modelled bug does on a named regime, by a margin the hardware's accumulation error could not hide."""
import numpy as np
import pytest

import oracle
from oracle import search_bound as sb

# (n, d, nq) of each regime on the CPU
SIZES = {"gaussian": (3000, 64, 24), "anisotropic": (3000, 96, 24), "coherent": (3000, 64, 24),
         "query_quant": (3000, 64, 24), "corpus_quant": (4000, 64, 24), "range_edges": (3000, 64, 24),
         "poisoned": (3000, 64, 24)}
K = 10
KP = K + sb.default_slack(K)

# regime on which each modelled bug must certify a wrong answer
BUG_REGIME = {"B1": "query_quant", "B2": "corpus_quant", "B3": "range_edges", "B4": "corpus_quant", "B5": "query_quant"}


def _regime(name, k=K, seed=1):
    n, d, nq = SIZES[name]
    x, q, premise, info = sb.make_regime(name, nq, n, d, k=k, seed=seed)
    premise()
    if name == "poisoned":
        q = np.delete(q, info["poisoned"], axis=0)
    return x, q, info


def _emulate_finalize(q, x, rows):
    """numpy float32 restatement of finalize_kernel's re-score of `rows` for every query: lane l runs an FMA chain over
    float4 chunks l, l + 32, ... (scalar elements when d % 4 != 0), then the 32 lane sums meet in an xor butterfly.
    An FMA is emulated as the exact float64 product added in float64, then cast to float32.  That is a double rounding
    (float64 sum, then float32), off a true FMA by at most 2^-53 of the partial sum per operation, which the float64
    term d 2^-52 sum |q_i x_i| of the re-score bound covers at the d tested here."""
    nq, d = q.shape
    out = np.empty((nq, len(rows)), np.float32)
    step = 4 if d % 4 == 0 else 1
    for j, r in enumerate(rows):
        prod = q.astype(np.float64) * x[r].astype(np.float64)[None, :]
        lanes = np.zeros((nq, 32), np.float32)
        for c0 in range(0, d, 32 * step):
            for lane in range(32):
                base = c0 + lane * step
                for t in range(step):
                    if base + t < d:
                        lanes[:, lane] = (lanes[:, lane].astype(np.float64) + prod[:, base + t]).astype(np.float32)
        for o in (16, 8, 4, 2, 1):
            lanes = (lanes + lanes[:, np.arange(32) ^ o]).astype(np.float32)
        out[:, j] = lanes[:, 0]
    return out


def _emulated_answer(q, x, k):
    """Top-k by the emulated fp32 re-score over every row (the exact scan's answer), ties by row."""
    s = _emulate_finalize(q, x, np.arange(x.shape[0]))
    nq = q.shape[0]
    D = np.empty((nq, k), np.float32)
    I = np.empty((nq, k), np.int64)
    for r in range(nq):
        o = np.lexsort((np.arange(x.shape[0]), -s[r].astype(np.float64)))[:k]
        D[r], I[r] = s[r, o], o
    return D, I


def test_model_matches_oracle_on_integer_data():
    rng = np.random.default_rng(3)
    for n, d, nq, k in ((2000, 32, 9, 10), (700, 17, 5, 100), (300, 8, 4, 400)):
        x = rng.integers(-4, 5, (n, d)).astype(np.float32)
        q = rng.integers(-4, 5, (nq, d)).astype(np.float32)
        D0, I0 = oracle.flat_ip_search(q, x, k)
        D, I, st = sb.search_model(q, x, k)
        np.testing.assert_array_equal(I, I0)
        np.testing.assert_array_equal(D, D0)
        m = sb.pipeline_model(q, x, k, min(k + sb.default_slack(k), sb.K_MAX))
        c = m["certified"]
        np.testing.assert_array_equal(m["I"][c], I0[c])


@pytest.mark.parametrize("d", [64, 37])
def test_check_topk_admits_emulation_and_rejects_broken_answers(d):
    rng = np.random.default_rng(d)
    n, nq, k = 600, 6, 20
    x = rng.standard_normal((n, d), dtype=np.float32)
    q = rng.standard_normal((nq, d), dtype=np.float32)
    x[5] = x[400]  # an exact duplicate pair: tie order matters
    D, I = _emulated_answer(q, x, k)
    sb.check_topk(q, x, D, I, k)
    # k > n: padding
    Dp, Ip = _emulated_answer(q, x[:7], 7)
    Dp = np.concatenate([Dp, np.full((nq, 3), sb.NEG_FILL, np.float32)], 1)
    Ip = np.concatenate([Ip, np.full((nq, 3), -1, np.int64)], 1)
    sb.check_topk(q, x[:7], Dp, Ip, 10)
    s = sb.score64(q, x)

    def rejects(Db, Ib, xx=x, kk=k):
        with pytest.raises(AssertionError):
            sb.check_topk(q, xx, Db, Ib, kk)

    # the k-th row swapped for a better unreturned row: the row ranked k + 5
    Ib, Db = I.copy(), D.copy()
    order = np.argsort(-s[0])
    Ib[0, -1] = order[k + 5]
    Db[0, -1] = np.float32(s[0, order[k + 5]])
    rejects(Db, Ib)
    # fp16 stage scores reported as D
    B = sb.stage_exact(q, x)
    rejects(np.take_along_axis(B, I, 1).astype(np.float32), I)
    # broken tie order: equal scores with descending ids
    Ib, Db = I.copy(), D.copy()
    Db[0, 1] = Db[0, 0]
    Ib[0, 0], Ib[0, 1] = max(I[0, 0], I[0, 1]), min(I[0, 0], I[0, 1])
    rejects(Db, Ib)
    # a duplicate id
    Ib = I.copy()
    Ib[1, 3] = Ib[1, 2]
    rejects(D, Ib)
    # padding with the wrong score
    Dq = Dp.copy()
    Dq[0, -1] = -np.inf
    rejects(Dq, Ip, x[:7], 10)


@pytest.mark.parametrize("regime", sb.REGIMES)
def test_correct_certificate_never_certifies_a_wrong_answer(regime):
    x, q, _ = _regime(regime)
    for kp in (K, KP, 4 * KP):
        assert sb.certified_wrong(q, x, K, kp, "correct") == [], regime
    D, I, st = sb.search_model(q, x, K)
    sb.check_topk(q, x, D, I, K)
    De, Ie = sb.exact_topk(q, x, K)
    np.testing.assert_array_equal(I, Ie)


@pytest.mark.parametrize("bug", sorted(BUG_REGIME))
def test_every_modelled_bug_certifies_a_wrong_answer(bug):
    x, q, _ = _regime(BUG_REGIME[bug])
    wrong = sb.certified_wrong(q, x, K, KP, bug)
    caught = [w for w in wrong if w[1] > w[2]]
    assert caught, "%s (%s) certifies no wrong answer on %s beyond the accumulation term: %s" % (
        bug, sb.BUGS[bug], BUG_REGIME[bug], wrong[:3])
    if bug in ("B5",):
        assert all(r != 0 for r, _, _ in caught)  # query 0 is the one whose norms the bug borrows
