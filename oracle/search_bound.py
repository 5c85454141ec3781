"""Float64 oracle of the search exactness certificate (csrc/search.cu ``certify_kernel``) and of the fp32 re-score.

TEST INFRASTRUCTURE ONLY (tests/test_search_model_cpu.py, tests/test_search_numerics_gpu.py).  numpy only; shares no
code with the kernels.

The search proves a query's top-k exact when ``s_k - tau > E(q)``: s_k is the k-th fp32 re-score, tau the stage score
of the last (kp-th) entry of the candidate list and, with x_h / q_h the fp16 scan operands,

    E(q) = 1.001 (a X_e + b X + (d + 16) 2^-22 (a + b)(X + X_e)),    a = |q_h|, b = |q - q_h|,
                                                                      X = max_r |x_r|, X_e = max_r |x_r - x_h,r|.

The first two terms bound |exact - B| (Cauchy-Schwarz), B being the exact sum of the fp16 products; the third bounds
|B - stage|, the tensor cores' fp32 accumulation, on the assumption that it errs by at most d 2^-23 of the running
magnitude (x2 head-room), which also has to cover the re-score's own rounding.

Re-score bound.  finalize_kernel sums in fp32: each lane runs an FMA chain of m = 4 ceil(d / 128) steps (float4 path,
d % 4 == 0) or ceil(d / 32) steps (scalar path), then a 5-level xor butterfly adds the 32 lane sums.  Every term goes
through at most m + 5 roundings, so with u = 2^-24 and gamma_n = n u / (1 - n u)
    |fp32 - exact| <= gamma_{m+5} sum_i |q_i x_i| + (d + 32) 2^-150
(the last term: gradual underflow, at most half the smallest subnormal per operation).  The float64 oracle's own
rounding, d 2^-52 sum_i |q_i x_i|, is added.

``pipeline_model`` is a CPU model of level 0 (stage score B, list = top kp by (B desc, row asc), tau = the list's
kp-th stage score, answer = top-k of the list by the float64 score) with the correct certificate or one of five
modelled bugs; ``search_model`` adds the escalation levels.  ``make_regime`` builds the input regimes that both the CPU
and the GPU tests run.
"""
from __future__ import annotations

import math

import numpy as np

NEG_FILL = np.float32(-3.4028234663852886e38)
K_MAX = 4096
VARIANTS = ("correct", "B1", "B2", "B3", "B4", "B5")
BUGS = {
    "B1": "drops the query-quantisation term b X of E",
    "B2": "drops the corpus-quantisation term a X_e of E",
    "B3": "takes the corpus norm maxima over the candidate list instead of the whole index",
    "B4": "sets tau = -inf whenever the list holds exactly kp entries",
    "B5": "uses query 0's norms a, b for the whole batch",
}


def f16_operand(x: np.ndarray) -> np.ndarray:
    """rows_to_f16_kernel's scan operand as float64: clamp to +-65504 (fmax / fmin: a NaN becomes -65504), then round
    to nearest even in fp16."""
    x = np.asarray(x, np.float32)
    c = np.fmin(np.fmax(x, np.float32(-65504.0)), np.float32(65504.0))
    return c.astype(np.float16).astype(np.float64)


def stage_exact(q: np.ndarray, x: np.ndarray) -> np.ndarray:
    """B [nq, n]: float64 sums of the products of the fp16 operands (each product is exact in float64)."""
    return f16_operand(q) @ f16_operand(x).T


def score64(q: np.ndarray, x: np.ndarray) -> np.ndarray:
    return np.asarray(q, np.float64) @ np.asarray(x, np.float64).T


def query_norms(q: np.ndarray):
    """(a, b) per query: |q_h| and |q - q_h|."""
    q64 = np.asarray(q, np.float64)
    qh = f16_operand(q)
    return np.linalg.norm(qh, axis=1), np.linalg.norm(q64 - qh, axis=1)


def corpus_maxima(x: np.ndarray):
    """(X, X_e): max |x_r| and max |x_r - x_h,r| over the rows."""
    if x.shape[0] == 0:
        return 0.0, 0.0
    x64 = np.asarray(x, np.float64)
    return float(np.linalg.norm(x64, axis=1).max()), float(np.linalg.norm(x64 - f16_operand(x), axis=1).max())


def acc_coef(d: int) -> float:
    return (d + 16) * 2.0 ** -22


def cert_E(q: np.ndarray, x: np.ndarray, terms: bool = False):
    """E(q) per query; terms=True: dict of the three terms (before the 1.001 factor) and E."""
    d = q.shape[1]
    a, b = query_norms(q)
    X, Xe = corpus_maxima(x)
    t = {"corpus_quant": a * Xe, "query_quant": b * X, "accumulation": acc_coef(d) * (a + b) * (X + Xe)}
    E = 1.001 * (t["corpus_quant"] + t["query_quant"] + t["accumulation"])
    if terms:
        t["E"] = E
        return t
    return E


def _gamma(n: int, u: float) -> float:
    return n * u / (1.0 - n * u)


def rescore_chain(d: int) -> int:
    """Roundings one product goes through in finalize_kernel: the lane's FMA chain plus the 5-level butterfly."""
    m = 4 * (-(-d // 128)) if d % 4 == 0 else -(-d // 32)
    return m + 5


def rescore_bound(q: np.ndarray, x: np.ndarray) -> np.ndarray:
    """beta [nq, n]: bound on |fp32 re-score - float64 oracle score| (module docstring)."""
    d = q.shape[1]
    A = np.abs(np.asarray(q, np.float64)) @ np.abs(np.asarray(x, np.float64)).T
    return (_gamma(rescore_chain(d), 2.0 ** -24) + d * 2.0 ** -52) * A + (d + 32) * 2.0 ** -150


def check_topk(q: np.ndarray, x: np.ndarray, D: np.ndarray, I: np.ndarray, k: int, id_offset: int = 0, s=None,
               beta=None) -> dict:
    """Rigorous validity of a search answer against the float64 scores s64 and the re-score bound beta:
      * |D[r] - s64(I[r])| <= beta(I[r]) for every returned row;
      * no unreturned row j has s64(j) - beta(j) > D[k-1] (it would have beaten the k-th answer);
      * D non-increasing, I ascending among equal D; ids unique and in range;
      * padding (-1, -FLT_MAX) exactly where k > n.
    s / beta: score64(q, x) / rescore_bound(q, x) when the caller already has them.  Returns {"rescore_ratio": max |D - s64| / beta}."""
    nq, n = q.shape[0], x.shape[0]
    kk = min(k, n)
    assert D.shape == (nq, k) and I.shape == (nq, k), "shape %s / %s" % (D.shape, I.shape)
    assert (I[:, kk:] == -1).all(), "padding ids must be -1"
    assert (D[:, kk:].view(np.uint32) == NEG_FILL.view(np.uint32)).all(), "padding scores must be -FLT_MAX"
    if kk == 0:
        return {"rescore_ratio": 0.0}
    ids = I[:, :kk] - id_offset
    assert ((ids >= 0) & (ids < n)).all(), "ids out of range"
    srt = np.sort(ids, axis=1)
    assert (np.diff(srt, axis=1) > 0).all(), "duplicate ids"
    s = score64(q, x) if s is None else s
    beta = rescore_bound(q, x) if beta is None else beta
    got = np.take_along_axis(s, ids, 1)
    bt = np.take_along_axis(beta, ids, 1)
    Dk = D[:, :kk].astype(np.float64)
    err = np.abs(Dk - got)
    assert (err <= bt).all(), "returned score off its float64 score by %.3g x the re-score bound" % float((err / bt).max())
    dd = np.diff(Dk, axis=1)
    assert (dd <= 0).all(), "scores not non-increasing"
    tie = dd == 0
    assert (np.diff(ids, axis=1)[tie] > 0).all(), "ids not ascending among equal scores"
    if kk < n:
        lower = s - beta
        np.put_along_axis(lower, ids, -np.inf, 1)
        best_out = lower.max(axis=1)
        bad = np.flatnonzero(best_out > Dk[:, -1])
        assert bad.size == 0, "query %d: an unreturned row beats the k-th answer by %.3g" % (
            bad[0], best_out[bad[0]] - Dk[bad[0], -1])
    return {"rescore_ratio": float((err / bt).max())}


# ------------------------------------------------------------------------------------------------------------------
# CPU model of the search levels
# ------------------------------------------------------------------------------------------------------------------
def _order(score: np.ndarray, rows: np.ndarray) -> np.ndarray:
    """Positions sorting one query's (score desc, row asc)."""
    return np.lexsort((rows, -score))


def pipeline_model(q: np.ndarray, x: np.ndarray, k: int, kp: int, variant: str = "correct") -> dict:
    """One level of the search on the CPU.  Returns D (float32 of s64), I [nq, k], certified [nq] bool, tau, E and the
    list [nq, kp_eff].  As in the library, kp_eff = min(kp, n); the list then holds exactly kp_eff rows and tau, its
    kp_eff-th stage score, is finite."""
    assert variant in VARIANTS
    nq, d = q.shape
    n = x.shape[0]
    kpe = min(kp, n)
    B = stage_exact(q, x)
    s = score64(q, x)
    lst = np.argsort(-B, axis=1, kind="stable")[:, :kpe]  # (B desc, row asc)
    tau = np.take_along_axis(B, lst, 1)[:, -1]
    a, b = query_norms(q)
    X, Xe = corpus_maxima(x)
    X = np.full(nq, X)
    Xe = np.full(nq, Xe)
    if variant == "B3":
        x64 = np.asarray(x, np.float64)
        xn, en = np.linalg.norm(x64, axis=1), np.linalg.norm(x64 - f16_operand(x), axis=1)
        X, Xe = xn[lst].max(axis=1), en[lst].max(axis=1)
    if variant == "B5":
        a, b = np.full(nq, a[0]), np.full(nq, b[0])
    cq = 0.0 if variant == "B2" else a * Xe
    qq = 0.0 if variant == "B1" else b * X
    E = 1.001 * (cq + qq + acc_coef(d) * (a + b) * (X + Xe))
    if variant == "B4":
        tau = np.full(nq, -np.inf)
    D = np.full((nq, k), NEG_FILL, np.float32)
    I = np.full((nq, k), -1, np.int64)
    sk = np.full(nq, -np.inf)
    kk = min(k, kpe)
    for r in range(nq):
        rows = lst[r]
        o = rows[_order(s[r, rows], rows)][:kk]
        D[r, :kk] = s[r, o]
        I[r, :kk] = o
        if kk == k:
            sk[r] = s[r, o[-1]]
    certified = np.where(np.isneginf(tau), True, sk - tau > E)
    return {"D": D, "I": I, "certified": certified, "tau": tau, "E": E, "list": lst, "s": s}


def exact_topk(q: np.ndarray, x: np.ndarray, k: int):
    """Top-k by the float64 score, (score desc, row asc); D as float32."""
    nq, n = q.shape[0], x.shape[0]
    s = score64(q, x)
    D = np.full((nq, k), NEG_FILL, np.float32)
    I = np.full((nq, k), -1, np.int64)
    kk = min(k, n)
    rows = np.arange(n)
    for r in range(nq):
        o = _order(s[r], rows)[:kk]
        D[r, :kk] = s[r, o]
        I[r, :kk] = o
    return D, I


def search_model(q: np.ndarray, x: np.ndarray, k: int, slack: int | None = None, variant: str = "correct"):
    """The whole search: level 0 (k + slack candidates), level 1 (uncertified queries, 4096 candidates, when the
    corpus is larger than level 0's list), level 2 (still uncertified: exact).  Returns (D, I, stats)."""
    n = x.shape[0]
    slack = max(128, k // 5) if slack is None else slack
    kp0 = min(k + slack, K_MAX)
    L0 = pipeline_model(q, x, k, kp0, variant)
    D, I = L0["D"].copy(), L0["I"].copy()
    flag = np.flatnonzero(~L0["certified"])
    st = {"uncertified": int(flag.size), "uncertified_wide": 0, "exact_queries": 0}
    if flag.size and kp0 < K_MAX and n > kp0:
        L1 = pipeline_model(q[flag], x, k, K_MAX, variant)
        D[flag], I[flag] = L1["D"], L1["I"]
        flag = flag[~L1["certified"]]
    st["uncertified_wide"] = int(flag.size)
    if flag.size:
        D[flag], I[flag] = exact_topk(q[flag], x, k)
        st["exact_queries"] = int(flag.size)
    return D, I, st


def certified_wrong(q: np.ndarray, x: np.ndarray, k: int, kp: int, variant: str) -> list:
    """Queries that `variant` certifies with a wrong level-0 answer, as (query, margin, accumulation term): margin is
    how far the best row left out of the answer lies above the emitted k-th (float64 scores), the accumulation term
    (d + 16) 2^-22 |q_h| (|x_h,j| + |x_h,k-th|) how far the tensor cores' accumulation may move the two apart.  A
    margin beyond it means the same data would expose the bug on hardware as well."""
    m = pipeline_model(q, x, k, kp, variant)
    out = []
    if x.shape[0] <= k:
        return out
    a, _ = query_norms(q)
    hn = np.linalg.norm(f16_operand(x), axis=1)
    for r in np.flatnonzero(m["certified"]):
        s = m["s"][r].copy()
        kth = m["I"][r, -1]
        s_k = s[kth]
        s[m["I"][r]] = -np.inf
        j = int(np.argmax(s))
        margin = float(s[j] - s_k)
        if margin > 0 or (margin == 0 and j < kth):
            out.append((int(r), margin, float(acc_coef(q.shape[1]) * a[r] * (hn[j] + hn[kth]))))
    return out


# ------------------------------------------------------------------------------------------------------------------
# input regimes: make_regime(name, nq, n, d, k, seed) -> (x, q, premise, info); premise() asserts in float64 that the
# regime's statistics are present
# ------------------------------------------------------------------------------------------------------------------
REGIMES = ("gaussian", "anisotropic", "coherent", "query_quant", "corpus_quant", "range_edges", "poisoned")
F16_MAX = 65504.0


def _f16(a) -> np.ndarray:
    return np.asarray(a, np.float32).astype(np.float16).astype(np.float32)


def default_slack(k: int) -> int:
    return max(128, k // 5)


def make_regime(name: str, nq: int, n: int, d: int, k: int = 10, seed: int = 0):
    rng = np.random.default_rng(seed)
    f32 = np.float32
    info = {}
    kp = min(k + default_slack(k), K_MAX)

    def no_premise():
        return None

    if name == "gaussian":
        return rng.standard_normal((n, d), dtype=f32), rng.standard_normal((nq, d), dtype=f32), no_premise, info

    if name == "anisotropic":
        # retrieval-like: a shared direction mu plus isotropic noise of variance 1/3 per unit, rows normalised, so the
        # expected cosine of two rows is 0.75 and every product of a score shares the sign of mu_i^2
        mu = rng.standard_normal(d)
        mu /= np.linalg.norm(mu)

        def emb(m):
            v = mu + math.sqrt(1.0 / 3.0) * rng.standard_normal((m, d)) / math.sqrt(d)
            return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(f32)

        x, q = emb(n), emb(nq)

        def premise():
            s = x[: min(n, 400)].astype(np.float64)
            c = s @ s.T
            med = float(np.median(c[np.triu_indices(c.shape[0], 1)]))
            assert med >= 0.6, "anisotropic: median pairwise cosine %.3f < 0.6" % med
            info["median_cosine"] = med

        return x, q, premise, info

    if name == "coherent":
        # fp16 values in [1, 2): both quantisation terms of E are exactly 0 and every product is positive, so the
        # accumulation grows monotonically and truncation errors never cancel
        x = _f16(rng.uniform(1.0, 2.0, (n, d)))
        q = _f16(rng.uniform(1.0, 2.0, (nq, d)))

        def premise():
            t = cert_E(q, x, terms=True)
            assert (t["corpus_quant"] == 0).all() and (t["query_quant"] == 0).all(), "coherent: operands not fp16-exact"
            assert (x > 0).all() and (q > 0).all(), "coherent: products of mixed sign"

        return x, q, premise, info

    if name == "query_quant":
        # Coarse queries: components of magnitude 1e-8 .. 8e-8, the bottom of the fp16 subnormals (spacing 2^-24 = 6e-8):
        # they round to 0 or +-2^-24, so the stage keeps only their signs and its ranking is mostly noise.  Every fourth
        # query (2, 6, 10, ...) spreads its components over the whole subnormal range instead, 1e-8 .. 6e-5, so that the
        # tensor cores multiply subnormals of every exponent.  Query 0 is clean: small multiples of 2^-24, with norms like
        # the coarse queries'.  The corpus is small integers (fp16-exact).
        x = rng.integers(-8, 9, (n, d)).astype(f32)
        spread = np.arange(nq) % 4 == 2
        lo = math.log(1e-8)
        hi = np.where(spread, math.log(6e-5), math.log(8e-8))[:, None]
        mag = np.exp(lo + (hi - lo) * rng.uniform(0.0, 1.0, (nq, d)))
        q = (mag * rng.choice([-1.0, 1.0], (nq, d))).astype(f32)
        q[0] = (rng.integers(-3, 4, d) * 2.0 ** -24).astype(f32)
        coarse = ~spread
        coarse[0] = False
        info["spread_queries"] = np.flatnonzero(spread)

        def premise():
            t = cert_E(q, x, terms=True)
            share = t["query_quant"][coarse] * 1.001 / t["E"][coarse]
            assert float(share.min()) >= 0.9, "query_quant: b X is only %.3f of E" % float(share.min())
            assert t["query_quant"][0] == 0, "query_quant: query 0 is not fp16-exact"
            if spread.any():
                qh = np.abs(f16_operand(q[spread]))
                sub = qh[(qh > 0) & (qh < 2.0 ** -14)]
                exps = np.unique(np.floor(np.log2(sub)))
                assert sub.size == qh.size - (qh == 0).sum() and exps.size == 10, \
                    "query_quant: the spread queries do not cover every subnormal exponent (%s)" % exps
            m = pipeline_model(q, x, k, kp)
            Dt, It = exact_topk(q, x, k)
            assert (m["I"] != It).any(axis=1).sum() >= 1, "query_quant: the stage list never misses a true top-k row"

        return x, q, premise, info

    if name == "corpus_quant":
        # One cluster of M rows v + t_j h, t_j = (j + 1/2) / M rising with the row id, h = 2^-11 (1 - 2^-10) in every
        # column: v is fp16 in [1, 2), where the half-ulp is 2^-11, so every copy rounds back to v and the copies tie at
        # the stage, which keeps the lowest row ids (the smallest t).  Every third query points at the cluster
        # (fp16-exact, positive, so q.h > 0: the true best copies are the last ones); the others are Gaussian over an
        # fp16-exact Gaussian background and are certified.
        M = max(4 * kp, 1000)
        v = _f16(rng.uniform(1.0, 2.0, d))
        h = np.float32(2.0 ** -11 * (1 - 2.0 ** -10))
        t = ((np.arange(M) + 0.5) / M).astype(f32)
        cl = (v[None, :] + t[:, None] * h).astype(f32)
        bg = _f16(2.0 * rng.standard_normal((n - M, d)))
        x = np.concatenate([bg, cl])
        q = _f16(rng.standard_normal((nq, d)))
        aim = np.arange(nq) % 3 == 0
        q[aim] = _f16(v[None, :] * (1 + 0.1 * rng.standard_normal((int(aim.sum()), d))))
        assert (q[aim] > 0).all()
        info["cluster_queries"] = np.flatnonzero(aim)
        info["cluster_rows"] = (n - M, n)

        def premise():
            assert (f16_operand(cl) == v[None, :]).all(), "corpus_quant: a copy does not round back to v"
            m = pipeline_model(q, x, k, kp)
            frac = 1.0 - float(m["certified"].mean())
            assert 0.1 <= frac <= 0.9, "corpus_quant: %.2f of the queries uncertified" % frac
            info["model_uncertified"] = frac

        return x, q, premise, info

    if name == "range_edges":
        # Gaussian rows with an offset column (x[:, 0] = 100, q[:, 0] = 1) and unit-variance scores, plus
        #   * an outlier row of 1e3 x the norm, pointing away from query 1;
        #   * a row of values at and beyond the half range: +-65504, +-65505, +-65519, +-65520 (which would round to
        #     inf without the clamp);
        #   * a row 1e5 e_c that saturates to 65504 e_c.  Query 1's component c is fp16-exact and chosen so that the
        #     row's stage score lies below query 1's candidate floor tau while its true score beats the k-th answer;
        #   * fp32-subnormal rows, all-zero rows, and exact duplicates of query 0's rows around rank k.
        assert d >= 16 and n >= 200
        x = rng.standard_normal((n, d), dtype=f32)
        x[:, 0] = 100.0
        q = (rng.standard_normal((nq, d)) / math.sqrt(d)).astype(f32)
        q[:, 0] = 1.0
        r_out, r_edge, r_sat = 3, n // 2, n - 5
        r_sub, r_zero = [7, n // 3], [11, n - 2]
        c_sat, edge_cols = d - 1, np.arange(1, 9)
        q[1, edge_cols] = 0.0
        q[1, c_sat] = 0.0
        x[r_edge] = 0.0
        x[r_edge, edge_cols] = [65504, -65504, 65505, -65505, 65519, -65519, 65520, -65520]
        x[:, c_sat] = 0.0
        x[r_sat] = 0.0
        x[r_sat, c_sat] = 1e5
        for r in r_sub:
            x[r] = (rng.standard_normal(d) * 1e-40).astype(f32)
        for r in r_zero:
            x[r] = 0.0
        base = x[r_out].copy()
        x[r_out] = (-1e3 * np.sign(float(q[1].astype(np.float64) @ base)) * base).astype(f32)
        # exact duplicates straddling query 0's rank k
        s0 = score64(q[:1], x)[0]
        o = _order(s0, np.arange(n))
        for sr, dr in zip(o[k - 2: k + 1], [20, n // 4, n - 10]):
            x[dr] = x[sr]
        # query 1's component c (no other row uses column c): fp16-exact e with 65504 e just below tau, so that
        # 1e5 e ~ 1.5 tau beats s_k by ~ 0.5 tau, more than the accumulation term of a row of norm 65504 at d <= 4096
        B = stage_exact(q[1:2], x)[0]
        tau = np.sort(B)[::-1][kp - 1]
        e = np.float16(0.999 * tau / F16_MAX)
        while float(e) * F16_MAX >= tau:
            e = np.nextafter(e, np.float16(0))
        q[1, c_sat] = np.float32(e)
        info.update(outlier=r_out, edge=r_edge, sat=r_sat, sleeper_query=1)

        def premise():
            s1 = score64(q[1:2], x)[0]
            B1 = stage_exact(q[1:2], x)[0]
            tau1 = np.sort(B1)[::-1][kp - 1]
            sk = np.sort(np.delete(s1, r_sat))[::-1][k - 1]
            assert B1[r_sat] < tau1 and s1[r_sat] > sk, "range_edges: the saturating row is not a sleeper"
            assert np.isfinite(f16_operand(x)).all()
            assert (np.abs(x[r_sub]) < np.finfo(np.float32).tiny).all() and (x[r_sub] != 0).any()

        return x, q, premise, info

    if name == "poisoned":
        x = rng.standard_normal((n, d), dtype=f32)
        q = rng.standard_normal((nq + 3, d), dtype=f32)
        bad = np.array([nq // 5, nq // 2 + 1, nq + 2])
        q[bad[0], d // 3] = np.nan
        q[bad[1], 0], q[bad[1], d - 1] = np.inf, -np.inf
        q[bad[2], d // 2] = 1e5
        info["poisoned"] = bad
        return x, q, no_premise, info

    raise ValueError(name)
