"""Float64 oracle and elementwise error model of the fused contrastive loss (csrc/loss.cu).

TEST INFRASTRUCTURE ONLY (tests/test_loss_numerics_gpu.py, tests/test_loss_model_cpu.py).

``loss64`` restates ``src/openmatch/loss.py:7-15`` (``logits = x @ y.T``; ``F.cross_entropy(logits, target,
reduction)``; autograd) in float64 on the bf16-rounded inputs, which is what the tensor cores see.  It shares no code
with the kernel and runs on whichever device its inputs live (cuBLAS DGEMM on the GPU, BLAS on the CPU).

``bounds`` returns, for every element of S, the loss, dX and dY, a bound on |kernel - oracle| computed in float64 from
the same inputs.  u = 2^-24 is the fp32 unit roundoff, 2^-8 the bf16 one.  Each term:

Logits.  bf16 x bf16 products are exact in fp32, so only the fp32 accumulation of d products errs:
    |S_k - S64|_ij <= eps_ij = (d + 16) 2^-22 (|xb| @ |yb|^T)_ij
(4u per term instead of u: the tensor core's accumulation order and rounding are not specified; this is the model of
the search certificate).  delta_i = max_j eps_ij.

Softmax of perturbed logits.  With S' = S + D, |D_ij| <= eps_ij, p' / p = 1 / (p_j + (1 - p_j) a) where a is a
p-weighted mean of exp(D_k - D_j), k != j, so a lies in [e^-2delta, e^2delta].  Hence exactly (not to first order)
    |p'_ij - p_ij| <= p_ij (1 - p_ij) (e^{2 delta_i} - 1)
and the row loss l = lse(S) - S_t moves by log(p_t + sum_{k != t} p_k e^{D_k - D_t}), so
    |l' - l| <= min(2 delta_i, (1 - p_it)(e^{2 delta_i} - 1)).
The (1 - p) factors keep the bound tight at the target of a confident row, where p_t - 1 cancels.

fp32 softmax.  The kernel evaluates m = max (exact), expf(S - m) (argument rounded: relative error u |x| on e^x;
expf <= 2 ulp), z = sum of np terms (relative <= np u), log z (1 ulp), m + log z and - S_t (u each).  Relative to z:
sum_k (e_k / z)(|x_k| u + 2^-22) + np u <= (np / e + 4 + np) 2^-24 <= (2 np + 8) 2^-23 after generous rounding up;
log z <= log np adds 2^-23 log np, the two fp32 additions 2^-24 (|m| + |S_t| + |l|) <= 2^-23 (|m| + |S_t| + log np).
With |m| <= |m64| + delta:
    row_fp32_i = 2^-22 (|m64_i| + delta_i + |S64_it| + 2 np + 8 + 4 log np).
Loss = fp32(w_f * sum_i row_i) with the sum in double, w_f = fp32(1/nq):
    |dloss| <= w sum_i (row_logit_i + row_fp32_i) + 2^-22 |loss|.

G, the bf16 softmax gradient.  G_ij = bf16(expf(S - m) * fp32(w / z) - [j = t] w).  The fp32 chain (exp, z, the
quotient, the product) is relative (np + 16) 2^-23 of w p'_ij <= w p_ij e^{2 delta}; the subtraction at the target
rounds by u w; underflow of tiny p_ij costs at most w 2^-126.  Then the bf16 rounding, 2^-8 of the pre-rounding value:
    E_ij = w p_ij [(1 - p_ij)(e^{2 delta_i} - 1) + e^{2 delta_i} (np + 16) 2^-23],
    |dG_ij| <= bG_ij = E_ij + 2^-8 (|G64_ij| + E_ij) + w 2^-22.

Gradients.  dX = G @ yb, accumulated in fp32 over K = np (split into S slices whose partials are added in fp32):
    |ddX| <= bG @ |yb| + (np + 16 + S) 2^-22 ((|G64| + bG) @ |yb|) + np 2^-126 max|yb|
and dY the same with G^T, xb and K = nq, S = 1.  For bf16 inputs the autograd wrapper casts the gradient back to bf16:
add 2^-8 (|grad64| + bound).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

F64 = torch.float64
_TINY = 2.0 ** -126


def bf16_round(a: torch.Tensor) -> torch.Tensor:
    return a.to(torch.bfloat16).to(F64)


def default_target(nq: int, n_p: int, device=None) -> torch.Tensor:
    return torch.arange(nq, dtype=torch.int64, device=device) * (n_p // nq)


def loss64(xb: torch.Tensor, yb: torch.Tensor, target=None, reduction: str = "mean") -> dict:
    """float64 logits, loss and both gradients (autograd), plus softmax P and dS = G for the bounds."""
    xb = xb.to(F64).detach().requires_grad_()
    yb = yb.to(F64).detach().requires_grad_()
    nq, n_p = xb.shape[0], yb.shape[0]
    t = default_target(nq, n_p, xb.device) if target is None else target.to(device=xb.device, dtype=torch.int64)
    S = xb @ yb.T
    loss = F.cross_entropy(S, t, reduction=reduction)
    loss.backward()
    S = S.detach()
    w = 1.0 / nq if reduction == "mean" else 1.0
    P = torch.softmax(S, dim=1)
    G = P * w
    G[torch.arange(nq, device=S.device), t] -= w
    return {"S": S, "loss": loss.detach(), "dX": xb.grad, "dY": yb.grad, "P": P, "G": G, "target": t, "w": w}


def bounds(xb: torch.Tensor, yb: torch.Tensor, o: dict, dq_split: int = 1, bf16_grads: bool = False) -> dict:
    """Elementwise bounds on |kernel - oracle| for S, loss, dX, dY (see the module docstring)."""
    xb, yb = xb.to(F64), yb.to(F64)
    nq, d = xb.shape
    n_p = yb.shape[0]
    S, P, G, t, w = o["S"], o["P"], o["G"], o["target"], o["w"]
    rows = torch.arange(nq, device=S.device)
    xa, ya = xb.abs(), yb.abs()
    eps = (d + 16) * 2.0 ** -22 * (xa @ ya.T)
    delta = eps.amax(dim=1)
    e2 = torch.expm1(2 * delta)
    pt = P[rows, t]
    row_logit = torch.minimum(2 * delta, (1 - pt) * e2)
    row_fp32 = 2.0 ** -22 * (S.amax(dim=1).abs() + delta + S[rows, t].abs() + 2 * n_p + 8 + 4 * math.log(n_p))
    b_loss = w * (row_logit + row_fp32).sum() + 2.0 ** -22 * o["loss"].abs()
    E = w * P * ((1 - P) * e2[:, None] + torch.exp(2 * delta)[:, None] * (n_p + 16) * 2.0 ** -23)
    bG = E + 2.0 ** -8 * (G.abs() + E) + w * 2.0 ** -22
    Ga = G.abs() + bG
    b_dx = bG @ ya + (n_p + 16 + dq_split) * 2.0 ** -22 * (Ga @ ya) + n_p * _TINY * float(ya.max())
    b_dy = bG.T @ xa + (nq + 17) * 2.0 ** -22 * (Ga.T @ xa) + nq * _TINY * float(xa.max())
    if bf16_grads:
        b_dx = b_dx + 2.0 ** -8 * (o["dX"].abs() + b_dx)
        b_dy = b_dy + 2.0 ** -8 * (o["dY"].abs() + b_dy)
    return {"S": eps, "loss": b_loss, "dX": b_dx, "dY": b_dy}


def ratio(got: torch.Tensor, want: torch.Tensor, bound: torch.Tensor) -> float:
    """max |got - want| / bound over all elements.  A NaN in want must be matched by a NaN in got (and vice versa);
    a zero bound admits only an exact match.  Returns inf on any mismatch of that kind."""
    got = got.to(device=want.device, dtype=F64)
    if got.shape != want.shape:
        return math.inf
    nan_w, nan_g = torch.isnan(want), torch.isnan(got)
    if not torch.equal(nan_w, nan_g):
        return math.inf
    ok = ~nan_w
    err = (got - want).abs()[ok]
    b = bound.expand_as(want)[ok]
    if not torch.isfinite(err).all():
        return math.inf
    if err.numel() == 0:
        return 0.0
    r = torch.where(b > 0, err / torch.where(b > 0, b, torch.ones_like(b)),
                    torch.where(err == 0, torch.zeros_like(err), torch.full_like(err, math.inf)))
    return float(r.max())


def ratios(got: dict, o: dict, b: dict) -> dict:
    """max(err / bound) per output present in got (keys S, loss, dX, dY)."""
    return {k: ratio(got[k], o[k], b[k]) for k in ("S", "loss", "dX", "dY") if got.get(k) is not None}


# ------------------------------------------------------------------------------------------------------------------
# modelled kernel bugs, applied to the oracle's answer: the checker must reject each of them
# ------------------------------------------------------------------------------------------------------------------
def _kper(n_p: int, dq_split: int) -> int:
    num_k = (n_p + 63) // 64
    return (num_k + max(dq_split, 2) - 1) // max(dq_split, 2)


def _from_logits(S, xb, yb, t, reduction):
    Sg = S.detach().clone().requires_grad_()
    loss = F.cross_entropy(Sg, t, reduction=reduction)
    loss.backward()
    return loss.detach(), Sg.grad @ yb, Sg.grad.T @ xb


def mutants(xb: torch.Tensor, yb: torch.Tensor, o: dict, reduction: str = "mean", dq_split: int = 1) -> dict:
    """name -> {S, loss, dX, dY}: the oracle's answer with one modelled bug applied."""
    xb, yb = xb.to(F64), yb.to(F64)
    nq, d = xb.shape
    n_p = yb.shape[0]
    G, t, w = o["G"], o["target"], o["w"]
    base = {k: o[k].clone() for k in ("S", "loss", "dX", "dY")}
    out = {}
    # the target subtraction omitted in one row: G_it = w p_it instead of w (p_it - 1)
    i = nq // 2
    m = {k: v.clone() for k, v in base.items()}
    m["dX"][i] += w * yb[t[i]]
    m["dY"][t[i]] += w * xb[i]
    out["target_subtraction_omitted"] = m
    # the last K block (64 passages) of dQ dropped
    k0 = 64 * ((n_p - 1) // 64)
    m = {k: v.clone() for k, v in base.items()}
    m["dX"] -= G[:, k0:] @ yb[k0:]
    out["dq_last_k_block_dropped"] = m
    # one K slice of the split counted twice (slice 0; with no split, the first half of K)
    k1 = min(n_p, 64 * _kper(n_p, dq_split))
    m = {k: v.clone() for k, v in base.items()}
    m["dX"] += G[:, :k1] @ yb[:k1]
    out["dq_k_slice_counted_twice"] = m
    # one 64-wide k block of the first logit tile dropped; softmax, loss and gradients follow the wrong logits
    r, c, kb = min(nq, 128), min(n_p, 128), min(d, 64)
    S = base["S"].clone()
    S[:r, :c] -= xb[:r, :kb] @ yb[:c, :kb].T
    loss, dx, dy = _from_logits(S, xb, yb, t, reduction)
    out["logit_k_block_dropped"] = {"S": S, "loss": loss, "dX": dx, "dY": dy}
    # the last (ragged) N tile of dP zeroed
    n0 = 128 * ((d - 1) // 128)
    m = {k: v.clone() for k, v in base.items()}
    m["dY"][:, n0:] = 0
    out["dp_last_n_tile_zeroed"] = m
    return out


# ------------------------------------------------------------------------------------------------------------------
# input regimes (float32 host tensors; the kernel and the oracle both see their bf16 rounding)
# ------------------------------------------------------------------------------------------------------------------
REGIMES = ("random", "cosine", "temp_0.05", "temp_0.01", "large", "ties", "nan")


def _unit(a):
    return a / a.norm(dim=1, keepdim=True)


def make_regime(name: str, nq: int, n_p: int, d: int, seed: int = 0):
    """(x, y, info) for the default target i * (np // nq).  info["hard"]: rows given a hard negative."""
    g = torch.Generator().manual_seed(seed)
    tpq = n_p // nq
    t = torch.arange(nq) * tpq
    info = {}
    if name in ("random", "nan"):
        x = torch.randn(nq, d, generator=g) * 0.5
        y = torch.randn(n_p, d, generator=g) * 0.5
        if name == "nan":
            x[nq // 3, d // 2] = float("nan")
            info["nan_row"] = nq // 3
        return x, y, info
    if name == "ties":
        # small multiples of 1/4: every product and every fp32 partial sum is exact; passages i*tpq + 1 and + 2
        # (never a target when tpq >= 3) are duplicates
        x = torch.randint(-2, 3, (nq, d), generator=g).float() * 0.25
        y = torch.randint(-2, 3, (n_p, d), generator=g).float() * 0.25
        assert tpq >= 3
        y[t + 2] = y[t + 1]
        info["dups"] = (t + 1, t + 2)
        return x, y, info
    q = _unit(torch.randn(nq, d, generator=g))
    y = _unit(torch.randn(n_p, d, generator=g))
    y[t] = _unit(q + 0.5 * _unit(torch.randn(nq, d, generator=g)))
    x = q
    if name.startswith("temp_"):
        tau = float(name[5:])
        # 1 row in 16 and the last row: a hard negative closer than the positive, next to the target or, for the last
        # row, in the last passage.  Confident rows have gradients below fp32 resolution; these rows keep the first
        # K slice and the last K block of dQ significant, so that losing them is visible.
        hard = torch.unique(torch.cat([torch.arange(0, nq, 16), torch.tensor([nq - 1])]))
        hcol = t[hard] + 1
        hcol[-1] = n_p - 1
        y[hcol] = _unit(q[hard] + 0.3 * _unit(torch.randn(len(hard), d, generator=g)))
        info["hard"], info["hcol"] = hard, hcol
        x = q / tau
    elif name == "large":
        # un-normalised CLS reps share a large common direction c: query norms 20-60 along c, passages 10 c, with the
        # cosine construction orthogonal to c.  S = 10 r_i + 3 * 3 cos(...) is in the hundreds, the softmax stays
        # informative (the common part is constant per row)
        c = _unit(torch.randn(1, d, generator=g))
        perp = lambda a: _unit(a - (a @ c.T) * c)  # noqa: E731
        r = 20 + 40 * torch.rand(nq, 1, generator=g)
        r[0] = 60.0
        x = r * c + 3 * perp(q)
        y = 10 * c + 3 * perp(y)
    elif name != "cosine":
        raise ValueError(name)
    return x, y, info


def premise(name: str, o: dict, info: dict) -> None:
    """Asserts on the oracle's logits that the regime's statistics are really present."""
    S, P, t = o["S"], o["P"], o["target"]
    nq, n_p = S.shape
    rows = torch.arange(nq, device=S.device)
    if name == "cosine":
        assert float(P.amax()) <= math.e ** 2 / n_p, "cosine: max row probability %.3g > e^2/np" % float(P.amax())
    elif name.startswith("temp_"):
        pmax = P.amax(dim=1)
        assert float((pmax >= 0.99).double().mean()) >= 0.9, "peaked: fewer than 90% of rows with p_max >= 0.99"
        hard, hcol = info["hard"].to(S.device), info["hcol"].to(S.device)
        above = S[hard, hcol] > S[hard, t[hard]]
        row_loss = torch.logsumexp(S, 1) - S[rows, t]
        assert bool(above.any()) and float(row_loss[hard].max()) > 1.0, "peaked: no hard negative above its target"
    elif name == "large":
        assert float(S.abs().max()) >= 500, "large: max |S| %.1f < 500" % float(S.abs().max())
        assert float(P.amax()) < 0.999, "large: degenerate (one-hot) softmax"
    elif name == "nan":
        assert torch.isnan(o["loss"])
