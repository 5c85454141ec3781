"""CPU checks of the loss error model (oracle/loss_bound.py) that tests/test_loss_numerics_gpu.py judges the kernel by:
the float64 oracle matches the fp32 oracle and the reference's golden vectors; the bound admits a numpy emulation of
the kernel's arithmetic (so it does not fail on honest rounding) and rejects every modelled bug (so it is not vacuous)."""
import os

import numpy as np
import pytest
import torch

import oracle
from oracle import loss_bound as lb

F64 = torch.float64


def test_float64_oracle_matches_fp32_oracle_and_golden(golden_dir):
    z = np.load(os.path.join(golden_dir, "misc.npz"))
    for tag, target, red in (("a", None, "mean"), ("b", None, "mean"), ("c", "loss_c_target", "sum")):
        x, y = z[f"loss_{tag}_x"], z[f"loss_{tag}_y"]
        t = z[target] if target else None
        o = lb.loss64(torch.from_numpy(x), torch.from_numpy(y), None if t is None else torch.from_numpy(t), red)
        # the reference ran in fp32: its logits carry fp32 rounding, the float64 oracle's do not
        assert abs(float(o["loss"]) - float(z[f"loss_{tag}_loss"])) < 2e-6 * max(1.0, abs(float(o["loss"])))
        np.testing.assert_allclose(o["dX"].numpy(), z[f"loss_{tag}_dx"], rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(o["dY"].numpy(), z[f"loss_{tag}_dy"], rtol=1e-4, atol=1e-6)
        loss, dx, dy, s = oracle.contrastive_loss_fwd_bwd(x, y, t, red)
        assert abs(float(o["loss"]) - loss) < 1e-6 * max(1.0, abs(loss))
        np.testing.assert_allclose(o["S"].numpy(), s, rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(o["dX"].numpy(), dx, rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(o["dY"].numpy(), dy, rtol=1e-5, atol=1e-7)
        # G is dS of the same autograd graph
        np.testing.assert_allclose((o["G"] @ torch.from_numpy(y).to(F64)).numpy(), o["dX"].numpy(), rtol=1e-12,
                                   atol=1e-15)


def _bf16(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(torch.bfloat16).float().numpy()


def _blocked_matmul(a, b, kblocks):
    """fp32 a @ b with K cut into the given column ranges: each block's product in fp32, blocks added in order."""
    acc = np.zeros((a.shape[0], b.shape[1]), np.float32)
    for k0, k1 in kblocks:
        acc = (acc + a[:, k0:k1] @ b[k0:k1]).astype(np.float32)
    return acc


def _emulate(x, y, t, reduction, dq_split, bf16_grads):
    """numpy float32 restatement of loss_fused_kernel's arithmetic: 64-wide k blocks accumulated in fp32, fp32 expf /
    sums, G rounded to bf16, the dQ split partials added in slice order, the row losses summed in double."""
    f32 = np.float32
    xb, yb = _bf16(x), _bf16(y)
    nq, d = xb.shape
    n_p = yb.shape[0]
    rows = np.arange(nq)
    S = _blocked_matmul(xb, yb.T, [(k, min(d, k + 64)) for k in range(0, d, 64)])
    with np.errstate(invalid="ignore"):
        m = S.max(axis=1)
        e = np.exp((S - m[:, None]).astype(f32)).astype(f32)
        z = e.sum(axis=1, dtype=f32)
        row = ((m + np.log(z)).astype(f32) - S[rows, t]).astype(f32)
        w = f32(1.0 / nq) if reduction == "mean" else f32(1.0)
        loss = f32(row.astype(np.float64).sum() * np.float64(w))
        g = (e * (w / z).astype(f32)[:, None]).astype(f32)
        g[rows, t] = (g[rows, t] - w).astype(f32)
    G = _bf16(g)
    num_k = (n_p + 63) // 64
    kper = (num_k + dq_split - 1) // dq_split
    parts = [_blocked_matmul(G, yb, [(k, min(n_p, k + 64)) for k in range(s * kper * 64, min(n_p, (s + 1) * kper * 64), 64)])
             for s in range(dq_split)]
    dx = parts[0]
    for p in parts[1:]:
        dx = (dx + p).astype(f32)
    dy = _blocked_matmul(G.T, xb, [(k, min(nq, k + 64)) for k in range(0, nq, 64)])
    if bf16_grads:
        dx, dy = _bf16(dx), _bf16(dy)
    return {k: torch.from_numpy(np.asarray(v)).to(F64) for k, v in (("S", S), ("loss", loss), ("dX", dx), ("dY", dy))}


CASES = [(32, 256, 72, 2, "mean"), (60, 300, 37, 3, "sum"), (48, 768, 130, 4, "mean")]


@pytest.mark.parametrize("regime", lb.REGIMES)
@pytest.mark.parametrize("nq,n_p,d,split,reduction", CASES)
def test_bound_admits_kernel_emulation_and_rejects_mutants(regime, nq, n_p, d, split, reduction):
    x, y, info = lb.make_regime(regime, nq, n_p, d, seed=nq + d)
    xb, yb = lb.bf16_round(x), lb.bf16_round(y)
    o = lb.loss64(xb, yb, None, reduction)
    lb.premise(regime, o, info)
    t = o["target"].numpy()
    for bf16_grads in (False, True):
        got = _emulate(x.numpy(), y.numpy(), t, reduction, split, bf16_grads)
        b = lb.bounds(xb, yb, o, split, bf16_grads)
        r = lb.ratios(got, o, b)
        assert max(r.values()) <= 1.0, "%s: emulation outside the bound: %s" % (regime, r)
        if regime == "ties":
            assert torch.equal(got["S"], o["S"])
    b = lb.bounds(xb, yb, o, split)
    for name, mut in lb.mutants(xb, yb, o, reduction, split).items():
        r = lb.ratios(mut, o, b)
        assert max(r.values()) > 1.0, "%s: mutant %s accepted: %s" % (regime, name, r)
