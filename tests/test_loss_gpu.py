"""GPU parity: fused contrastive loss (C ABI) vs the CPU oracle (oracle/loss.py) and vs the golden vectors
from the reference's SimpleContrastiveLoss + autograd.  Tolerance (SURVEY 8c): |dloss| <= 1e-3 * max(1, |loss|)
against the fp32 oracle evaluated on bf16-rounded inputs; gradients rel-L2 <= 1e-2 (G is bf16 on the tensor
cores)."""
import os

import numpy as np
import pytest
import torch

import oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import loss
    return loss


def _bf16_round(a):
    return torch.from_numpy(np.asarray(a, np.float32)).to(torch.bfloat16).float().numpy()


def _rel(a, b):
    return np.linalg.norm(np.asarray(a, np.float64) - b) / max(np.linalg.norm(b), 1e-30)


@pytest.mark.parametrize("nq,n_p,d,dtype", [(64, 512, 768, torch.float32), (64, 512, 768, torch.bfloat16),
                                             (512, 4096, 768, torch.bfloat16), (5, 15, 24, torch.float32),
                                             (8, 64, 32, torch.float32), (130, 1040, 1024, torch.float32),
                                             # np > 4096 / np % 4 != 0: looped softmax; ragged K slices of dQ
                                             (96, 4100, 200, torch.float32), (33, 2052, 72, torch.float32),
                                             (40, 1001, 136, torch.float32),
                                             # bf16: a 72-byte row pitch is not 16-byte aligned, so the rows are
                                             # copied; a 400-byte pitch is, so they are read in place
                                             (12, 24, 36, torch.bfloat16), (130, 1040, 200, torch.bfloat16)])
def test_loss_and_grads_vs_oracle(L, nq, n_p, d, dtype):
    gen = torch.Generator().manual_seed(nq + d)
    x = (torch.randn(nq, d, generator=gen) * 0.5)
    y = (torch.randn(n_p, d, generator=gen) * 0.5)
    xr, yr = _bf16_round(x), _bf16_round(y)
    want_loss, want_dx, want_dy, want_s = oracle.contrastive_loss_fwd_bwd(xr, yr)
    xg = x.cuda().to(dtype).requires_grad_()
    yg = y.cuda().to(dtype).requires_grad_()
    loss, scores = L.fused_contrastive_loss(xg, yg, return_scores=True)
    loss.backward()
    assert abs(loss.item() - want_loss) <= 1e-3 * max(1.0, abs(want_loss))
    np.testing.assert_allclose(scores.cpu().numpy(), want_s, rtol=1e-4, atol=1e-3)
    assert _rel(xg.grad.float().cpu().numpy(), want_dx) <= 1e-2
    assert _rel(yg.grad.float().cpu().numpy(), want_dy) <= 1e-2


def test_gradients_are_run_to_run_identical(L):
    # dQ is reduced over K slices computed by different CTAs: the slice order of the sum is fixed
    gen = torch.Generator().manual_seed(9)
    x = (torch.randn(512, 768, generator=gen) * 0.5).cuda().to(torch.bfloat16)
    y = (torch.randn(4096, 768, generator=gen) * 0.5).cuda().to(torch.bfloat16)
    outs = []
    for _ in range(3):
        xg, yg = x.clone().requires_grad_(), y.clone().requires_grad_()
        loss = L.fused_contrastive_loss(xg, yg)
        loss.backward()
        outs.append((loss.item(), xg.grad.clone(), yg.grad.clone()))
    for o in outs[1:]:
        assert o[0] == outs[0][0]
        assert torch.equal(o[1], outs[0][1]) and torch.equal(o[2], outs[0][2])


def test_reference_golden(L, golden_dir):
    z = np.load(os.path.join(golden_dir, "misc.npz"))
    for tag in ("a", "b"):
        x = torch.from_numpy(z[f"loss_{tag}_x"]).cuda().requires_grad_()
        y = torch.from_numpy(z[f"loss_{tag}_y"]).cuda().requires_grad_()
        loss = L.SimpleContrastiveLoss()(x, y)
        loss.backward()
        # inputs are fp32 here; the kernel rounds them to bf16 for the tensor cores (reference under autocast
        # does the same) => 2e-2 relative on the loss value, 3e-2 on gradients
        assert abs(loss.item() - float(z[f"loss_{tag}_loss"])) <= 2e-2 * max(1.0, abs(float(z[f"loss_{tag}_loss"])))
        assert _rel(x.grad.cpu().numpy(), z[f"loss_{tag}_dx"]) <= 3e-2
        assert _rel(y.grad.cpu().numpy(), z[f"loss_{tag}_dy"]) <= 3e-2
    x = torch.from_numpy(z["loss_c_x"]).cuda().requires_grad_()
    y = torch.from_numpy(z["loss_c_y"]).cuda().requires_grad_()
    loss = L.SimpleContrastiveLoss()(x, y, target=torch.from_numpy(z["loss_c_target"]).cuda(), reduction="sum")
    loss.backward()
    want = oracle.contrastive_loss_fwd_bwd(_bf16_round(z["loss_c_x"]), _bf16_round(z["loss_c_y"]), z["loss_c_target"], "sum")
    assert abs(loss.item() - want[0]) <= 1e-3 * max(1.0, abs(want[0]))
    assert _rel(x.grad.cpu().numpy(), want[1]) <= 1e-2


def test_integer_logits_exact(L):
    # small integers: bf16 products and fp32 sums are exact => logits must match bit for bit
    rng = np.random.default_rng(0)
    x = rng.integers(-3, 4, (7, 64)).astype(np.float32)
    y = rng.integers(-3, 4, (21, 64)).astype(np.float32)
    _, scores = L.fused_contrastive_loss(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), return_scores=True)
    np.testing.assert_array_equal(scores.cpu().numpy(), x @ y.T)


def test_upstream_gradient_scaling_and_errors(L):
    x = torch.randn(4, 32, device="cuda", requires_grad=True)
    y = torch.randn(8, 32, device="cuda", requires_grad=True)
    (L.SimpleContrastiveLoss()(x, y) * 3.0).backward()
    g3 = x.grad.clone()
    x.grad = None
    L.SimpleContrastiveLoss()(x, y).backward()
    torch.testing.assert_close(g3, 3.0 * x.grad)
    with pytest.raises(RuntimeError):
        L.SimpleContrastiveLoss()(torch.randn(4, 32), torch.randn(8, 32))  # CPU tensors: no CPU path
    bad = L.SimpleContrastiveLoss()(x, y, target=torch.tensor([0, 1, 99, 2], device="cuda"))
    assert torch.isnan(bad)
    # no ignore_index: PyTorch's -100 is out of range like any other (DESIGN section 6)
    bad = L.SimpleContrastiveLoss()(x, y, target=torch.tensor([0, 1, -100, 2], device="cuda"))
    assert torch.isnan(bad)
