"""CPU: tests/loss_ref.py, the float64 restatement the fused loss (csrc/loss.cu) is measured against, checked against
itself: autograd against the closed-form adjoint and against finite differences (gradcheck), at shapes below the
11-tap window and across 32-pixel tiles, with flat, saturated and out-of-range regions."""
import numpy as np
import pytest
import torch

import loss_ref


def _pair(C, H, W, seed, kind="noise"):
    g = torch.Generator().manual_seed(seed)
    y = torch.rand(C, H, W, generator=g, dtype=torch.float64)
    if kind == "noise":
        x = y + 0.1 * torch.randn(C, H, W, generator=g, dtype=torch.float64)
    elif kind == "near":
        x = y + 1e-3 * torch.randn(C, H, W, generator=g, dtype=torch.float64)
    elif kind == "flat":     # regions at exactly 0 and 1 in both images; a band where only x is flat
        x = y + 0.1 * torch.randn(C, H, W, generator=g, dtype=torch.float64)
        x[:, : H // 3], y[:, : H // 3] = 0.0, 0.0
        x[:, H // 3: 2 * H // 3], y[:, H // 3: 2 * H // 3] = 1.0, 1.0
        x[..., : W // 4] = 1.0
    else:                    # out of range, as the rasterizer returns it
        x = -0.2 + 1.7 * torch.rand(C, H, W, generator=g, dtype=torch.float64)
    return x, y


@pytest.mark.parametrize("C,H,W", [(1, 1, 1), (1, 2, 5), (3, 5, 11), (1, 10, 12), (3, 12, 31), (1, 33, 37), (3, 37, 65)])
@pytest.mark.parametrize("kind", ["noise", "near", "flat", "range"])
@pytest.mark.parametrize("lam", [0.0, 0.2, 1.0])
def test_autograd_equals_closed_form(C, H, W, kind, lam):
    x, y = _pair(C, H, W, H * 131 + W + len(kind), kind)
    _, _, _, g_auto = loss_ref.loss_and_grad(x, y, lam, grad_scale=3.0)
    g_closed = loss_ref.closed_form_grad(x.numpy(), y.numpy(), lam, grad_scale=3.0)
    scale = max(float(np.abs(g_closed).max()), 1e-300)
    assert np.abs(g_auto.numpy() - g_closed).max() <= 1e-12 * scale


@pytest.mark.parametrize("C,H,W", [(1, 3, 4), (3, 6, 7), (1, 12, 13)])
@pytest.mark.parametrize("lam", [0.2, 1.0])
def test_gradcheck(C, H, W, lam):
    g = torch.Generator().manual_seed(C * 100 + H)
    y = torch.rand(C, H, W, generator=g, dtype=torch.float64)
    # |x - y| >= 0.05 everywhere: the L1 term is differentiable at every pixel
    x = (y + (0.05 + 0.2 * torch.rand(C, H, W, generator=g, dtype=torch.float64))
         * torch.where(torch.rand(C, H, W, generator=g) < 0.5, -1.0, 1.0).double()).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda a: loss_ref.loss_terms(a, y, lam)[0], (x,), eps=1e-6, atol=1e-9, rtol=1e-6)


def test_identical_images():
    """x == y: l1 0, SSIM 1, and a zero gradient (SSIM is at its maximum; torch's sign(0) = 0)"""
    x, _ = _pair(3, 40, 45, 1, "range")
    loss, l1, s, g = loss_ref.loss_and_grad(x, x.clone(), 0.2)
    assert float(l1) == 0.0 and abs(float(s) - 1.0) < 1e-15 and abs(float(loss)) < 1e-15
    assert float(g.abs().max()) < 1e-15
    assert np.abs(loss_ref.closed_form_grad(x.numpy(), x.numpy(), 0.2)).max() < 1e-15


def test_moments_and_window():
    """the float64 window sums to 1 and is the outer product of one 1-D Gaussian; a constant image has mu = the
    constant away from the border and zero variance"""
    w = loss_ref.metrics_ref._ref_window(1, torch.float64, "cpu")[0, 0]
    assert abs(float(w.sum()) - 1.0) < 1e-15
    assert torch.allclose(w, torch.outer(w.sum(1), w.sum(0)), rtol=0, atol=1e-17)
    x = torch.full((1, 30, 30), 0.7, dtype=torch.float64)
    m1, m2, s11, s22, s12 = loss_ref.moments(x, x)
    assert float((m1[:, 5:-5, 5:-5] - 0.7).abs().max()) < 1e-15
    assert float(s11[:, 5:-5, 5:-5].abs().max()) < 1e-15


def test_float32_arm_is_close_to_float64():
    """the fp32 comparator is the same formula: within fp32 rounding of the float64 arm"""
    x, y = _pair(3, 64, 70, 7, "noise")
    l64, _, _, g64 = loss_ref.loss_and_grad(x, y, 0.2)
    l32, _, _, g32 = loss_ref.loss_and_grad(x.float(), y.float(), 0.2)
    assert abs(float(l32) - float(l64)) < 1e-6
    assert float((g32.double() - g64).norm() / g64.norm()) < 1e-4
