"""The reference's photometric loss of the training step restated in any dtype: l1_loss (utils/loss_utils.py:18-19) and
ssim (:39-64), combined as train.py:115-117, loss = (1 - lambda) * l1 + lambda * (1 - ssim), on [C,H,W] images.

  loss_terms       (loss, l1, ssim) through the reference's op sequence in torch: the 2D window of
                   metrics_ref._ref_window (the 1-D Gaussian in float32, or in float64 for float64 inputs, then the outer
                   product), F.conv2d with zero padding 5 over x, y, x*x, y*y, x*y.  At float32 this is the "torch fp32"
                   comparator (run it under metrics_ref.no_tf32); at float64 the precise evaluation.
  loss_and_grad    the value and d(grad_scale * loss)/dx by autograd, in the inputs' dtype.
  closed_form_grad numpy float64: the adjoint form csrc/loss.cu's header states,
                     dL/dx = (1 - lambda)/N sign(x - y) - lambda/N (G*a + 2 x (G*b) + y (G*c)),
                   with a = dS/dmu_x, b = dS/dE[xx], c = dS/dE[xy] per pixel (ground-truth moments fixed) and G the same
                   zero-padded Gaussian filter (it is symmetric, so it is its own adjoint).
  moments          the windowed moments mu_x, mu_y, sigma_xx, sigma_yy, sigma_xy, for the regime checks.
TEST INFRASTRUCTURE."""
import numpy as np
import torch
import torch.nn.functional as F

import metrics_ref

C1, C2 = metrics_ref.C1, metrics_ref.C2


def ssim(x, y):
    """utils/loss_utils.py:39-64 with size_average: the mean of the SSIM map of [C,H,W] images"""
    return metrics_ref.torch_ssim(x[None], y[None])[0]


def loss_terms(x, y, lam):
    """train.py:115-117: (loss, Ll1, ssim)"""
    l1 = torch.abs(x - y).mean()
    s = ssim(x, y)
    return (1.0 - lam) * l1 + lam * (1.0 - s), l1, s


def loss_and_grad(x, y, lam, grad_scale=1.0):
    """(loss, l1, ssim, d(grad_scale * loss)/dx), all in x's dtype"""
    xr = x.detach().clone().requires_grad_(True)
    loss, l1, s = loss_terms(xr, y.detach(), lam)
    (grad_scale * loss).backward()
    return loss.detach(), l1.detach(), s.detach(), xr.grad


def moments(x, y):
    """windowed moments of [C,H,W] images in x's dtype (zero padding 5): mu_x, mu_y, s_xx, s_yy, s_xy"""
    C = x.shape[0]
    w = metrics_ref._ref_window(C, x.dtype, x.device)
    f = lambda a: F.conv2d(a[None], w, padding=5, groups=C)[0]
    m1, m2 = f(x), f(y)
    return m1, m2, f(x * x) - m1 * m1, f(y * y) - m2 * m2, f(x * y) - m1 * m2


def closed_form_grad(x, y, lam, grad_scale=1.0):
    """numpy float64 d(grad_scale * loss)/dx of [C,H,W] images by the adjoint filter of (a, b, c)"""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    m1, m2, s11, s22, s12 = metrics_ref._moments(x, y, valid=False)
    A1, A2 = 2 * m1 * m2 + C1, 2 * s12 + C2
    B1, B2 = m1 * m1 + m2 * m2 + C1, s11 + s22 + C2
    inv = 1.0 / (B1 * B2)
    S = A1 * A2 * inv
    a = 2 * m2 * (A2 - A1) * inv + 2 * m1 * S * (1 / B2 - 1 / B1)
    b = -S / B2
    c = 2 * A1 * inv
    g = metrics_ref._gauss64()
    Ga, Gb, Gc = (metrics_ref._filter(t, g, valid=False) for t in (a, b, c))
    n = x.size
    return grad_scale * ((1 - lam) / n * np.sign(x - y) - lam / n * (Ga + 2 * x * Gb + y * Gc))
