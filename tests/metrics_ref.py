"""Restatements of the evaluation metrics of the reference's training_report (train.py:312-334), per view of a
[B,C,H,W] batch: l1_loss (utils/loss_utils.py:18-19), psnr (utils/image_utils.py:17-19), ssim
(utils/loss_utils.py:34-64) and torchmetrics 0.11.4's MultiScaleStructuralSimilarityIndexMeasure(data_range=1.0)
(utils/loss_utils.py:66-71).

  numpy_metrics   the four numbers in numpy float64 (separable filters, exact Gaussian window)
  torch_metrics   the reference's op sequence in torch at a given dtype: 2D windows through F.conv2d (zero padding 5 for
                  SSIM; reflect pad 5, valid window, crop 5 for MS-SSIM), avg_pool2d between scales.  At float32 this is
                  the "torch fp32" comparator; run it with cuDNN TF32 off (`no_tf32`).
TEST INFRASTRUCTURE."""
import contextlib
import math

import numpy as np
import torch
import torch.nn.functional as F

BETAS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)
C1, C2 = 0.01 ** 2, 0.03 ** 2
MIN_SIZE = 176


def check_size(H, W):
    """torchmetrics' rule (_multiscale_ssim_update): H // 16 and W // 16 must exceed kernel_size - 1 = 10"""
    if H // 16 <= 10 or W // 16 <= 10:
        raise ValueError("MS-SSIM needs H and W of at least %d, got %dx%d" % (MIN_SIZE, H, W))


def pyramid_sizes(H, W, scales=5):
    out = []
    for _ in range(scales):
        out.append((H, W))
        H, W = H // 2, W // 2
    return out


# ---- numpy float64 --------------------------------------------------------------------------------------------------
def _gauss64():
    g = np.exp(-((np.arange(11) - 5.0) ** 2) / (2 * 1.5 ** 2))
    return g / g.sum()


def _filter(a, g, valid):
    """separable 11x11 correlation over the last two axes: zero padding 5 (same size) or valid windows only"""
    if not valid:
        a = np.pad(a, [(0, 0)] * (a.ndim - 2) + [(5, 5), (5, 5)])
    H, W = a.shape[-2] - 10, a.shape[-1] - 10
    h = sum(g[k] * a[..., :, k:k + W] for k in range(11))
    return sum(g[k] * h[..., k:k + H, :] for k in range(11))


def _moments(x, y, valid):
    g = _gauss64()
    m1, m2 = _filter(x, g, valid), _filter(y, g, valid)
    s11 = _filter(x * x, g, valid) - m1 * m1
    s22 = _filter(y * y, g, valid) - m2 * m2
    s12 = _filter(x * y, g, valid) - m1 * m2
    return m1, m2, s11, s22, s12


def numpy_metrics(x, y, clamp=False):
    """[B,4] float64: l1, psnr, ssim, msssim per view of x, y [B,C,H,W] (any float arrays)"""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    if clamp:
        x = np.clip(x, 0.0, 1.0)
    check_size(*x.shape[-2:])
    B = x.shape[0]
    d = x - y
    l1 = np.abs(d).reshape(B, -1).mean(1)
    with np.errstate(divide="ignore"):
        mse = (d * d).reshape(B, x.shape[1], -1).mean(2)
        psnr = (20 * np.log10(1.0 / np.sqrt(mse))).mean(1)
    m1, m2, s11, s22, s12 = _moments(x, y, valid=False)
    smap = ((2 * m1 * m2 + C1) * (2 * s12 + C2)) / ((m1 * m1 + m2 * m2 + C1) * (s11 + s22 + C2))
    ssim = smap.reshape(B, -1).mean(1)
    ms = np.ones(B)
    for s, beta in enumerate(BETAS):
        m1, m2, s11, s22, s12 = _moments(x, y, valid=True)
        upper, lower = 2 * s12 + C2, s11 + s22 + C2
        cs = (upper / lower).reshape(B, -1).mean(1)
        sim = (((2 * m1 * m2 + C1) * upper) / ((m1 * m1 + m2 * m2 + C1) * lower)).reshape(B, -1).mean(1)
        ms = ms * np.maximum(sim if s == len(BETAS) - 1 else cs, 0.0) ** beta
        H, W = x.shape[-2] // 2, x.shape[-1] // 2
        x = x[..., :2 * H, :2 * W].reshape(*x.shape[:-2], H, 2, W, 2).mean((-3, -1))
        y = y[..., :2 * H, :2 * W].reshape(*y.shape[:-2], H, 2, W, 2).mean((-3, -1))
    return np.stack([l1, psnr, ssim, ms], 1)


# ---- torch, the reference's op sequence -----------------------------------------------------------------------------
@contextlib.contextmanager
def no_tf32():
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _ref_window(C, dtype, device):
    """utils/loss_utils.py:24-32: the 1D Gaussian in float32 (float64 for a float64 restatement), outer product"""
    wdt = torch.float64 if dtype == torch.float64 else torch.float32
    g = torch.tensor([math.exp(-(i - 5) ** 2 / float(2 * 1.5 ** 2)) for i in range(11)], dtype=wdt)
    g = (g / g.sum()).unsqueeze(1)
    return g.mm(g.t()).to(dtype).expand(C, 1, 11, 11).contiguous().to(device)


def _tm_window(C, dtype, device):
    """torchmetrics 0.11.4 _gaussian_kernel_2d(channel, (11, 11), (1.5, 1.5))"""
    dist = torch.arange(-5.0, 6.0, 1.0, dtype=dtype, device=device)
    g = torch.exp(-torch.pow(dist / 1.5, 2) / 2)
    g = (g / g.sum()).unsqueeze(0)
    return torch.matmul(g.t(), g).expand(C, 1, 11, 11)


def _tm_ssim(x, y, w):
    """torchmetrics 0.11.4 _ssim_update(return_contrast_sensitivity=True), data_range 1: per-view means"""
    B, C = x.shape[:2]
    xp, yp = F.pad(x, (5, 5, 5, 5), mode="reflect"), F.pad(y, (5, 5, 5, 5), mode="reflect")
    out = F.conv2d(torch.cat((xp, yp, xp * xp, yp * yp, xp * yp)), w, groups=C)
    o = out.split(B)
    mu_xx, mu_yy, mu_xy = o[0].pow(2), o[1].pow(2), o[0] * o[1]
    sxx, syy, sxy = o[2] - mu_xx, o[3] - mu_yy, o[4] - mu_xy
    upper = 2 * sxy + C2
    lower = sxx + syy + C2
    sim = ((2 * mu_xy + C1) * upper) / ((mu_xx + mu_yy + C1) * lower)
    cs = upper / lower
    sim, cs = sim[..., 5:-5, 5:-5], cs[..., 5:-5, 5:-5]
    return sim.reshape(B, -1).mean(-1), cs.reshape(B, -1).mean(-1)


def torch_msssim(x, y):
    """[B] MS-SSIM per view (torchmetrics' _multiscale_ssim_update, normalize="relu")"""
    check_size(*x.shape[-2:])
    w = _tm_window(x.shape[1], x.dtype, x.device)
    mcs = []
    for _ in BETAS:
        sim, cs = _tm_ssim(x, y, w)
        mcs.append(torch.relu(cs))
        x, y = F.avg_pool2d(x, (2, 2)), F.avg_pool2d(y, (2, 2))
    mcs[-1] = torch.relu(sim)
    betas = torch.tensor(BETAS, device=x.device, dtype=x.dtype).view(-1, 1)
    return torch.prod(torch.stack(mcs) ** betas, 0)


def torch_ssim(x, y):
    """[B] the reference's ssim (utils/loss_utils.py:44-64) per view"""
    C = x.shape[1]
    w = _ref_window(C, x.dtype, x.device)
    mu1, mu2 = F.conv2d(x, w, padding=5, groups=C), F.conv2d(y, w, padding=5, groups=C)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    s1 = F.conv2d(x * x, w, padding=5, groups=C) - mu1_sq
    s2 = F.conv2d(y * y, w, padding=5, groups=C) - mu2_sq
    s12 = F.conv2d(x * y, w, padding=5, groups=C) - mu1_mu2
    m = ((2 * mu1_mu2 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s1 + s2 + C2))
    return m.reshape(x.shape[0], -1).mean(1)


def torch_metrics(x, y, clamp=False):
    """[B,4] (l1, psnr, ssim, msssim) in x's dtype, the reference's per-view expressions (train.py:318, 327-330)"""
    if clamp:
        x = torch.clamp(x, 0.0, 1.0)
    B = x.shape[0]
    l1 = (x - y).abs().reshape(B, -1).mean(1)
    mse = ((x - y) ** 2).reshape(B, x.shape[1], -1).mean(2)
    psnr = (20 * torch.log10(1.0 / torch.sqrt(mse))).mean(1)
    return torch.stack([l1, psnr, torch_ssim(x, y), torch_msssim(x, y)], 1)
