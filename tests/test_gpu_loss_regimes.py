"""GPU (-m gpu): the fused L1 + SSIM loss (csrc/loss.cu, fdgs.loss) against the float64 restatement of
tests/loss_ref.py, in the regimes training reaches, with torch's fp32 evaluation of the reference's formula (cuDNN, TF32
off) as the yardstick:

  value, l1 and ssim terms   |ours - f64| <= max(2 |torch32 - f64|, 16 fp32 ulps of the value)
  gradient, relative L2      ||ours - f64|| <= max(2 ||torch32 - f64||, 1e-5 ||f64||)
  gradient, per pixel        |ours - f64| <= 2 |torch32 - f64| + 3e-5 max|grad|

The floors are what the kernel's fp32 arithmetic meets today: the value of near-identical textured renders is up to
~10 ulps from float64 where torch's is within one, and a few pixels per image (more in flat regions next to textured
ones) are up to ~1.3e-5 max|grad| further than twice torch's error; a 1x1 image's gradient is 6e-6 from float64.  The kernel before the difference form of
csrc/loss.cu failed the per-pixel bar on 10-40 % of the pixels of the near-identical regime.

Regimes, each asserting that it is reached: near-identical renders (x = gt + delta * noise, delta 1e-2 .. 1e-4, over
textured and smooth gt), flat regions at exactly 0 and 1 in both images (x == y there) and in one image only, renders
outside [0, 1], shapes below the 11-tap window and around the 32-pixel tile, C = 1, non-contiguous inputs, an upstream
gradient scale, and the two-call `l1_loss` / `ssim` form train.py uses."""
import numpy as np
import pytest
import torch

import loss_ref
from metrics_ref import no_tf32

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


# ---- inputs -----------------------------------------------------------------------------------------------------------
def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def textured(C, H, W, g):
    """sinusoids of a 7..23-pixel period plus 2 % noise, in [0, 1]"""
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    out = []
    for c in range(C):
        f = 2 * np.pi / (7 + 16 * torch.rand(4, generator=g, dtype=torch.float64))
        v = 0.5 + 0.1 * (torch.sin(f[0] * xx + f[1] * yy) + torch.sin(f[2] * xx - f[3] * yy + c))
        out.append(v + 0.02 * torch.randn(H, W, generator=g, dtype=torch.float64))
    return torch.stack(out).clamp(0, 1).float()


def smooth(C, H, W, g):
    """a ramp and one slow wave: the windowed variance stays far below C2"""
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H, dtype=torch.float64), torch.linspace(0, 1, W, dtype=torch.float64), indexing="ij")
    o = torch.rand(C, 1, 1, generator=g, dtype=torch.float64)
    return (0.2 + 0.3 * o + 0.2 * xx + 0.1 * torch.sin(3 * yy)).float()


def _b2(x, y):
    _, _, s11, s22, _ = loss_ref.moments(x.double(), y.double())
    return s11 + s22 + loss_ref.C2


# ---- the three evaluations and the bars ---------------------------------------------------------------------------------
def _ours(x, y, lam, gs=1.0, two_call=False):
    from fdgs import loss as L
    xr = x.detach().clone().requires_grad_(True) if x.is_contiguous() else x.detach().requires_grad_(True)
    if two_call:                          # train.py:115-117 with fdgs.loss's drop-ins
        l1 = L.l1_loss(xr, y)
        s = L.ssim(xr, y)
        loss = (1.0 - lam) * l1 + lam * (1.0 - s)
    else:
        loss, l1, s = L.l1_ssim_loss(xr, y, lam, return_terms=True)
    (gs * loss).backward()
    return loss.detach(), l1.detach(), s.detach(), xr.grad


def _ulp(v):
    v = abs(np.float32(v))
    return float(np.spacing(v)) if v > 0 else float(np.finfo(np.float32).smallest_subnormal)


def compare(x, y, lam, gs=1.0, two_call=False, label=""):
    xc, yc = x.contiguous(), y.contiguous()
    with no_tf32():
        t32 = loss_ref.loss_and_grad(xc, yc, lam, gs)
    f64 = loss_ref.loss_and_grad(xc.double(), yc.double(), lam, gs)
    ours = _ours(x, y, lam, gs, two_call)
    for i, name in enumerate(("loss", "l1", "ssim")):
        want = float(f64[i])
        eo, et = abs(float(ours[i]) - want), abs(float(t32[i]) - want)
        assert eo <= max(2 * et, 16 * _ulp(want)), (label, name, float(ours[i]), float(t32[i]), want, eo, et)
    go, gt, gw = ours[3].double(), t32[3].double(), f64[3]
    eo, et = (go - gw), (gt - gw)
    no, nt = float(eo.norm()), float(et.norm())
    assert no <= max(2 * nt, 1e-5 * float(gw.norm())), (label, "grad rel L2", no / max(float(gw.norm()), 1e-300), nt / max(float(gw.norm()), 1e-300))
    floor = 3e-5 * float(gw.abs().max())
    bad = eo.abs() > 2 * et.abs() + floor
    assert not bool(bad.any()), (label, "grad per pixel", int(bad.sum()), float((eo.abs() - 2 * et.abs()).max()), floor)
    return no / max(nt, 1e-300)


# ---- regimes ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("delta", [1e-2, 1e-3, 1e-4])
@pytest.mark.parametrize("gt_kind", ["textured", "smooth"])
@pytest.mark.parametrize("lam", [0.2, 1.0])
def test_near_identical(delta, gt_kind, lam):
    g = _gen(int(-np.log10(delta)) * 10 + len(gt_kind))
    C, H, W = 3, 176, 203
    gt = (textured if gt_kind == "textured" else smooth)(C, H, W, g)
    x = gt + delta * torch.randn(C, H, W, generator=g)
    x, gt = x.to(DEV), gt.to(DEV)
    med = float((x - gt).abs().median())
    assert 0.5 * delta <= med <= 0.9 * delta, med
    frac = float((_b2(x, gt) < 2 * loss_ref.C2).double().mean())
    if gt_kind == "smooth":
        assert frac > 0.8, frac           # B2 within a factor 2 of C2 (all but the zero-padded border)
    else:
        assert frac < 0.5, frac
    compare(x, gt, lam, label=(delta, gt_kind))


def test_near_identical_full_size():
    """a 1014 x 1352 render 1e-3 from its textured ground truth"""
    g = _gen(11)
    gt = textured(3, 1014, 1352, g)
    x = (gt + 1e-3 * torch.randn(gt.shape, generator=g)).to(DEV)
    compare(x, gt.to(DEV), 0.2)


def test_flat_and_saturated():
    """large regions at exactly 0 and exactly 1 in both images (x == y there: sign(0) = 0), and a band where only the
    render is flat"""
    g = _gen(3)
    C, H, W = 3, 150, 170
    y = textured(C, H, W, g)
    x = (y + 0.05 * torch.randn(C, H, W, generator=g)).clamp(0, 1)
    x[:, :50], y[:, :50] = 0.0, 0.0
    x[:, 50:100], y[:, 50:100] = 1.0, 1.0
    x[:, 100:, :40] = 1.0                 # only x flat (white background render over textured gt)
    x, y = x.to(DEV), y.to(DEV)
    both0 = float(((x == 0) & (y == 0)).double().mean())
    both1 = float(((x == 1) & (y == 1)).double().mean())
    only_x = float(((x == 1) & (y != 1)).double().mean())
    assert both0 > 0.3 and both1 > 0.3 and only_x > 0.05, (both0, both1, only_x)
    for lam in (0.0, 0.2, 1.0):
        compare(x, y, lam, label=lam)


def test_out_of_range():
    """unclamped renders in [-0.2, 1.5], as the rasterizer returns them"""
    g = _gen(4)
    C, H, W = 3, 131, 97
    y = textured(C, H, W, g)
    x = (y + 0.4 * torch.randn(C, H, W, generator=g)).clamp(-0.2, 1.5)
    x, y = x.to(DEV), y.to(DEV)
    assert float(x.min()) < -0.15 and float(x.max()) > 1.45
    for lam in (0.2, 1.0):
        compare(x, y, lam, label=lam)


SHAPES = [(1, 1, 1), (3, 1, 65), (1, 2, 33), (3, 5, 12), (1, 10, 37), (3, 11, 11), (1, 12, 64), (3, 31, 2), (1, 32, 32),
          (3, 33, 5), (1, 37, 63), (3, 63, 10), (1, 64, 31), (3, 65, 65), (1, 33, 37)]


@pytest.mark.parametrize("C,H,W", SHAPES)
def test_shapes(C, H, W):
    """below the window, one tile, and 1..5 pixels into the last tile (where the halo meets the zero padding)"""
    g = _gen(H * 100 + W)
    y = textured(C, H, W, g)
    x = (y + 0.1 * torch.randn(C, H, W, generator=g)).to(DEV)
    compare(x, y.to(DEV), 0.2, label=(C, H, W))
    compare(x, y.to(DEV), 1.0, label=(C, H, W))


@pytest.mark.parametrize("C,H,W", [(3, 1014, 1352), (3, 800, 800), (1, 800, 800)])
def test_full_size(C, H, W):
    g = _gen(H + C)
    y = textured(C, H, W, g)
    x = (y + 0.05 * torch.randn(C, H, W, generator=g)).to(DEV)
    compare(x, y.to(DEV), 0.2, label=(C, H, W))


def test_non_contiguous_inputs():
    """a slice x[:, :, 1:] and a channel view of a [B, 3, H, W] stack; the gradient lands in the base tensor"""
    from fdgs.loss import l1_ssim_loss
    g = _gen(6)
    y = textured(3, 70, 91, g).to(DEV)
    big = (textured(3, 70, 92, g) + 0.05 * torch.randn(3, 70, 92, generator=g)).to(DEV)
    x = big[:, :, 1:]
    assert not x.is_contiguous()
    compare(x, y, 0.2, label="slice")
    stack = (textured(4 * 3, 60, 50, g).view(4, 3, 60, 50)).to(DEV)
    gts = textured(4 * 3, 60, 50, g).view(4, 3, 60, 50).to(DEV)
    xv, yv = stack[:, 1], gts[:, 1]       # [B, H, W] views, stride 3 H W
    assert not xv.is_contiguous() and not yv.is_contiguous()
    compare(xv, yv, 0.2, label="channel view")
    base = stack.clone().requires_grad_(True)
    l1_ssim_loss(base[:, 1], gts[:, 1], 0.2).backward()
    _, _, _, gref = _ours(xv.contiguous(), yv.contiguous(), 0.2)
    assert torch.equal(base.grad[:, 1], gref) and float(base.grad[:, [0, 2]].abs().max()) == 0.0


@pytest.mark.parametrize("gs", [3.7, 0.25])
def test_grad_scale(gs):
    """a composite loss scales the upstream gradient: grad_scale != 1 reaches the kernel as a device scalar"""
    g = _gen(7)
    y = textured(3, 90, 120, g)
    x = (y + 0.02 * torch.randn(y.shape, generator=g)).to(DEV)
    compare(x, y.to(DEV), 0.2, gs=gs, label=gs)


@pytest.mark.parametrize("lam", [0.0, 0.2, 1.0])
def test_two_call_form(lam):
    """train.py:115-117 as written: Ll1 = l1_loss(image, gt); loss = (1 - l) Ll1 + l (1 - ssim(image, gt)), each term
    its own autograd node"""
    g = _gen(8)
    y = textured(3, 120, 77, g)
    x = (y + 0.01 * torch.randn(y.shape, generator=g)).to(DEV)
    compare(x, y.to(DEV), lam, two_call=True, label=lam)


def test_determinism():
    """gradients bit-identical run to run; the value, whose two double sums are formed by atomicAdd in CTA order,
    identical once rounded to fp32 (the double sums may differ in their last bits)"""
    g = _gen(9)
    y = textured(3, 1014, 1352, g)
    x = (y + 1e-3 * torch.randn(y.shape, generator=g)).to(DEV)
    y = y.to(DEV)
    runs = [_ours(x, y, 0.2) for _ in range(3)]
    for r in runs[1:]:
        assert torch.equal(r[3], runs[0][3])
        for i in range(3):
            assert torch.equal(r[i], runs[0][i])
