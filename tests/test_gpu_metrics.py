"""H100: the native evaluation metrics (fdgs.metrics over csrc/metrics.cu) against the float64 restatement of
tests/metrics_ref.py, at the project's bar: |ours - f64| <= max(2 |torch fp32 - f64|, 2 fp32 ulps of the f64 value),
with the reference's op sequence in torch fp32 (cuDNN TF32 off) as the comparator.

Shapes: 176x176 (a 1x1 interior at the fifth scale), 177x255 (odd at every level), 800x800 and 1014x1352, B = 4 and 1.
Inputs: uniform noise pairs; y = 1 - x (negative contrast means: MS-SSIM = 0 after the relu); identical pairs; constant
planes (sigma = 0); a lego render against a perturbed copy (noise 0.01 plus a one-pixel shift: values near 1, where
E[x^2] - mu^2 cancels); a render outside [0, 1] with the clamp flag.
Also: the per-view SSIM agrees with fdgs.loss.ssim (the training loss's fp32 evaluation of the same expression);
results are bit-identical run to run and between a batch and single-view calls (outputs and accumulator);
image_metrics and MetricAccumulator.add never synchronise the host."""
import numpy as np
import pytest
import torch

import metrics_ref as M

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPES = {"176": (4, 176, 176), "177x255": (4, 177, 255), "800": (1, 800, 800), "1014x1352": (1, 1014, 1352)}
KINDS = ("noise", "inverse", "identical", "constant", "lego_near", "lego_clamp")
NAMES = ("l1", "psnr", "ssim", "msssim")


def _lego_renders(B, H, W, seed=0):
    import lego
    from lego import LegoModel, lego_render, lego_setup
    cams, init, _ = lego_setup(20_000, W, H, seed=seed)
    with torch.no_grad():
        m = LegoModel({k: v.to(DEV) for k, v in init.items()})
        return torch.stack([lego_render(m, cams[b % len(cams)].to(DEV), "ours").clone() for b in range(B)])


def make_pair(kind, B, H, W, seed=0):
    """(x, y, clamp) float32 [B,3,H,W] on the GPU"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    if kind == "noise":
        return torch.rand(B, 3, H, W, generator=g, device=DEV), torch.rand(B, 3, H, W, generator=g, device=DEV), False
    if kind == "inverse":
        x = torch.rand(B, 3, H, W, generator=g, device=DEV)
        return x, 1 - x, False
    if kind == "identical":
        x = torch.rand(B, 3, H, W, generator=g, device=DEV)
        return x, x.clone(), False
    if kind == "constant":
        a = torch.tensor([0.3, 0.55, 0.8], device=DEV).view(1, 3, 1, 1).expand(B, 3, H, W).contiguous()
        return a, (0.9 - 0.5 * a).contiguous(), False
    r = _lego_renders(B, H, W, seed)
    if kind == "lego_near":
        y = torch.roll(r, 1, dims=-1) + 0.01 * torch.randn(r.shape, generator=g, device=DEV)
        return r.clamp(0, 1).contiguous(), y.clamp(0, 1).contiguous(), False
    y = r.clamp(0, 1).contiguous()
    x = (4.0 * r - 0.5 + 0.02 * torch.randn(r.shape, generator=g, device=DEV)).contiguous()
    assert float(x.min()) < 0 and float(x.max()) > 1
    return x, y, True


def ulp32(v):
    return np.spacing(np.abs(v).astype(np.float32)).astype(np.float64)


def check_bars(ours, f32, f64, label):
    ours, f32, f64 = (np.asarray(a, np.float64) for a in (ours, f32, f64))
    for j, name in enumerate(NAMES):
        o, t, r = ours[:, j], f32[:, j], f64[:, j]
        inf = np.isinf(r)
        assert np.array_equal(o[inf], r[inf]), (label, name, o, r)
        fin = ~inf
        err, terr = np.abs(o[fin] - r[fin]), np.abs(t[fin] - r[fin])
        bar = np.maximum(2 * terr, 2 * ulp32(r[fin]))
        assert np.all(err <= bar), (label, name, err, terr, r[fin])


def _f64(x, y, clamp):
    with M.no_tf32():
        return M.torch_metrics(x.double(), y.double(), clamp).cpu().numpy()


def _f32(x, y, clamp):
    with M.no_tf32():
        return M.torch_metrics(x, y, clamp).cpu().numpy()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_against_the_float64_restatement(shape, kind):
    from fdgs import loss, metrics
    B, H, W = SHAPES[shape]
    x, y, clamp = make_pair(kind, B, H, W)
    ours = metrics.image_metrics(x, y, clamp=clamp)
    assert ours.dtype == torch.float64 and ours.shape == (B, 4) and ours.is_cuda
    ours = ours.cpu().numpy()
    f64, f32 = _f64(x, y, clamp), _f32(x, y, clamp)
    print(shape, kind, "ours", ours[0], "f64", f64[0], "f32", f32[0])
    check_bars(ours, f32, f64, (shape, kind))
    if kind == "identical":
        assert np.all(ours[:, 0] == 0) and np.all(np.isposinf(ours[:, 1]))
        assert np.all(np.abs(ours[:, 2:] - 1) <= 2 * ulp32(np.ones(1)))
    if kind == "inverse":
        assert np.all(ours[:, 3] == 0)
    # the SSIM of the training loss (loss.cu: the same expression on fp32 moments, returned as 1 - (1 - ssim) in fp32)
    # on the same pair.  loss.cu's fp32 moments were up to 2.9 ulps from float64 on the near-identical 176x176 renders
    # (torch's fp32 convolutions: 0.7), hence 4 x the larger of torch fp32's distance and 1 ulp, plus the ulp of 1 - ssim
    xc = x.clamp(0, 1) if clamp else x
    for b in range(B):
        s = float(loss.ssim(xc[b], y[b]))
        bar = 4 * max(abs(f32[b, 2] - f64[b, 2]), ulp32(f64[b, 2])) + ulp32(1 - f64[b, 2])
        assert abs(ours[b, 2] - s) <= bar, (b, ours[b, 2], s, f64[b, 2], f32[b, 2])


def test_odd_shape_matches_numpy():
    """the numpy float64 restatement (separable, exact window) as a second float64 reference on 177x255"""
    from fdgs import metrics
    x, y, _ = make_pair("noise", 2, 177, 255, seed=5)
    ours = metrics.image_metrics(x, y).cpu().numpy()
    ref = M.numpy_metrics(x.cpu().numpy(), y.cpu().numpy())
    with M.no_tf32():
        f32 = M.torch_metrics(x, y).cpu().numpy()
    check_bars(ours, f32, ref, "numpy")


def test_bit_identical_run_to_run_and_batch_vs_single_views():
    from fdgs import metrics
    x, y, _ = make_pair("lego_clamp", 4, 1014, 1352, seed=3)
    a = metrics.image_metrics(x, y, clamp=True)
    b = metrics.image_metrics(x, y, clamp=True)
    assert torch.equal(a, b)
    single = torch.cat([metrics.image_metrics(x[i], y[i], clamp=True) for i in range(4)])
    assert torch.equal(a, single)
    acc_batch, acc_single = metrics.MetricAccumulator(), metrics.MetricAccumulator()
    acc_batch.add(x[:3], y[:3])
    acc_batch.add(x[3], y[3])
    for i in range(4):
        acc_single.add(x[i], y[i])
    assert torch.equal(acc_batch.sums, acc_single.sums)
    assert float(acc_single.sums[4]) == 4.0
    r = acc_single.result()
    ref = a.mean(0).tolist()
    for j in range(4):
        assert abs(r[j] - ref[j]) <= 1e-14 * max(1.0, abs(ref[j])), (j, r[j], ref[j])


def test_msssim_drop_in():
    from fdgs import metrics
    x, y, _ = make_pair("noise", 2, 200, 300, seed=6)
    v = metrics.msssim(x, y)
    assert isinstance(v, float)
    assert v == float(metrics.image_metrics(x, y)[:, 3].mean())
    with M.no_tf32():
        ref = float(M.torch_msssim(x.double(), y.double()).mean())
    assert abs(v - ref) <= 1e-6


def test_no_host_synchronisation():
    from fdgs import metrics
    x, y, _ = make_pair("noise", 2, 400, 500, seed=7)
    acc = metrics.MetricAccumulator()
    acc.add(x[0], y[0])                  # allocates the sums
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = metrics.image_metrics(x, y, clamp=True)
        for i in range(2):
            acc.add(x[i], y[i])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(out).all()
    assert float(acc.sums[4]) == 3.0
