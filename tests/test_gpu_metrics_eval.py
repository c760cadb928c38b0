"""H100: a 20-view evaluation of the lego scene (tests/lego.py) through render() and fdgs.metrics.MetricAccumulator --
the loop INTEGRATION.md gives for training_report (train.py:312-334) -- against the reference's loop restated: torch on
the GPU for L1 / PSNR / SSIM (utils/loss_utils.py, utils/image_utils.py) and the float64 restatement for MS-SSIM.
Bars: the test-set means are within max(2 |torch fp32 - f64|, 2 fp32 ulps) of the float64 means."""
import math

import numpy as np
import pytest
import torch

import metrics_ref as M

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
VIEWS, W, H = 20, 800, 800


def _test_cameras():
    from fdgs import synth
    cams = []
    for k in range(VIEWS):     # a circle of radius 4 around the origin, as tests/lego.py places its training cameras
        ang = 2 * math.pi * k / VIEWS + 0.1
        eye = torch.tensor([4 * math.cos(ang), 0.3 * math.sin(3 * ang), 4 * math.sin(ang)])
        fwd = torch.nn.functional.normalize(-eye, dim=0)
        right = torch.nn.functional.normalize(torch.linalg.cross(torch.tensor([0.0, 1.0, 0.0]), fwd), dim=0)
        up = torch.linalg.cross(fwd, right)
        R = torch.stack([right, up, fwd], 1)
        cams.append(synth.make_camera(W, H, timestamp=k / VIEWS, focal_scale=1.1, R=R, T=-(R.t() @ eye)).to(DEV))
    return cams


def test_lego_evaluation_matches_the_restated_training_report():
    from fdgs.metrics import MetricAccumulator
    from gaussian_renderer import render
    from lego import LegoModel, _Pipe, lego_setup
    _, init, teacher = lego_setup(50_000, W, H, seed=11)
    cams = _test_cameras()
    bg = torch.zeros(3, device=DEV)
    with torch.no_grad():
        model = LegoModel({k: v.to(DEV) for k, v in init.items()})
        gts = [render(c, LegoModel({k: v.to(DEV) for k, v in teacher.items()}), _Pipe(), bg)["render"].clamp(0, 1)
               for c in cams]

        # the loop of INTEGRATION.md
        acc = MetricAccumulator()
        for gt_image, viewpoint in zip(gts, cams):
            render_pkg = render(viewpoint, model, _Pipe(), bg)
            image = torch.clamp(render_pkg["render"], 0.0, 1.0)
            acc.add(image, gt_image)
        l1_test, psnr_test, ssim_test, msssim_test = acc.result()

        # the reference's loop (train.py:312-334), restated; and the float64 restatement of every number
        ref32 = np.zeros(4)
        ref64 = np.zeros(4)
        with M.no_tf32():
            for gt_image, viewpoint in zip(gts, cams):
                image = torch.clamp(render(viewpoint, model, _Pipe(), bg)["render"], 0.0, 1.0)
                l1 = (image - gt_image).abs().mean().double()
                mse = ((image - gt_image) ** 2).view(image.shape[0], -1).mean(1, keepdim=True)
                psnr = (20 * torch.log10(1.0 / torch.sqrt(mse))).mean().double()
                ssim = M.torch_ssim(image[None], gt_image[None]).mean().double()
                ms = M.torch_msssim(image[None].double(), gt_image[None].double())[0]     # the float64 MS-SSIM
                ref32 += torch.stack([l1, psnr, ssim, ms]).cpu().numpy()
                ref64 += M.torch_metrics(image[None].double(), gt_image[None].double())[0].cpu().numpy()
    ref32 /= VIEWS
    ref64 /= VIEWS
    ours = np.array([l1_test, psnr_test, ssim_test, msssim_test])
    print("ours", ours, "reference loop", ref32, "float64", ref64)
    assert 0.2 < msssim_test < 0.999 and 5 < psnr_test < 60
    for j, name in enumerate(("l1", "psnr", "ssim", "msssim")):
        ulp2 = 2 * float(np.spacing(np.float32(abs(ref64[j]))))
        assert abs(ours[j] - ref64[j]) <= max(2 * abs(ref32[j] - ref64[j]), ulp2), (name, ours[j], ref32[j], ref64[j])
