"""Evaluation metrics of a test set (csrc/metrics.cu over the C-ABI): L1, PSNR, SSIM and MS-SSIM in float64 on the GPU.

Replaces the per-view evaluation of the reference's `training_report` (train.py:312-334): `l1_loss`, `psnr`
(utils/image_utils.py:17-19), `ssim` and torchmetrics' MS-SSIM on a host copy (`msssim`, utils/loss_utils.py:66-71).
Nothing here synchronises the host except `msssim` (a Python float, as the reference returns) and
`MetricAccumulator.result`.  CUDA only; there is no CPU fallback.
"""
from collections import namedtuple

import torch

import fdgs

MIN_SIZE = 176          # torchmetrics' MS-SSIM needs H // 16 > 10 and W // 16 > 10 (five scales of an 11x11 window)

Metrics = namedtuple("Metrics", ("l1", "psnr", "ssim", "msssim"))


def _batch(image, gt):
    if not isinstance(image, torch.Tensor) or not isinstance(gt, torch.Tensor):
        raise TypeError("fdgs.metrics: image and gt must be tensors")
    if image.shape != gt.shape:
        raise ValueError("fdgs.metrics: image %s and gt %s differ in shape" % (tuple(image.shape), tuple(gt.shape)))
    if image.dim() == 3:
        image, gt = image[None], gt[None]
    if image.dim() != 4:
        raise ValueError("fdgs.metrics: images must be [C,H,W] or [B,C,H,W], got %s" % (tuple(image.shape),))
    H, W = image.shape[-2:]
    if H < MIN_SIZE or W < MIN_SIZE:
        raise ValueError("fdgs.metrics: MS-SSIM needs H and W of at least %d, got %dx%d" % (MIN_SIZE, H, W))
    if not (image.is_cuda and gt.is_cuda):
        raise ValueError("fdgs.metrics: CUDA tensors only")
    return image.detach().float().contiguous(), gt.detach().float().contiguous()


def image_metrics(image, gt, clamp=False):
    """[B,4] float64 CUDA tensor of (l1, psnr, ssim, msssim) per view; image, gt: [C,H,W] or [B,C,H,W].
    clamp=True clamps `image` (not `gt`) to [0, 1] first, as train.py:318 clamps the render."""
    x, y = _batch(image, gt)
    return fdgs.ext().image_metrics(x, y, bool(clamp), torch.empty(0))


def msssim(rgb, gts):
    """reference: utils/loss_utils.py:68-71 -- MS-SSIM (torchmetrics 0.11.4 defaults, data_range 1) averaged over the
    batch, as a Python float."""
    return float(image_metrics(rgb, gts)[:, 3].mean())


class MetricAccumulator:
    """The four test-set means of training_report: `add` each rendered view (no host synchronisation), then `result`
    (one synchronisation).  The sums are float64 and added in view order, so a test set evaluated one view at a time
    or in batches gives the same bits."""

    def __init__(self, device=None):
        self.device = device
        self.sums = None

    def add(self, image, gt, clamp=True):
        x, y = _batch(image, gt)
        if self.sums is None:
            self.sums = torch.zeros(5, dtype=torch.float64, device=self.device if self.device is not None else x.device)
        return fdgs.ext().image_metrics(x, y, bool(clamp), self.sums)

    def result(self):
        """Metrics(l1, psnr, ssim, msssim): the means over every view added (NaN before the first)."""
        if self.sums is None:
            return Metrics(*([float("nan")] * 4))
        s = self.sums.tolist()
        return Metrics(*(v / s[4] for v in s[:4]))
