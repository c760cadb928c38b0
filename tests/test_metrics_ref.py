"""CPU: the restatements of tests/metrics_ref.py agree with each other (numpy float64 vs the torch op sequence in
float64), give the known values on identical images, follow avg_pool2d's floor on odd sizes, enforce torchmetrics'
176-pixel rule, and -- where torchmetrics is installed -- match it."""
import numpy as np
import pytest
import torch

import metrics_ref as M


def _pair(B, C, H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, C, H, W, generator=g, dtype=torch.float64)
    y = (x + 0.1 * torch.randn(B, C, H, W, generator=g, dtype=torch.float64)).clamp(0, 1)
    return x, y


@pytest.mark.parametrize("shape", [(2, 3, 176, 176), (1, 3, 177, 255), (1, 1, 200, 190)])
def test_numpy_and_torch_float64_agree(shape):
    x, y = _pair(*shape)
    a = M.numpy_metrics(x.numpy(), y.numpy())
    b = M.torch_metrics(x, y).numpy()
    assert np.abs(a - b).max() <= 1e-12, np.abs(a - b).max()


def test_clamp_acts_on_the_render_only():
    x, y = _pair(1, 3, 180, 180, seed=1)
    x = x * 1.4 - 0.2
    a = M.numpy_metrics(x.numpy(), y.numpy(), clamp=True)
    b = M.numpy_metrics(x.clamp(0, 1).numpy(), y.numpy())
    assert np.array_equal(a, b)
    assert np.abs(M.torch_metrics(x, y, clamp=True).numpy() - a).max() <= 1e-12


def test_identical_images():
    x, _ = _pair(2, 3, 176, 200, seed=2)
    for v in (M.numpy_metrics(x.numpy(), x.numpy()), M.torch_metrics(x, x).numpy()):
        assert np.all(v[:, 0] == 0) and np.all(np.isposinf(v[:, 1]))
        assert np.abs(v[:, 2] - 1).max() < 1e-12 and np.abs(v[:, 3] - 1).max() < 1e-12


def test_pyramid_sizes_on_odd_shapes():
    assert M.pyramid_sizes(1014, 1352) == [(1014, 1352), (507, 676), (253, 338), (126, 169), (63, 84)]
    assert M.pyramid_sizes(177, 255) == [(177, 255), (88, 127), (44, 63), (22, 31), (11, 15)]
    assert M.pyramid_sizes(176, 176)[-1] == (11, 11)          # a 1x1 interior at the last scale
    x = torch.arange(177 * 255, dtype=torch.float64).reshape(1, 1, 177, 255)
    p = torch.nn.functional.avg_pool2d(x, (2, 2))
    assert tuple(p.shape[-2:]) == (88, 127)
    n = x.numpy()[..., :176, :254].reshape(1, 1, 88, 2, 127, 2).mean((-3, -1))
    assert np.abs(n - p.numpy()).max() == 0


def test_the_176_rule():
    for H, W in ((175, 300), (300, 175), (160, 160)):
        x = torch.zeros(1, 3, H, W, dtype=torch.float64)
        with pytest.raises(ValueError):
            M.numpy_metrics(x.numpy(), x.numpy())
        with pytest.raises(ValueError):
            M.torch_msssim(x, x)
    M.check_size(176, 176)


def test_matches_torchmetrics():
    tm = pytest.importorskip("torchmetrics")
    from torchmetrics import MultiScaleStructuralSimilarityIndexMeasure
    x, y = _pair(2, 3, 200, 240, seed=3)
    x, y = x.float(), y.float()
    ours = M.numpy_metrics(x.numpy(), y.numpy())[:, 3]
    for b in range(2):
        ref = float(MultiScaleStructuralSimilarityIndexMeasure(data_range=1.0)(x[b:b + 1], y[b:b + 1]))
        assert abs(ref - ours[b]) <= 1e-5, (tm.__version__, ref, ours[b])
    with pytest.raises(ValueError):
        MultiScaleStructuralSimilarityIndexMeasure(data_range=1.0)(torch.zeros(1, 3, 175, 200), torch.zeros(1, 3, 175, 200))
