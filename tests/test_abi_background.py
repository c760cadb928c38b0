"""CPU: the per-pixel background image and sky-sampler entry points of the C-ABI are declared, exported and listed,
reject null arguments without touching a GPU, and the Python layer validates bg_image before any GPU work."""
import ctypes

import pytest
import torch

import helpers
from test_abi_and_host import _header_symbols

NEW = ("fdgs_forward_bg", "fdgs_backward_bg", "fdgs_sky_forward", "fdgs_sky_backward")


def test_new_symbols_declared_exported_and_listed(repo_root):
    import fdgs
    lib = fdgs.lib()
    for s in NEW:
        assert s in _header_symbols(repo_root)
        assert s in fdgs.ABI_SYMBOLS
        assert hasattr(lib, s)
    assert lib.fdgs_version() == 2


def test_new_entries_reject_null_arguments():
    import fdgs
    lib = fdgs.lib()
    for fn in (lib.fdgs_forward_bg, lib.fdgs_backward_bg, lib.fdgs_sky_forward, lib.fdgs_sky_backward):
        fn.restype = ctypes.c_int
    assert lib.fdgs_forward_bg(None, None, None, None, None, None, None, None, None, None) == 1
    assert b"null" in lib.fdgs_last_error()
    assert lib.fdgs_backward_bg(None, None, None, None) == 1
    assert lib.fdgs_sky_forward(None, None, None, None) == 1
    assert b"null" in lib.fdgs_last_error()
    assert lib.fdgs_sky_backward(None, None, None, None) == 1
    assert lib.fdgs_union_maps(ctypes.c_longlong(0), None, None, None, None, None) == 0   # a call that succeeds clears the error
    assert lib.fdgs_last_error() == b""


def test_extension_exposes_the_extended_bindings():
    import fdgs
    C = fdgs.ext()
    for name in ("rasterize_gaussians_ext", "rasterize_gaussians_backward_ext", "sky_forward", "sky_backward"):
        assert hasattr(C, name), name
    # the per-variant bindings the two extended entries replace
    for suffix in ("bg", "raw", "raw_bg", "backward_bg", "backward_raw", "backward_raw_bg", "backward_factors"):
        assert not hasattr(C, "rasterize_gaussians_" + suffix), suffix


def test_bg_image_is_validated_before_any_gpu_work():
    from gaussian_renderer import GaussianRasterizationSettings, GaussianRasterizer
    cfg, cam, sc, st = helpers.build("tiny")
    r = GaussianRasterizer(GaussianRasterizationSettings(**st))
    m2 = torch.zeros_like(sc.means3D)
    kw = dict(shs=sc.shs, ts=sc.ts, scales=sc.scales, scales_t=sc.scales_t, rotations=sc.rotations,
              rotations_r=sc.rotations_r)
    H, W = cfg["H"], cfg["W"]
    with pytest.raises(ValueError, match="shape"):
        r(sc.means3D, m2, sc.opacities, bg_image=torch.zeros(3, W, H), **kw)
    with pytest.raises(ValueError, match="float32"):
        r(sc.means3D, m2, sc.opacities, bg_image=torch.zeros(3, H, W, dtype=torch.float64), **kw)
    with pytest.raises(ValueError, match="shape"):
        r.forward_raw(sc.means3D, m2, sc.opacities, sc.shs[:, :1], sc.shs[:, 1:], sc.scales, sc.rotations,
                      ts=sc.ts, log_scales_t=sc.scales_t, rotations_r_raw=sc.rotations_r, bg_image=torch.zeros(1, H, W))
    with pytest.raises(TypeError):
        r(sc.means3D, m2, sc.opacities, bg_image=0.5, **kw)


def test_sky_rejects_a_malformed_environment_map():
    from fdgs.sky import sky_background
    with pytest.raises(ValueError, match="env_map"):
        sky_background(torch.zeros(4, 8, 8), None)
