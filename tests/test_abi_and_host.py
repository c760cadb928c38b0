"""CPU: the C-ABI library loads and exports every symbol include/fdgs.h declares (no compute
calls without a GPU), and the host-side mirror of the reference interface behaves like the
reference's (argument validation, settings tuple, empty-tensor placeholders)."""
import ctypes
import os
import re

import pytest
import torch

import helpers


def _header_symbols(root):
    text = open(os.path.join(root, "include", "fdgs.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(fdgs_[a-z_0-9]+)\s*\(", text)) - {"fdgs_alloc_fn"})


def test_header_declares_expected_entry_points(repo_root):
    syms = _header_symbols(repo_root)
    for s in ("fdgs_forward", "fdgs_backward", "fdgs_mark_visible", "fdgs_last_error", "fdgs_version",
              "fdgs_geom_bytes", "fdgs_image_bytes", "fdgs_binning_bytes"):
        assert s in syms


def test_library_exports_every_declared_symbol(repo_root):
    import fdgs
    lib = fdgs.lib()   # raises FdgsNotBuilt if the CUDA library was not compiled: no fallback
    for s in _header_symbols(repo_root):
        assert hasattr(lib, s), "libfdgs.so does not export %s" % s
    assert set(_header_symbols(repo_root)) == set(fdgs.ABI_SYMBOLS)
    assert lib.fdgs_version() == 2
    assert lib.fdgs_last_error() == b""


def test_c_abi_rejects_null_arguments_without_touching_the_gpu():
    import fdgs
    lib = fdgs.lib()
    lib.fdgs_forward.restype = ctypes.c_int
    rc = lib.fdgs_forward(None, None, None, None, None, None, None, None, None)
    assert rc == 1   # FDGS_ERR_INVALID_ARG
    assert b"null" in lib.fdgs_last_error()
    lib.fdgs_backward.restype = ctypes.c_int
    assert lib.fdgs_backward(None, None) == 1


def test_debug_activate_rejects_other_norm_orders_without_touching_the_gpu():
    # the library has one summation order of the quaternion norm (ATen's, mode 0); the exported signature keeps the argument
    import fdgs
    lib = fdgs.lib()
    lib.fdgs_debug_activate.restype = ctypes.c_int
    buf = [(ctypes.c_float * 4)() for _ in range(6)]
    assert lib.fdgs_debug_activate(1, *buf[:3], 1, *buf[3:], None) == 1   # FDGS_ERR_INVALID_ARG
    assert b"mode" in lib.fdgs_last_error()


def test_extension_module_mirrors_reference_entry_points():
    import fdgs
    C = fdgs.ext()
    for name in ("rasterize_gaussians", "rasterize_gaussians_backward", "mark_visible"):
        assert hasattr(C, name)   # reference: diff-gaussian-rasterization/ext.cpp:15-19


def test_settings_fields_and_order():
    from gaussian_renderer import GaussianRasterizationSettings
    # reference: gaussian_renderer/diff_gaussian_rasterization.py:227-245
    assert GaussianRasterizationSettings._fields == (
        "image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix", "projmatrix",
        "sh_degree", "sh_degree_t", "campos", "timestamp", "time_duration", "rot_4d", "gaussian_dim", "force_sh_3d",
        "prefiltered", "debug")


def _rasterizer(rot_4d=True):
    from gaussian_renderer import GaussianRasterizationSettings, GaussianRasterizer
    cfg, cam, sc, st = helpers.build("tiny")
    st = dict(st)
    st["rot_4d"] = rot_4d
    return GaussianRasterizer(GaussianRasterizationSettings(**st)), sc


def test_argument_validation_matches_reference():
    r, sc = _rasterizer()
    m2 = torch.zeros_like(sc.means3D)
    # exactly one of shs / colors_precomp (reference: diff_gaussian_rasterization.py:271-272)
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        r(sc.means3D, m2, sc.opacities, scales=sc.scales, rotations=sc.rotations)
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        r(sc.means3D, m2, sc.opacities, shs=sc.shs, colors_precomp=sc.means3D, scales=sc.scales, rotations=sc.rotations)
    # exactly one of scale/rotation pair or cov3D_precomp (:274-275)
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        r(sc.means3D, m2, sc.opacities, shs=sc.shs)
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        r(sc.means3D, m2, sc.opacities, shs=sc.shs, scales=sc.scales, rotations=sc.rotations,
          cov3D_precomp=torch.zeros(sc.P, 6))
    # rot_4d needs rotations_r, scales_t, ts (:277-280)
    with pytest.raises(Exception, match="rotations_r and scales_t and ts"):
        r(sc.means3D, m2, sc.opacities, shs=sc.shs, scales=sc.scales, rotations=sc.rotations)


def test_means3d_shape_check_raises_before_any_gpu_work():
    import fdgs
    C = fdgs.ext()
    e = torch.Tensor([])
    bad = torch.zeros(10, 4)
    with pytest.raises(Exception, match="means3D must have dimensions"):   # reference: rasterize_points.cu:69-71
        C.rasterize_gaussians(torch.zeros(3), bad, e, e, e, e, e, e, e, e, 1.0, e, -1.0, torch.eye(4), torch.eye(4), 1.0,
                              1.0, 16, 16, e, 0, 0, torch.zeros(3), 0.0, 1.0, True, 4, False, False, False)


def test_tile_cull_option_round_trip():
    """fdgs_set_tile_cull is process-wide state of the library: returns the previous mode, defaults to 1 (no GPU needed)."""
    import fdgs
    prev = fdgs.set_tile_cull(0)
    try:
        assert prev in (0, 1)
        assert fdgs.set_tile_cull(1) == 0
        with fdgs.tile_cull(0):
            assert fdgs.set_tile_cull(0) == 0
        assert fdgs.set_tile_cull(1) == 1          # the context manager restored mode 1
    finally:
        fdgs.set_tile_cull(prev)
