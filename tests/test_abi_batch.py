"""CPU: the batched-view entry points of the C-ABI are declared, exported and listed; a bad view count, a missing camera
table or output, a background image of another view count and every single-view check are rejected before any GPU
work; the extension bindings check dtype, layout, shape and device first; render_batch names what it does not cover."""
import ctypes

import pytest
import torch

from test_abi_and_host import _header_symbols

NEW = ("fdgs_geom_batch_bytes", "fdgs_image_batch_bytes", "fdgs_backward_batch_scratch_bytes", "fdgs_forward_batch",
       "fdgs_backward_batch", "fdgs_debug_export_binning_view")
F = ctypes.POINTER(ctypes.c_float)
ALLOC = ctypes.CFUNCTYPE(ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t)


def _fwd_fields():
    """include/fdgs.h fdgs_forward_args, in order"""
    i, f, p = ctypes.c_int, ctypes.c_float, F
    return [("P", i), ("D", i), ("D_t", i), ("M", i), ("background", p), ("width", i), ("height", i), ("means3D", p),
            ("shs", p), ("colors_precomp", p), ("flows_precomp", p), ("opacities", p), ("ts", p), ("scales", p),
            ("scales_t", p), ("scale_modifier", f), ("rotations", p), ("rotations_r", p), ("cov3D_precomp", p),
            ("prefilter_var", f), ("viewmatrix", p), ("projmatrix", p), ("cam_pos", p), ("timestamp", f),
            ("time_duration", f), ("rot_4d", i), ("gaussian_dim", i), ("force_sh_3d", i), ("tan_fovx", f),
            ("tan_fovy", f), ("prefiltered", i), ("debug", i), ("out_means3D", p), ("out_color", p), ("out_flow", p),
            ("out_depth", p), ("out_T", p), ("radii", ctypes.POINTER(ctypes.c_int)), ("raw_params", i), ("shs_rest", p)]


class ForwardArgs(ctypes.Structure):
    _fields_ = _fwd_fields()


class ForwardBatchArgs(ctypes.Structure):     # include/fdgs.h fdgs_forward_batch_args
    _fields_ = [("view", ForwardArgs), ("B", ctypes.c_int), ("timestamps", F), ("tan_fovx", F), ("tan_fovy", F),
                ("bg_image", F), ("bg_views", ctypes.c_int)]


class ForwardResult(ctypes.Structure):
    _fields_ = [("num_rendered", ctypes.c_int), ("geom_buffer", ctypes.c_void_p), ("binning_buffer", ctypes.c_void_p),
                ("image_buffer", ctypes.c_void_p), ("geom_bytes", ctypes.c_size_t), ("binning_bytes", ctypes.c_size_t),
                ("image_bytes", ctypes.c_size_t), ("cov3D", F)]


_calls = []


@ALLOC
def _alloc(ctx, n):
    _calls.append(n)      # must never be reached: the checks come first
    return None


@pytest.fixture(autouse=True)
def _clear_last_error():
    yield
    import fdgs
    assert fdgs.lib().fdgs_reset_opacity(ctypes.c_longlong(0), None, None, None, None) == 0


def _fake(n=64):
    return ctypes.cast(ctypes.pointer((ctypes.c_float * n)()), F)


def _valid():
    b = ForwardBatchArgs()
    a = b.view
    a.P, a.D, a.D_t, a.M, a.width, a.height = 10, 3, 2, 48, 64, 48
    for name in ("background", "means3D", "shs", "opacities", "ts", "scales", "scales_t", "rotations", "rotations_r",
                 "viewmatrix", "projmatrix", "cam_pos", "out_means3D", "out_color", "out_flow", "out_depth", "out_T"):
        setattr(a, name, _fake())
    a.radii = ctypes.cast(ctypes.pointer((ctypes.c_int * 64)()), ctypes.POINTER(ctypes.c_int))
    a.rot_4d, a.gaussian_dim, a.scale_modifier, a.time_duration = 1, 4, 1.0, 1.0
    b.B, b.timestamps, b.tan_fovx, b.tan_fovy = 3, _fake(), _fake(), _fake()
    return b


def test_symbols_declared_exported_and_listed(repo_root):
    import fdgs
    lib = fdgs.lib()
    for s in NEW:
        assert s in _header_symbols(repo_root)
        assert s in fdgs.ABI_SYMBOLS
        assert hasattr(lib, s)
    assert lib.fdgs_version() == 2
    for f in ("fdgs_geom_batch_bytes", "fdgs_backward_batch_scratch_bytes", "fdgs_geom_bytes"):
        getattr(lib, f).restype = ctypes.c_size_t
    lib.fdgs_image_batch_bytes.restype = ctypes.c_size_t
    lib.fdgs_image_bytes.restype = ctypes.c_size_t
    # B views hold at least B single views' scratch; sizes are 64-bit (2M Gaussians x 24 views > 2^32 bytes)
    assert lib.fdgs_geom_batch_bytes(300000, 24) >= 24 * (lib.fdgs_geom_bytes(300000) - 256)
    assert lib.fdgs_image_batch_bytes(1352, 1014, 4) >= 4 * (lib.fdgs_image_bytes(1352, 1014) - 256) // 2
    assert lib.fdgs_backward_batch_scratch_bytes(2000000, 24) > 2 ** 32


def test_rejects_bad_arguments_before_gpu_work():
    import fdgs
    lib = fdgs.lib()
    lib.fdgs_forward_batch.restype = ctypes.c_int
    res = ForwardResult()

    def call(b):
        return lib.fdgs_forward_batch(ctypes.byref(b), _alloc, None, _alloc, None, _alloc, None, None, ctypes.byref(res))

    assert lib.fdgs_forward_batch(None, _alloc, None, _alloc, None, _alloc, None, None, ctypes.byref(res)) == 1
    cases = []
    b = _valid(); b.B = 0; cases.append((b, b"view count"))
    b = _valid(); b.B = -2; cases.append((b, b"view count"))
    b = _valid(); b.B = 65536; cases.append((b, b"view count"))
    b = _valid(); b.bg_image, b.bg_views = _fake(), 2; cases.append((b, b"bg_image view count"))
    for f in ("timestamps", "tan_fovx", "tan_fovy"):
        b = _valid(); setattr(b, f, None); cases.append((b, b"camera table"))
    for f in ("viewmatrix", "projmatrix", "cam_pos"):
        b = _valid(); setattr(b.view, f, None); cases.append((b, b"camera table"))
    for f in ("out_color", "out_T", "background"):
        b = _valid(); setattr(b.view, f, None); cases.append((b, b"output images"))
    for f in ("out_means3D", "radii"):
        b = _valid(); setattr(b.view, f, None); cases.append((b, b"output pointers"))
    b = _valid(); b.view.P = -1; cases.append((b, b"bad P"))
    b = _valid(); b.view.M = 4; cases.append((b, b"SH degree"))
    b = _valid(); b.view.rotations_r = None; cases.append((b, b"rot_4d"))
    b = _valid(); b.view.colors_precomp = _fake(); cases.append((b, b"precomputed"))
    b = _valid(); b.view.cov3D_precomp = _fake(); cases.append((b, b"precomputed"))
    for b, msg in cases:
        assert call(b) == 1
        assert msg in lib.fdgs_last_error(), (msg, lib.fdgs_last_error())
    assert _calls == []
    lib.fdgs_backward_batch.restype = ctypes.c_int
    assert lib.fdgs_backward_batch(None, None) == 1
    lib.fdgs_debug_export_binning_view.restype = ctypes.c_int
    assert lib.fdgs_debug_export_binning_view(None, 16, 16, 2, 0, None, None, None) == 1
    scratch = ctypes.cast(_fake(), ctypes.c_char_p)
    assert lib.fdgs_debug_export_binning_view(scratch, 16, 16, 2, 2, None, None, None) == 1
    assert b"view" in lib.fdgs_last_error()


def _binding_args(B=2, P=5, **over):
    c = dict(viewmatrix=torch.zeros(B, 4, 4), projmatrix=torch.zeros(B, 4, 4), campos=torch.zeros(B, 3),
             timestamps=torch.zeros(B), tanfovx=torch.ones(B), tanfovy=torch.ones(B), bg_image=torch.Tensor([]))
    c.update(over)
    e = torch.Tensor([])
    return (torch.zeros(3), torch.zeros(P, 3), e, torch.zeros(P, 1), e, torch.zeros(P, 3), e, torch.zeros(P, 4), e, 1.0,
            -1.0, c["viewmatrix"], c["projmatrix"], c["campos"], c["timestamps"], c["tanfovx"], c["tanfovy"], 16, 16,
            torch.zeros(P, 16, 3), e, 3, 0, 1.0, False, 3, False, False, False, False, c["bg_image"])


def test_extension_rejects_wrong_dtype_layout_shape_and_device_before_gpu_work():
    import fdgs
    C = fdgs.ext()
    with pytest.raises(RuntimeError, match="Float"):
        C.rasterize_gaussians_batch(*_binding_args(viewmatrix=torch.zeros(2, 4, 4, dtype=torch.float64)))
    with pytest.raises(RuntimeError, match="contiguous"):
        C.rasterize_gaussians_batch(*_binding_args(projmatrix=torch.zeros(4, 4, 2).permute(2, 0, 1)))
    with pytest.raises(RuntimeError, match="shape"):
        C.rasterize_gaussians_batch(*_binding_args(campos=torch.zeros(2, 4)))
    with pytest.raises(RuntimeError, match="shape"):
        C.rasterize_gaussians_batch(*_binding_args(timestamps=torch.zeros(3)))
    with pytest.raises(RuntimeError, match="view count"):
        C.rasterize_gaussians_batch(*_binding_args(B=0))
    with pytest.raises(RuntimeError, match="CUDA"):                     # well-formed, but on the host
        C.rasterize_gaussians_batch(*_binding_args())


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False
    env_map_res = 0


class _Cam:
    def __init__(self, W=32, H=24):
        self.image_width, self.image_height = W, H


def test_render_batch_names_what_it_does_not_cover():
    from gaussian_renderer import render_batch
    from fdgs.dist import ViewParallelStep
    pc = object()
    bg = torch.zeros(3)
    with pytest.raises(ValueError, match="at least one"):
        render_batch([], pc, _Pipe(), bg)
    with pytest.raises(ValueError, match="override_color"):
        render_batch([_Cam()], pc, _Pipe(), bg, override_color=torch.zeros(5, 3))
    p = _Pipe(); p.compute_cov3D_python = True
    with pytest.raises(ValueError, match="compute_cov3D_python"):
        render_batch([_Cam()], pc, p, bg)
    p = _Pipe(); p.convert_SHs_python = True
    with pytest.raises(ValueError, match="convert_SHs_python"):
        render_batch([_Cam()], pc, p, bg)
    with pytest.raises(ValueError, match="image size"):
        render_batch([_Cam(), _Cam(W=40)], pc, _Pipe(), bg)
    step = ViewParallelStep.__new__(ViewParallelStep)
    old = ViewParallelStep.current
    ViewParallelStep.current = classmethod(lambda cls: step)
    try:
        with pytest.raises(ValueError, match="ViewParallelStep"):
            render_batch([_Cam()], pc, _Pipe(), bg)
    finally:
        ViewParallelStep.current = old
