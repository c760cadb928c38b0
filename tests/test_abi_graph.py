"""CPU: the batched forward sized by an instance capacity (fdgs_forward_batch_capacity) is declared, exported and
listed; a missing status word, a negative capacity, a missing device camera array, a bad view count, precomputed colours
and every check of fdgs_forward_batch are rejected before any GPU work; its extension binding checks dtype, layout, shape
and device (the per-view scalars must be CUDA tensors) first; render_batch with StaticViews names what it does not
cover."""
import ctypes

import pytest
import torch

from test_abi_and_host import _header_symbols
from test_abi_batch import ALLOC, F, ForwardBatchArgs, ForwardResult, _Cam, _Pipe, _binding_args, _fake, _valid


class ForwardCapacityArgs(ctypes.Structure):     # include/fdgs.h fdgs_forward_capacity_args
    _fields_ = [("batch", ForwardBatchArgs), ("timestamps", F), ("tan_fovx", F), ("tan_fovy", F), ("capacity", ctypes.c_int),
                ("status", ctypes.POINTER(ctypes.c_int))]


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


def _valid_capacity():
    c = ForwardCapacityArgs()
    c.batch = _valid()
    c.batch.timestamps = c.batch.tan_fovx = c.batch.tan_fovy = None   # ignored by this entry
    c.timestamps, c.tan_fovx, c.tan_fovy = _fake(), _fake(), _fake()
    c.capacity = 100
    c.status = ctypes.cast(ctypes.pointer((ctypes.c_int * 4)()), ctypes.POINTER(ctypes.c_int))
    return c


def test_symbol_declared_exported_and_listed(repo_root):
    import fdgs
    lib = fdgs.lib()
    assert "fdgs_forward_batch_capacity" in _header_symbols(repo_root)
    assert "fdgs_forward_batch_capacity" in fdgs.ABI_SYMBOLS
    assert hasattr(lib, "fdgs_forward_batch_capacity")
    assert lib.fdgs_version() == 2


def test_rejects_bad_arguments_before_gpu_work():
    import fdgs
    lib = fdgs.lib()
    lib.fdgs_forward_batch_capacity.restype = ctypes.c_int
    res = ForwardResult()

    def call(c):
        return lib.fdgs_forward_batch_capacity(ctypes.byref(c), _alloc, None, _alloc, None, _alloc, None, None,
                                               ctypes.byref(res))

    assert lib.fdgs_forward_batch_capacity(None, _alloc, None, _alloc, None, _alloc, None, None, ctypes.byref(res)) == 1
    cases = []
    c = _valid_capacity(); c.status = None; cases.append((c, b"status"))
    c = _valid_capacity(); c.capacity = -1; cases.append((c, b"capacity"))
    for f in ("timestamps", "tan_fovx", "tan_fovy"):
        c = _valid_capacity(); setattr(c, f, None); cases.append((c, b"camera table"))
    for f in ("viewmatrix", "projmatrix", "cam_pos"):
        c = _valid_capacity(); setattr(c.batch.view, f, None); cases.append((c, b"camera table"))
    c = _valid_capacity(); c.batch.B = 0; cases.append((c, b"view count"))
    c = _valid_capacity(); c.batch.B = 65536; cases.append((c, b"view count"))
    c = _valid_capacity(); c.batch.bg_image, c.batch.bg_views = _fake(), 2; cases.append((c, b"bg_image view count"))
    c = _valid_capacity(); c.batch.view.colors_precomp = _fake(); cases.append((c, b"precomputed"))
    c = _valid_capacity(); c.batch.view.cov3D_precomp = _fake(); cases.append((c, b"precomputed"))
    c = _valid_capacity(); c.batch.view.out_color = None; cases.append((c, b"output images"))
    c = _valid_capacity(); c.batch.view.M = 4; cases.append((c, b"SH degree"))
    for c, msg in cases:
        assert call(c) == 1
        assert msg in lib.fdgs_last_error(), (msg, lib.fdgs_last_error())
    assert _calls == []


def _capacity_args(capacity=10, B=2, **over):
    return _binding_args(B=B, **over) + (capacity,)


def test_extension_rejects_wrong_dtype_layout_shape_and_device_before_gpu_work():
    import fdgs
    C = fdgs.ext()
    with pytest.raises(RuntimeError, match="Float"):
        C.rasterize_gaussians_batch_capacity(*_capacity_args(tanfovx=torch.ones(2, dtype=torch.float64)))
    with pytest.raises(RuntimeError, match="contiguous"):
        C.rasterize_gaussians_batch_capacity(*_capacity_args(projmatrix=torch.zeros(4, 4, 2).permute(2, 0, 1)))
    with pytest.raises(RuntimeError, match="shape"):
        C.rasterize_gaussians_batch_capacity(*_capacity_args(timestamps=torch.zeros(3)))
    with pytest.raises(RuntimeError, match="shape"):
        C.rasterize_gaussians_batch_capacity(*_capacity_args(tanfovy=torch.zeros(1, 2)))
    with pytest.raises(RuntimeError, match="view count"):
        C.rasterize_gaussians_batch_capacity(*_capacity_args(B=0))
    with pytest.raises(RuntimeError, match="capacity"):
        C.rasterize_gaussians_batch_capacity(*_capacity_args(capacity=-1))
    with pytest.raises(RuntimeError, match="capacity"):
        C.rasterize_gaussians_batch_capacity(*_capacity_args(capacity=2 ** 31))
    # well-formed, but the per-view scalars are CPU tensors (the exact entry's convention)
    with pytest.raises(RuntimeError, match="must be CUDA tensors"):
        C.rasterize_gaussians_batch_capacity(*_capacity_args())


def _static_views(B=1, H=24, W=32):
    """A StaticViews shell: enough for the argument checks, which run before any of its tensors is touched"""
    from fdgs.graph import StaticViews
    v = StaticViews.__new__(StaticViews)
    v.B, v.H, v.W, v.capacity = B, H, W, 0
    return v


def test_render_batch_with_static_views_names_what_it_does_not_cover():
    from gaussian_renderer import render_batch
    from fdgs.dist import ViewParallelStep
    pc = object()
    bg = torch.zeros(3)
    views = _static_views()
    p = _Pipe(); p.env_map_res = 500
    with pytest.raises(ValueError, match="environment map"):
        render_batch(views, pc, p, bg)
    p = _Pipe(); p.debug = True
    with pytest.raises(ValueError, match="debug"):
        render_batch(views, pc, p, bg)
    with pytest.raises(ValueError, match="override_color"):
        render_batch(views, pc, _Pipe(), bg, override_color=torch.zeros(5, 3))
    p = _Pipe(); p.compute_cov3D_python = True
    with pytest.raises(ValueError, match="compute_cov3D_python"):
        render_batch(views, pc, p, bg)
    p = _Pipe(); p.convert_SHs_python = True
    with pytest.raises(ValueError, match="convert_SHs_python"):
        render_batch(views, pc, p, bg)
    step = ViewParallelStep.__new__(ViewParallelStep)
    old = ViewParallelStep.current
    ViewParallelStep.current = classmethod(lambda cls: step)
    try:
        with pytest.raises(ValueError, match="ViewParallelStep"):
            render_batch(views, pc, _Pipe(), bg)
    finally:
        ViewParallelStep.current = old


def test_graphed_step_checks_its_arguments():
    from fdgs.graph import GraphedStep, StaticViews
    with pytest.raises(ValueError, match="margin"):
        GraphedStep(lambda v, g: None, [], margin=0.5)
    with pytest.raises(ValueError, match="at least one"):
        GraphedStep(lambda v, g: None, [])([], torch.zeros(1))
    with pytest.raises(ValueError, match="B, H, W"):
        StaticViews(0, 24, 32, "cpu")
    views = _static_views(B=2)
    with pytest.raises(ValueError, match="holds 2 views"):
        StaticViews.load(views, [_Cam(W=32, H=24)])
    with pytest.raises(ValueError, match="32x24"):
        StaticViews.load(views, [_Cam(W=32, H=24), _Cam(W=40, H=24)])
