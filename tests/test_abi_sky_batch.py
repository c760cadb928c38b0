"""CPU: the batched sky sampler that lets environment-map scenes run in the captured training iteration.

fdgs_sky_forward_batch / fdgs_sky_backward_batch are declared, exported and listed (the ABI version stays 2); null
pointers, a view count below 1 and empty sizes are rejected with status 1 before any GPU work (called with host
pointers); the extension binds both; StaticViews(..., sky=True).load() refuses a camera without pinhole intrinsics, and
GraphedStep refuses a learned env_map that is not a parameter group of the model's FusedAdam, before any GPU work."""
import ctypes

import pytest
import torch

from test_abi_and_host import _header_symbols
from test_abi_batch import _Cam

NEW = ("fdgs_sky_forward_batch", "fdgs_sky_backward_batch")
F = ctypes.POINTER(ctypes.c_float)


class _Args(ctypes.Structure):
    """include/fdgs.h: fdgs_sky_batch_args"""
    _fields_ = [("env_map", F), ("env_height", ctypes.c_int), ("env_width", ctypes.c_int), ("c2w", F), ("campos", F),
                ("intrinsics", F), ("radius", ctypes.c_float), ("width", ctypes.c_int), ("height", ctypes.c_int),
                ("B", ctypes.c_int)]


def _lib():
    import fdgs
    lib = fdgs.lib()
    for n in NEW:
        getattr(lib, n).restype = ctypes.c_int
    lib.fdgs_last_error.restype = ctypes.c_char_p
    return lib


def _fake(n=16):
    """A non-null host address: the checks must fail before anything dereferences it."""
    return ctypes.cast(ctypes.pointer((ctypes.c_float * n)()), F)


def _args(**kw):
    a = _Args(env_map=_fake(), env_height=8, env_width=16, c2w=_fake(), campos=_fake(), intrinsics=_fake(), radius=60.0,
              width=32, height=24, B=2)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.fixture(autouse=True)
def _clear_last_error():
    yield
    assert _lib().fdgs_reset_opacity(ctypes.c_longlong(0), None, None, None, None) == 0


def test_symbols_declared_exported_and_listed(repo_root):
    import fdgs
    lib = _lib()
    header = _header_symbols(repo_root)
    for s in NEW:
        assert s in header
        assert s in fdgs.ABI_SYMBOLS
        assert hasattr(lib, s)
    assert set(header) == set(fdgs.ABI_SYMBOLS)
    assert lib.fdgs_version() == 2


@pytest.mark.parametrize("entry", NEW)
def test_bad_arguments_are_rejected_before_gpu_work(entry):
    lib = _lib()
    fn = getattr(lib, entry)

    def call(a, p1=True, p2=True):
        out = _fake() if p1 else None
        if entry == "fdgs_sky_forward_batch":
            return fn(ctypes.byref(a), out, None, None)      # a null miss flag is allowed
        return fn(ctypes.byref(a), out, _fake() if p2 else None, None)

    assert fn(None, _fake(), _fake(), None) == 1
    assert b"null" in lib.fdgs_last_error()
    for kw, msg in ((dict(env_map=None), b"required"), (dict(c2w=None), b"required"), (dict(campos=None), b"required"),
                    (dict(intrinsics=None), b"required"), (dict(B=0), b"view count"), (dict(B=-3), b"view count"),
                    (dict(B=70000), b"view count"), (dict(width=0), b"size"), (dict(height=0), b"size"),
                    (dict(env_height=0), b"size"), (dict(env_width=-1), b"size"), (dict(radius=0.0), b"radius"),
                    (dict(radius=float("nan")), b"radius"), (dict(width=40000, height=40000), b"size")):
        assert call(_args(**kw)) == 1, kw
        assert msg in lib.fdgs_last_error(), (kw, lib.fdgs_last_error())
    assert call(_args(), p1=False) == 1 and b"null" in lib.fdgs_last_error()
    if entry == "fdgs_sky_backward_batch":
        assert call(_args(), p2=False) == 1 and b"null" in lib.fdgs_last_error()


def test_extension_binds_the_batched_sampler():
    import fdgs
    C = fdgs.ext()
    assert hasattr(C, "sky_forward_batch") and hasattr(C, "sky_backward_batch")
    env, c2w, campos, k = torch.zeros(3, 8, 16), torch.zeros(2, 4, 4), torch.zeros(2, 3), torch.zeros(2, 4)
    with pytest.raises(RuntimeError, match="c2w"):
        C.sky_forward_batch(env, torch.zeros(2, 16), campos, k, 60.0, 24, 32)
    with pytest.raises(RuntimeError, match="intrinsics"):
        C.sky_forward_batch(env, c2w, campos, torch.zeros(2, 3), 60.0, 24, 32)
    with pytest.raises(RuntimeError, match="campos"):
        C.sky_forward_batch(env, c2w, torch.zeros(3, 3), k, 60.0, 24, 32)
    with pytest.raises(RuntimeError, match="float32"):
        C.sky_forward_batch(env.double(), c2w, campos, k, 60.0, 24, 32)
    with pytest.raises(RuntimeError, match="CUDA tensors"):                  # well-formed, but on the host
        C.sky_forward_batch(env, c2w, campos, k, 60.0, 24, 32)
    with pytest.raises(RuntimeError, match="dL_dsky"):
        C.sky_backward_batch(env, c2w, campos, k, 60.0, torch.zeros(3, 3, 24, 32))


def _sky_views(B=2, H=24, W=32):
    """A StaticViews(sky=True) shell: the camera checks of load() run before any of its tensors is touched"""
    from fdgs.graph import StaticViews
    v = StaticViews.__new__(StaticViews)
    v.B, v.H, v.W, v.sky, v.capacity = B, H, W, True, 0
    return v


class _SkyCam(_Cam):
    def __init__(self, fl_x=30.0):
        super().__init__()
        self.timestamp, self.FoVx, self.FoVy = 0.5, 1.0, 0.8
        self.fl_x, self.fl_y, self.cx, self.cy = fl_x, 30.0, 16.0, 12.0


def test_static_views_with_sky_reject_a_camera_without_intrinsics():
    views = _sky_views()
    for bad in (_Cam(), _SkyCam(fl_x=0.0), _SkyCam(fl_x=-5.0)):
        with pytest.raises(ValueError, match="intrinsics"):
            views.load([_SkyCam(), bad])
    with pytest.raises(ValueError, match="2 views"):
        views.load([_SkyCam()])


def test_render_batch_with_sky_views_checks_before_touching_the_model():
    from gaussian_renderer import render_batch
    from test_abi_graph import _Pipe, _static_views
    p = _Pipe(); p.env_map_res = 500
    with pytest.raises(ValueError, match="environment map.*sky=True"):
        render_batch(_static_views(), object(), p, torch.zeros(3))


class _Model:
    """A shell with named parameter groups and an environment map"""

    def __init__(self, env_group=None):
        from fdgs.optim import FusedAdam
        self._xyz = torch.zeros(4, 3, requires_grad=True)
        self.env_map = torch.zeros(3, 8, 16, requires_grad=True)
        groups = [{"params": [self._xyz], "name": "xyz"}]
        if env_group is not None:
            groups.append({"params": [self.env_map], "name": env_group})
        self.optimizer = FusedAdam(groups)
        self.gaussian_dim = 3


def test_graphed_step_rejects_an_env_map_outside_the_optimiser():
    from fdgs.graph import GraphedStep
    cams, gt = [_SkyCam()], torch.zeros(1, 3, 24, 32)
    fn = lambda v, g: None    # noqa: E731  (never reached)
    for m in (_Model(), _Model(env_group="features")):
        with pytest.raises(ValueError, match="env_map"):
            GraphedStep(fn, m)(cams, gt)
        with pytest.raises(ValueError, match="env_map"):
            GraphedStep(fn, m, optimizer=m.optimizer)(cams, gt)
    m = _Model()
    m.optimizer = torch.optim.Adam([{"params": [m._xyz], "name": "xyz"}, {"params": [m.env_map], "name": "env_map"}])
    with pytest.raises(ValueError, match="env_map"):
        GraphedStep(fn, m)(cams, gt)
