"""CPU: the pieces that put the optimiser and the densification statistics inside the captured training step.

fdgs_adam_scalars, fdgs_adam_step_staged and fdgs_densify_stats_status are declared, exported and listed; their bad
counts, null pointers and widths are rejected before any GPU work (called with host pointers); fdgs_adam_scalars equals
torch's double-precision bias correction for steps 1..30000 at several learning rates; the extension bindings check
their tables; GraphedStep refuses an optimiser it cannot capture, a hold it cannot apply and statistics without the
model's accumulators, before any GPU work."""
import ctypes
import math

import numpy as np
import pytest
import torch

from test_abi_and_host import _header_symbols
from test_abi_batch import _Cam

NEW = ("fdgs_adam_scalars", "fdgs_adam_step_staged", "fdgs_densify_stats_status")
F = ctypes.POINTER(ctypes.c_float)
I = ctypes.POINTER(ctypes.c_int)
LL = ctypes.POINTER(ctypes.c_longlong)


def _lib():
    import fdgs
    lib = fdgs.lib()
    for n in NEW:
        getattr(lib, n).restype = ctypes.c_int
    return lib


def _fake(n=16, t=ctypes.c_float, p=F):
    """A non-null host address: the checks must fail before anything dereferences it."""
    return ctypes.cast(ctypes.pointer((t * n)()), p)


@pytest.fixture(autouse=True)
def _clear_last_error():
    yield
    assert _lib().fdgs_reset_opacity(ctypes.c_longlong(0), None, None, None, None) == 0


def test_symbols_declared_exported_and_listed(repo_root):
    import fdgs
    lib = _lib()
    for s in NEW:
        assert s in _header_symbols(repo_root)
        assert s in fdgs.ABI_SYMBOLS
        assert hasattr(lib, s)
    assert lib.fdgs_version() == 2


def _ptrs(n):
    return (F * 16)(*[_fake() for _ in range(16)]) if n else None


def test_staged_adam_rejects_bad_arguments_before_gpu_work():
    lib = _lib()
    widths = (ctypes.c_int * 16)(*([3] * 16))

    def call(n=2, params=True, grads=True, m=True, v=True, w=widths, P=10, scalars=True, status=None):
        return lib.fdgs_adam_step_staged(n, _ptrs(params), _ptrs(grads), _ptrs(m), _ptrs(v), w, ctypes.c_longlong(P),
                                         _fake() if scalars else None, status, ctypes.c_double(0.9),
                                         ctypes.c_double(0.999), ctypes.c_double(1e-15), None)

    for kw, msg in ((dict(n=-1), b"tensor count"), (dict(n=17), b"tensor count"), (dict(P=-1), b"row count"),
                    (dict(params=False), b"null"), (dict(grads=False), b"null"), (dict(m=False), b"null"),
                    (dict(v=False), b"null"), (dict(w=None), b"null"), (dict(scalars=False), b"null"),
                    (dict(w=(ctypes.c_int * 16)(3, 0)), b"table entry"),
                    (dict(w=(ctypes.c_int * 16)(-2, 3)), b"table entry")):
        assert call(**kw) == 1, kw
        assert msg in lib.fdgs_last_error(), (kw, lib.fdgs_last_error())
    one_null = (F * 16)(*[_fake() for _ in range(16)])
    one_null[1] = None
    assert lib.fdgs_adam_step_staged(2, one_null, _ptrs(1), _ptrs(1), _ptrs(1), widths, ctypes.c_longlong(10), _fake(),
                                     None, ctypes.c_double(0.9), ctypes.c_double(0.999), ctypes.c_double(1e-15), None) == 1
    assert b"table entry" in lib.fdgs_last_error()
    # nothing to do: accepted without touching a pointer
    assert call(n=0, params=False, grads=False, m=False, v=False, w=None, scalars=False) == 0
    assert call(P=0) == 0


def test_adam_scalars_rejects_bad_arguments():
    lib = _lib()
    lrs, table = _fake(), _fake(48)
    steps = (ctypes.c_longlong * 16)(*range(1, 17))
    enable = (ctypes.c_int * 16)(*([1] * 16))
    b1, b2 = ctypes.c_double(0.9), ctypes.c_double(0.999)
    for args, msg in (((-1, lrs, steps, enable, b1, b2, table), b"tensor count"),
                      ((17, lrs, steps, enable, b1, b2, table), b"tensor count"),
                      ((2, None, steps, enable, b1, b2, table), b"null"),
                      ((2, lrs, None, enable, b1, b2, table), b"null"),
                      ((2, lrs, steps, None, b1, b2, table), b"null"),
                      ((2, lrs, steps, enable, b1, b2, None), b"null"),
                      ((2, lrs, (ctypes.c_longlong * 16)(1, 0), enable, b1, b2, table), b"step count")):
        assert lib.fdgs_adam_scalars(*args) == 1, msg
        assert msg in lib.fdgs_last_error()
    # a held tensor's step count is not read: 0 (never stepped) is fine
    assert lib.fdgs_adam_scalars(2, lrs, (ctypes.c_longlong * 16)(1, 0), (ctypes.c_int * 16)(1, 0), b1, b2, table) == 0


def test_densify_stats_status_rejects_bad_arguments_before_gpu_work():
    lib = _lib()
    status = _fake(4, ctypes.c_int, I)
    args = [ctypes.c_longlong(5), 1, _fake(), 3, None, _fake(4, ctypes.c_int, I), None, _fake(), _fake(), None, _fake(),
            status, None]
    for i, val, msg in ((7, None, b"null"), (1, 4, b"stride"), (6, _fake(), b"t_grad"), (0, ctypes.c_longlong(-1), b"P"),
                        (1, 0, b"batch size"), (5, None, b"null")):
        bad = list(args)
        bad[i] = val
        assert lib.fdgs_densify_stats_status(*bad) == 1, msg
        assert msg in lib.fdgs_last_error(), (msg, lib.fdgs_last_error())
    empty = list(args)
    empty[0] = ctypes.c_longlong(0)
    assert lib.fdgs_densify_stats_status(*empty) == 0


@pytest.mark.parametrize("lr", [1.6e-4, 0.0025, 0.05, 0.005, 0.001, 1.7e-6, 0.0])
def test_adam_scalars_equal_the_double_bias_correction(lr):
    """table = float32(float64(float32(lr)) / (1 - b1**s)), float32(sqrt(1 - b2**s)), 1 for s = 1 .. 30000."""
    lib = _lib()
    b1, b2 = 0.9, 0.999
    S = 30000
    got = np.empty((S, 3), dtype=np.float32)
    lrs = (ctypes.c_float * 16)(*([lr] * 16))
    enable = (ctypes.c_int * 16)(*([1] * 16))
    for s0 in range(1, S + 1, 16):
        n = min(16, S + 1 - s0)
        steps = (ctypes.c_longlong * 16)(*range(s0, s0 + n))
        table = (ctypes.c_float * 48)()
        assert lib.fdgs_adam_scalars(n, lrs, steps, enable, ctypes.c_double(b1), ctypes.c_double(b2), table) == 0
        got[s0 - 1:s0 - 1 + n] = np.frombuffer(table, dtype=np.float32).reshape(16, 3)[:n]
    lr32 = float(np.float32(lr))
    want = np.array([[np.float32(lr32 / (1 - b1 ** s)), np.float32(math.sqrt(1 - b2 ** s)), 1.0] for s in range(1, S + 1)],
                    dtype=np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_adam_scalars_hold_entries():
    lib = _lib()
    table = (ctypes.c_float * 48)()
    lrs = (ctypes.c_float * 16)(0.1, 0.2, 0.3)
    steps = (ctypes.c_longlong * 16)(5, 0, 7)
    enable = (ctypes.c_int * 16)(1, 0, 1)
    assert lib.fdgs_adam_scalars(3, lrs, steps, enable, ctypes.c_double(0.9), ctypes.c_double(0.999), table) == 0
    t = np.frombuffer(table, dtype=np.float32).reshape(16, 3)[:3]
    assert t[1].tolist() == [0.0, 1.0, 0.0]
    assert t[0, 2] == 1.0 and t[2, 2] == 1.0
    assert t[2, 0] == np.float32(float(np.float32(0.3)) / (1 - 0.9 ** 7))


def test_extension_bindings_check_their_tables_before_gpu_work():
    import fdgs
    C = fdgs.ext()
    with pytest.raises(RuntimeError, match="mismatch"):
        C.adam_scalars([0.1, 0.2], [1], [1, 1], 0.9, 0.999, torch.zeros(6))
    with pytest.raises(RuntimeError, match="shape"):
        C.adam_scalars([0.1, 0.2], [1, 1], [1, 1], 0.9, 0.999, torch.zeros(5))
    with pytest.raises(RuntimeError, match="float32"):
        C.adam_scalars([0.1], [1], [1], 0.9, 0.999, torch.zeros(3, dtype=torch.float64))
    with pytest.raises(RuntimeError, match="step count"):
        C.adam_scalars([0.1], [0], [1], 0.9, 0.999, torch.zeros(3))
    table = torch.zeros(6)
    C.adam_scalars([0.1, 0.2], [1, 3], [1, 0], 0.9, 0.999, table)     # host-only: runs here
    assert table[0].item() == np.float32(float(np.float32(0.1)) / (1 - 0.9)) and table[3:].tolist() == [0.0, 1.0, 0.0]
    P = 8
    t = [torch.zeros(P, 3)]
    with pytest.raises(RuntimeError, match="mismatch"):
        C.adam_step_staged(t, t, t, [], torch.zeros(3), torch.empty(0), 0.9, 0.999, 1e-15)
    with pytest.raises(RuntimeError, match="shape"):
        C.adam_step_staged(t, t, t, t, torch.zeros(6), torch.empty(0), 0.9, 0.999, 1e-15)
    with pytest.raises(RuntimeError, match="int32"):
        C.adam_step_staged(t, t, t, t, torch.zeros(3), torch.zeros(4), 0.9, 0.999, 1e-15)
    with pytest.raises(RuntimeError, match="CUDA tensors"):                               # well-formed, but on the host
        C.adam_step_staged(t, t, t, t, torch.zeros(3), torch.zeros(4, dtype=torch.int32), 0.9, 0.999, 1e-15)
    with pytest.raises(RuntimeError, match="shape"):
        C.densify_stats(1, torch.zeros(P, 3), torch.empty(0), torch.zeros(P, dtype=torch.int32), torch.empty(0),
                        torch.zeros(P, 1), torch.zeros(P, 1), torch.empty(0), torch.zeros(P), torch.zeros(3, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        C.densify_stats(1, torch.zeros(P, 3), torch.empty(0), torch.zeros(P, dtype=torch.int32), torch.empty(0),
                        torch.zeros(P, 1), torch.zeros(P, 1), torch.empty(0), torch.zeros(P), torch.zeros(4, dtype=torch.int32))


class _Model:
    """A shell with named parameter groups: enough for the argument checks."""

    def __init__(self, stats=True):
        from fdgs.optim import FusedAdam
        self._xyz, self._opacity = torch.zeros(4, 3), torch.zeros(4, 1)
        self.optimizer = FusedAdam([{"params": [self._xyz], "name": "xyz"}, {"params": [self._opacity], "name": "opacity"}])
        self.gaussian_dim = 3
        if stats:
            self.xyz_gradient_accum, self.denom, self.max_radii2D = torch.zeros(4, 1), torch.zeros(4, 1), torch.zeros(4)


def test_graphed_step_rejects_what_it_cannot_capture():
    from fdgs.graph import GraphedStep
    from fdgs.optim import FusedAdam
    m = _Model()
    cams, gt = [_Cam()], torch.zeros(1, 3, 24, 32)
    fn = lambda v, g: None    # noqa: E731  (never reached)
    with pytest.raises(ValueError, match="FusedAdam"):
        GraphedStep(fn, m, optimizer=torch.optim.Adam([torch.zeros(2, requires_grad=True)]))
    other = FusedAdam([{"params": [m._xyz], "name": "xyz"}])
    with pytest.raises(ValueError, match="exactly the step's leaves"):
        GraphedStep(fn, m, optimizer=other)(cams, gt)
    extra = FusedAdam([{"params": [m._xyz, torch.zeros(4, 3)], "name": "xyz"}, {"params": [m._opacity], "name": "opacity"}])
    with pytest.raises(ValueError, match="exactly the step's leaves"):
        GraphedStep(fn, m, optimizer=extra)(cams, gt)
    with pytest.raises(ValueError, match="features"):
        GraphedStep(fn, m, optimizer=m.optimizer)(cams, gt, hold={"opacity", "features"})
    with pytest.raises(ValueError, match="hold needs"):
        GraphedStep(fn, m)(cams, gt, hold=True)
    with pytest.raises(ValueError, match="xyz_gradient_accum"):
        GraphedStep(fn, _Model(stats=False))(cams, gt, densify_stats=True)
    with pytest.raises(ValueError, match="xyz_gradient_accum"):
        GraphedStep(fn, [m._xyz, m._opacity])(cams, gt, densify_stats=True)
    four = _Model()
    four.gaussian_dim = 4
    with pytest.raises(ValueError, match="t_gradient_accum"):
        GraphedStep(fn, four)(cams, gt, densify_stats=True)


def test_fused_adam_hold_names_its_groups():
    m = _Model()
    opt = m.optimizer
    assert opt.held(()) == set() and opt.held(False) == set()
    assert opt.held(True) == {id(m._xyz), id(m._opacity)}
    assert opt.held({"opacity"}) == {id(m._opacity)} and opt.held("opacity") == {id(m._opacity)}
    with pytest.raises(ValueError, match="rotation"):
        opt.held(["xyz", "rotation"])
    with pytest.raises(RuntimeError, match="init_state"):
        opt.step_staged([m._xyz])
