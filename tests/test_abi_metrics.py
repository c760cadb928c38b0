"""CPU: the evaluation-metric entry points of the C-ABI are declared, exported and listed; null pointers, non-positive
sizes, H or W below 176, more than 65535 image planes and size overflow are rejected before any GPU work; the
extension binding and fdgs.metrics check dtype, layout, shape and device first."""
import ctypes

import pytest
import torch

from test_abi_and_host import _header_symbols

NEW = ("fdgs_metrics_scratch_bytes", "fdgs_image_metrics")
F = ctypes.POINTER(ctypes.c_float)
D = ctypes.POINTER(ctypes.c_double)


class MetricsArgs(ctypes.Structure):     # include/fdgs.h fdgs_metrics_args
    _fields_ = [("B", ctypes.c_int), ("C", ctypes.c_int), ("H", ctypes.c_int), ("W", ctypes.c_int), ("x", F), ("y", F),
                ("clamp", ctypes.c_int), ("out", D), ("accum", D)]


@pytest.fixture(autouse=True)
def _clear_last_error():
    yield
    import fdgs
    assert fdgs.lib().fdgs_reset_opacity(ctypes.c_longlong(0), None, None, None, None) == 0    # a call that succeeds clears it


def _fake(ptr=F, n=4):
    """A non-null host address: the checks must fail before anything dereferences it."""
    base = ctypes.c_float if ptr is F else ctypes.c_double
    return ctypes.cast(ctypes.pointer((base * n)()), ptr)


def _valid():
    a = MetricsArgs()
    a.B, a.C, a.H, a.W = 2, 3, 200, 300
    a.x, a.y, a.out, a.accum = _fake(), _fake(), _fake(D), _fake(D)
    return a


def test_symbols_declared_exported_and_listed(repo_root):
    import fdgs
    lib = fdgs.lib()
    for s in NEW:
        assert s in _header_symbols(repo_root)
        assert s in fdgs.ABI_SYMBOLS
        assert hasattr(lib, s)
    assert lib.fdgs_version() == 2
    assert lib.fdgs_metrics_scratch_bytes.restype == ctypes.c_size_t
    one = lib.fdgs_metrics_scratch_bytes(1, 3, 1014, 1352)
    assert one > 0 and lib.fdgs_metrics_scratch_bytes(4, 3, 1014, 1352) > 3 * one
    # pyramid levels 2..5 of both images in float64: at least 2 * 8 * (1/4 + 1/16 + ...) bytes per input value
    assert one >= 2 * 8 * 3 * (507 * 676 + 253 * 338 + 126 * 169 + 63 * 84)
    for bad in ((0, 3, 200, 200), (1, 0, 200, 200), (1, 3, 175, 200), (1, 3, 200, 175), (70000, 1, 200, 200),
                (-1, 3, 200, 200)):
        assert lib.fdgs_metrics_scratch_bytes(*bad) == 0, bad


def test_rejects_bad_arguments():
    import fdgs
    lib = fdgs.lib()
    lib.fdgs_image_metrics.restype = ctypes.c_int
    scratch = ctypes.cast(_fake(), ctypes.c_char_p)
    assert lib.fdgs_image_metrics(None, scratch, None) == 1
    assert b"null" in lib.fdgs_last_error()
    cases = []
    a = _valid(); a.B = 0; cases.append((a, b"B / C / H / W"))
    a = _valid(); a.C = -1; cases.append((a, b"B / C / H / W"))
    a = _valid(); a.H = 0; cases.append((a, b"B / C / H / W"))
    a = _valid(); a.W = -5; cases.append((a, b"B / C / H / W"))
    a = _valid(); a.H = 175; cases.append((a, b"176"))
    a = _valid(); a.W = 16; cases.append((a, b"176"))
    a = _valid(); a.B, a.C = 30000, 3; cases.append((a, b"65535"))
    a = _valid(); a.B, a.C, a.H, a.W = 60000, 1, 2_000_000_000, 2_000_000_000; cases.append((a, b"overflow"))
    a = _valid(); a.B, a.C, a.H, a.W = 1, 1, 2_100_000, 200; cases.append((a, b"overflow"))
    a = _valid(); a.x = None; cases.append((a, b"null"))
    a = _valid(); a.y = None; cases.append((a, b"null"))
    a = _valid(); a.out = None; cases.append((a, b"null"))
    for args, msg in cases:
        assert lib.fdgs_image_metrics(ctypes.byref(args), scratch, None) == 1
        assert msg in lib.fdgs_last_error(), (msg, lib.fdgs_last_error())
    assert lib.fdgs_image_metrics(ctypes.byref(_valid()), None, None) == 1              # no scratch
    assert b"scratch" in lib.fdgs_last_error()


def test_extension_rejects_wrong_dtype_layout_shape_and_device_before_gpu_work():
    import fdgs
    C = fdgs.ext()
    x = torch.zeros(1, 3, 180, 190)
    none = torch.empty(0)
    with pytest.raises(RuntimeError, match="Float"):
        C.image_metrics(x.double(), x.double(), False, none)
    with pytest.raises(RuntimeError, match="contiguous"):
        C.image_metrics(x.transpose(2, 3), x.transpose(2, 3), False, none)
    with pytest.raises(RuntimeError, match="shape"):
        C.image_metrics(x, x[:, :, :179].contiguous(), False, none)
    with pytest.raises(RuntimeError, match="shape"):
        C.image_metrics(x[0], x[0], False, none)
    with pytest.raises(RuntimeError, match="accum"):
        C.image_metrics(x, x, False, torch.zeros(5))
    with pytest.raises(RuntimeError, match="accum"):
        C.image_metrics(x, x, False, torch.zeros(4, dtype=torch.float64))
    with pytest.raises(RuntimeError, match="CUDA tensors"):                           # well-formed, but on the host
        C.image_metrics(x, x, True, torch.zeros(5, dtype=torch.float64))


def test_python_interface_rejects_what_torchmetrics_rejects():
    from fdgs import metrics
    x = torch.zeros(3, 175, 200)
    with pytest.raises(ValueError, match="176"):
        metrics.msssim(x[None], x[None])
    with pytest.raises(ValueError, match="176"):
        metrics.image_metrics(torch.zeros(2, 3, 200, 160), torch.zeros(2, 3, 200, 160))
    with pytest.raises(ValueError, match="shape"):
        metrics.image_metrics(torch.zeros(3, 200, 200), torch.zeros(3, 200, 201))
    with pytest.raises(ValueError, match=r"\[C,H,W\]"):
        metrics.image_metrics(torch.zeros(200, 200), torch.zeros(200, 200))
    with pytest.raises(ValueError, match="CUDA"):                                      # no CPU fallback
        metrics.msssim(torch.zeros(1, 3, 200, 200), torch.zeros(1, 3, 200, 200))
    with pytest.raises(ValueError, match="CUDA"):
        metrics.MetricAccumulator().add(torch.zeros(3, 200, 200), torch.zeros(3, 200, 200))
    r = metrics.MetricAccumulator().result()
    assert all(v != v for v in r) and r._fields == ("l1", "psnr", "ssim", "msssim")
