"""CPU: the densification entry points of the C-ABI are declared, exported and listed, and null, mismatched-width,
wrong-dtype and non-contiguous arguments are rejected before any GPU work."""
import ctypes

import pytest
import torch

from test_abi_and_host import _header_symbols

NEW = ("fdgs_densify_scratch_bytes", "fdgs_densify_plan", "fdgs_densify_apply", "fdgs_reset_opacity", "fdgs_densify_stats")
MAXT = 32
F = ctypes.POINTER(ctypes.c_float)


class DensifyArgs(ctypes.Structure):     # include/fdgs.h fdgs_densify_args
    _fields_ = [("P", ctypes.c_longlong), ("N", ctypes.c_int), ("gaussian_dim", ctypes.c_int), ("rot_4d", ctypes.c_int),
                ("prune_only", ctypes.c_int), ("use_max_screen_size", ctypes.c_int), ("max_grad", ctypes.c_float),
                ("min_opacity", ctypes.c_float), ("dense_extent", ctypes.c_float), ("big_extent", ctypes.c_float),
                ("max_screen_size", ctypes.c_float)] + \
               [(n, F) for n in ("xyz_gradient_accum", "denom", "max_radii2D", "xyz", "t", "scaling", "scaling_t",
                                 "rotation", "rotation_r", "opacity", "samples", "samples_t")] + \
               [("num_tensors", ctypes.c_int), ("kind", ctypes.c_int * MAXT), ("width", ctypes.c_int * MAXT),
                ("src", F * MAXT), ("dst", F * MAXT)]


def _lib():
    import fdgs
    lib = fdgs.lib()
    for n in ("fdgs_densify_plan", "fdgs_densify_apply", "fdgs_reset_opacity", "fdgs_densify_stats"):
        getattr(lib, n).restype = ctypes.c_int
    return lib


def _fake(n=1):
    """A non-null host address: the checks must fail before anything dereferences it."""
    return ctypes.cast(ctypes.pointer((ctypes.c_float * n)()), F)


def _valid_args():
    a = DensifyArgs()
    a.P, a.N, a.gaussian_dim = 10, 2, 3
    for n in ("xyz_gradient_accum", "denom", "max_radii2D", "xyz", "scaling", "rotation", "opacity"):
        setattr(a, n, _fake())
    a.num_tensors = 2
    a.kind[0], a.width[0], a.src[0], a.dst[0] = 2, 3, _fake(), _fake()       # XYZ
    a.kind[1], a.width[1], a.src[1], a.dst[1] = 0, 45, _fake(), _fake()      # COPY (f_rest)
    return a


def test_symbols_declared_exported_and_listed(repo_root):
    import fdgs
    lib = fdgs.lib()
    for s in NEW:
        assert s in _header_symbols(repo_root)
        assert s in fdgs.ABI_SYMBOLS
        assert hasattr(lib, s)
    assert lib.fdgs_version() == 2


def test_plan_and_apply_reject_null_and_inconsistent_arguments():
    lib = _lib()
    tot = (ctypes.c_int * 4)()
    assert lib.fdgs_densify_plan(None, None, tot, None) == 1
    assert b"null" in lib.fdgs_last_error()
    cases = []
    a = _valid_args(); a.scaling = None; cases.append((a, b"null"))
    a = _valid_args(); a.denom = None; cases.append((a, b"null"))
    a = _valid_args(); a.width[0] = 4; cases.append((a, b"width"))                 # xyz row of 4 floats
    a = _valid_args(); a.kind[1] = 5; a.width[1] = 3; cases.append((a, b"width"))   # scaling_t must be 1 wide
    a = _valid_args(); a.src[1] = None; cases.append((a, b"null"))
    a = _valid_args(); a.kind[0] = 9; cases.append((a, b"kind"))
    a = _valid_args(); a.N = 0; cases.append((a, b"N"))
    a = _valid_args(); a.rot_4d = 1; cases.append((a, b"gaussian_dim"))
    a = _valid_args(); a.gaussian_dim = 4; cases.append((a, b"gaussian_dim 4"))     # no t / scaling_t
    a = _valid_args(); a.num_tensors = 33; cases.append((a, b"tensor count"))
    a = _valid_args(); a.prune_only, a.use_max_screen_size, a.max_radii2D = 1, 1, None; cases.append((a, b"max_radii2D"))
    for args, msg in cases:
        assert lib.fdgs_densify_plan(ctypes.byref(args), ctypes.cast(_fake(), ctypes.c_char_p), tot, None) == 1
        assert msg in lib.fdgs_last_error(), (msg, lib.fdgs_last_error())
    a = _valid_args()
    assert lib.fdgs_densify_plan(ctypes.byref(a), None, tot, None) == 1                 # no scratch
    host = (ctypes.c_int * 4)(5, 0, 3, 3)                                                 # S = 3 split rows ...
    assert lib.fdgs_densify_apply(ctypes.byref(a), ctypes.cast(_fake(), ctypes.c_char_p), host, None) == 1
    assert b"samples" in lib.fdgs_last_error()                                            # ... but no samples
    host = (ctypes.c_int * 4)(5, 0, 3, 4)                                                 # more children kept than split
    assert lib.fdgs_densify_apply(ctypes.byref(a), ctypes.cast(_fake(), ctypes.c_char_p), host, None) == 1
    assert b"inconsistent" in lib.fdgs_last_error()
    host = (ctypes.c_int * 4)(11, 0, 0, 0)                                                # more rows than P
    assert lib.fdgs_densify_apply(ctypes.byref(a), ctypes.cast(_fake(), ctypes.c_char_p), host, None) == 1
    assert lib.fdgs_reset_opacity(ctypes.c_longlong(0), None, None, None, None) == 0     # a call that succeeds clears the error
    assert lib.fdgs_last_error() == b""


def test_reset_and_stats_reject_null_arguments():
    lib = _lib()
    assert lib.fdgs_reset_opacity(ctypes.c_longlong(5), None, None, None, None) == 1
    assert b"null" in lib.fdgs_last_error()
    assert lib.fdgs_reset_opacity(ctypes.c_longlong(0), None, None, None, None) == 0
    args = [ctypes.c_longlong(5), 1, _fake(), 3, None, ctypes.cast(_fake(), ctypes.POINTER(ctypes.c_int)), None,
            _fake(), _fake(), None, _fake(), None]
    bad = list(args); bad[7] = None                                                       # no xyz_gradient_accum
    assert lib.fdgs_densify_stats(*bad) == 1 and b"null" in lib.fdgs_last_error()
    bad = list(args); bad[1] = 4                                                          # a batch needs stride 1 + counts
    assert lib.fdgs_densify_stats(*bad) == 1 and b"stride" in lib.fdgs_last_error()
    bad = list(args); bad[6] = _fake()                                                    # t_grad without t_gradient_accum
    assert lib.fdgs_densify_stats(*bad) == 1 and b"t_grad" in lib.fdgs_last_error()
    bad = list(args); bad[3] = 1                                                          # one view: [P, >= 2] gradient
    assert lib.fdgs_densify_stats(*bad) == 1
    assert lib.fdgs_reset_opacity(ctypes.c_longlong(0), None, None, None, None) == 0


def _geo(P, dtype=torch.float32):
    return [torch.zeros(P, 3, dtype=dtype), torch.empty(0), torch.zeros(P, 3, dtype=dtype), torch.empty(0),
            torch.zeros(P, 4, dtype=dtype), torch.empty(0), torch.zeros(P, 1, dtype=dtype)]


def test_extension_rejects_wrong_dtype_layout_and_shape_before_gpu_work():
    import fdgs
    C = fdgs.ext()
    P = 8
    stats = [torch.zeros(P, 1), torch.zeros(P, 1), torch.zeros(P)]
    thr, flags = [2e-4, 0.005, 0.04, 0.4, 20.0], [2, 3, 0, 0, 1]
    with pytest.raises(RuntimeError, match="float32"):
        C.densify_plan(_geo(P, torch.float64), stats, thr, flags)
    geo = _geo(P)
    geo[0] = torch.zeros(3, P).t()                                                        # non-contiguous xyz
    with pytest.raises(RuntimeError, match="contiguous"):
        C.densify_plan(geo, stats, thr, flags)
    geo = _geo(P)
    geo[4] = torch.zeros(P, 3)                                                            # rotation rows of 3
    with pytest.raises(RuntimeError, match="shape"):
        C.densify_plan(geo, stats, thr, flags)
    with pytest.raises(RuntimeError, match="CUDA tensors"):                               # well-formed, but on the host
        C.densify_plan(_geo(P), stats, thr, flags)
    with pytest.raises(RuntimeError, match="float32"):
        C.reset_opacity(torch.zeros(P, 1, dtype=torch.float16), torch.empty(0), torch.empty(0))
    with pytest.raises(RuntimeError, match="contiguous"):
        C.densify_stats(1, torch.zeros(3, P).t(), torch.empty(0), torch.zeros(P, dtype=torch.int32), torch.empty(0),
                        torch.zeros(P, 1), torch.zeros(P, 1), torch.empty(0), torch.zeros(P))
    with pytest.raises(RuntimeError, match="int32"):
        C.densify_stats(1, torch.zeros(P, 3), torch.empty(0), torch.zeros(P, dtype=torch.int64), torch.empty(0),
                        torch.zeros(P, 1), torch.zeros(P, 1), torch.empty(0), torch.zeros(P))


def test_stats_refuse_the_reference_call_signature():
    """add_densification_stats(viewspace_point_tensor, visibility_filter, ...) -- the reference's own call -- would pass
    the zero screen-space tensor and a bool filter: refused before any GPU work instead of accumulating nothing."""
    from fdgs import densify as D

    class M:
        gaussian_dim = 3

    P = 8
    screen = torch.zeros(P, 3, requires_grad=True) + 0
    with pytest.raises(ValueError, match="viewspace_points.grad"):
        D.add_densification_stats(M(), screen, torch.zeros(P, dtype=torch.int32))
    with pytest.raises(ValueError, match="bool"):
        D.add_densification_stats(M(), torch.zeros(P, 3), torch.ones(P, dtype=torch.bool))
