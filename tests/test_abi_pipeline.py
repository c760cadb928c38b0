"""CPU: fdgs_backward checks every argument before its first CUDA call.  A call that is valid up to one of the checks
tied to the per-Gaussian backward (the rot_4d inputs, the split SH rows) is rejected with FDGS_ERR_INVALID_ARG and
queues no GPU work; the pointers below are host memory, so any launch would surface as a CUDA error instead."""
import ctypes

import pytest

F = ctypes.POINTER(ctypes.c_float)
i, f = ctypes.c_int, ctypes.c_float
FDGS_ERR_INVALID_ARG = 1


class BackwardArgs(ctypes.Structure):     # include/fdgs.h fdgs_backward_args, in order
    _fields_ = [("P", i), ("D", i), ("D_t", i), ("M", i), ("R", i), ("background", F), ("width", i), ("height", i),
                ("out_means3D", F), ("shs", F), ("colors_precomp", F), ("flows_2d", F), ("opacities", F), ("ts", F),
                ("scales", F), ("scales_t", F), ("scale_modifier", f), ("rotations", F), ("rotations_r", F),
                ("cov3D_precomp", F), ("prefilter_var", f), ("viewmatrix", F), ("projmatrix", F), ("campos", F),
                ("timestamp", f), ("time_duration", f), ("rot_4d", i), ("gaussian_dim", i), ("force_sh_3d", i),
                ("tan_fovx", f), ("tan_fovy", f), ("radii", ctypes.POINTER(ctypes.c_int)), ("geom_buffer", ctypes.c_void_p),
                ("binning_buffer", ctypes.c_void_p), ("image_buffer", ctypes.c_void_p), ("dL_dpix", F), ("dL_depths", F),
                ("dL_masks", F), ("dL_dpix_flow", F), ("debug", i), ("dL_dmean2D", F), ("dL_dconic", F),
                ("dL_dopacity", F), ("dL_dcolor", F), ("dL_dflows", F), ("dL_dmean3D", F), ("dL_dcov3D", F),
                ("dL_dsh", F), ("dL_dts", F), ("dL_dscale", F), ("dL_dscale_t", F), ("dL_drot", F), ("dL_drot_r", F),
                ("sh_factors", F), ("raw_params", i), ("shs_rest", F), ("dL_dsh_rest", F)]


_keep = []


def _fake(n=64):
    buf = (ctypes.c_float * n)()
    _keep.append(buf)
    return ctypes.cast(buf, F)


def _valid():
    """a 4D call with instances to blend (R > 0) whose every input and output is set"""
    a = BackwardArgs()
    a.P, a.D, a.D_t, a.M, a.R, a.width, a.height = 10, 3, 2, 48, 20, 32, 32
    for name in ("background", "out_means3D", "shs", "opacities", "ts", "scales", "scales_t", "rotations", "rotations_r",
                 "viewmatrix", "projmatrix", "campos", "dL_dpix", "dL_dmean2D", "dL_dconic", "dL_dopacity", "dL_dcolor",
                 "dL_dflows", "dL_dmean3D", "dL_dcov3D", "dL_dsh", "dL_dts", "dL_dscale", "dL_dscale_t", "dL_drot",
                 "dL_drot_r"):
        setattr(a, name, _fake())
    a.radii = ctypes.cast((ctypes.c_int * 64)(), ctypes.POINTER(ctypes.c_int))
    for name in ("geom_buffer", "binning_buffer", "image_buffer"):
        setattr(a, name, ctypes.cast(_fake(4096), ctypes.c_void_p))
    a.rot_4d, a.gaussian_dim, a.scale_modifier, a.time_duration, a.tan_fovx, a.tan_fovy = 1, 4, 1.0, 1.0, 1.0, 1.0
    return a


def _rot_4d_without_rotations_r():
    a = _valid()
    a.rotations_r = None
    return a


def _shs_rest_without_dL_dsh_rest():
    a = _valid()
    a.shs_rest = _fake()
    return a


def _dL_dsh_rest_without_shs_rest():
    a = _valid()
    a.dL_dsh_rest = _fake()
    return a


@pytest.mark.parametrize("make, message", [
    (_rot_4d_without_rotations_r, b"rot_4d backward needs rotations_r, scales_t, ts, opacities"),
    (_shs_rest_without_dL_dsh_rest, b"split SH rows need dL_dsh_rest"),
    (_dL_dsh_rest_without_shs_rest, b"dL_dsh_rest without shs_rest"),
], ids=["rot_4d", "shs_rest", "dL_dsh_rest"])
def test_backward_rejects_before_any_gpu_work(make, message):
    import fdgs
    lib = fdgs.lib()
    lib.fdgs_backward.restype = ctypes.c_int
    a = make()
    assert lib.fdgs_backward(ctypes.byref(a), None) == FDGS_ERR_INVALID_ARG, lib.fdgs_last_error()
    assert lib.fdgs_last_error() == message
