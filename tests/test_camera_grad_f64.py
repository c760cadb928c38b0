"""CPU: the camera gradient's float64 restatement (camera_f64) and the C-ABI of the camera-gradient backward.

The restatement is checked against central finite differences of its own loss, on the float64 twin of a small scene with
the frustum-clamped rows removed (the reference's backward treats the clamp differently from its derivative), and
against the translation identity: moving the world and the camera by the same offset leaves the image unchanged, so
sum_i dL/dmeans3D[i] = Wt[:3,:] @ dL/dWt[3,:] + Pt[:3,:] @ dL/dPt[3,:] (no campos term: colours are precomputed).
fdgs_backward_camera / fdgs_backward_batch_camera reject null outputs, missing scratch and a bad view count with status
1 before any GPU work (called with host pointers)."""
import ctypes

import numpy as np
import pytest
import torch

import camera_f64 as CF
import helpers
import oracle_py
import regimes

NEW = ("fdgs_camera_grad_scratch_bytes", "fdgs_backward_camera", "fdgs_backward_batch_camera")


def _twin(name):
    """the twin of scene `name` without frustum-clamped rows, its oracle tile lists and masked upstream gradients"""
    cfg, cam, sc, st = helpers.build(name)
    f = oracle_py.forward(helpers.oracle_inputs(st, sc, cfg))
    _, st3, t = regimes.twin(cfg, sc, st, f)
    V = torch.as_tensor(st3["viewmatrix"]).double()
    Pm = torch.as_tensor(st3["projmatrix"]).double()
    m = torch.as_tensor(t["means3D"]).double()
    clamp = CF.project(st3, m, torch.as_tensor(t["cov3D"]).double(), V, Pm)[4].numpy()
    t = {k: np.ascontiguousarray(v[~clamp]) for k, v in t.items()}
    lists = regimes.f64_lists(oracle_py.forward(regimes.twin_oracle_inputs(st3, t)))
    grads = [helpers.to_np(g) for g in helpers.pixel_grads(cfg)]
    _, _, amb = CF.loss(st3, lists, t, grads, V, Pm)
    keep = (~amb).astype(np.float32)
    grads = [g * keep for g in grads]
    return st3, lists, t, grads


@pytest.fixture(scope="module")
def tiny():
    return _twin("tiny")


def test_restatement_matches_central_differences(tiny):
    st3, lists, t, grads = tiny
    g = CF.camera_grads(st3, lists, t, grads)
    assert not g["frustum_clamp"].any()
    V0 = torch.as_tensor(st3["viewmatrix"]).double()
    P0 = torch.as_tensor(st3["projmatrix"]).double()
    rng = np.random.default_rng(3)
    for k in range(6):
        dV = torch.from_numpy(rng.standard_normal((4, 4))) * (k % 2 == 0)
        dP = torch.from_numpy(rng.standard_normal((4, 4))) * (k % 3 != 0)
        h = 1e-7
        Lp = CF.loss(st3, lists, t, grads, V0 + h * dV, P0 + h * dP)[0].item()
        Lm = CF.loss(st3, lists, t, grads, V0 - h * dV, P0 - h * dP)[0].item()
        fd = (Lp - Lm) / (2 * h)
        an = float((g["view"] * dV.numpy()).sum() + (g["proj"] * dP.numpy()).sum())
        scale = float((np.abs(g["view"]) * np.abs(dV.numpy())).sum() + (np.abs(g["proj"]) * np.abs(dP.numpy())).sum())
        assert abs(fd - an) <= 1e-6 * scale, (k, fd, an, scale)


def test_restatement_translation_identity(tiny):
    st3, lists, t, grads = tiny
    g = CF.camera_grads(st3, lists, t, grads)
    Wt = np.asarray(st3["viewmatrix"], np.float64)
    Pt = np.asarray(st3["projmatrix"], np.float64)
    lhs = g["means3D"].sum(0)
    rhs = Wt[:3, :] @ g["view"][3, :] + Pt[:3, :] @ g["proj"][3, :]
    scale = np.abs(g["means3D"]).sum(0) + np.abs(Wt[:3, :]) @ np.abs(g["view"][3, :]) + np.abs(Pt[:3, :]) @ np.abs(g["proj"][3, :])
    assert np.all(np.abs(lhs - rhs) <= 1e-12 * scale), (lhs, rhs, scale)
    # the entries the forward does not read
    assert np.all(g["view"][:, 3] == 0) and np.all(g["proj"][:, 2] == 0)


# ---- C-ABI ---------------------------------------------------------------------------------------------------------
F = ctypes.POINTER(ctypes.c_float)


class _CamOut(ctypes.Structure):
    """include/fdgs.h: fdgs_camera_grad_out"""
    _fields_ = [("dL_dviewmatrix", F), ("dL_dprojmatrix", F), ("dL_dcampos", F), ("scratch", ctypes.c_char_p)]


def _lib():
    import fdgs
    lib = fdgs.lib()
    for n in NEW[1:]:
        getattr(lib, n).restype = ctypes.c_int
    lib.fdgs_camera_grad_scratch_bytes.restype = ctypes.c_size_t
    lib.fdgs_last_error.restype = ctypes.c_char_p
    return lib


def _fake(n=64):
    """A non-null host address: the checks must fail before anything dereferences it."""
    return ctypes.cast(ctypes.pointer((ctypes.c_float * n)()), F)


def _cam(**kw):
    c = _CamOut(dL_dviewmatrix=_fake(), dL_dprojmatrix=_fake(), dL_dcampos=_fake(), scratch=b"x" * 256)
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def test_symbols_declared_exported_and_listed(repo_root):
    import fdgs
    from test_abi_and_host import _header_symbols
    lib = _lib()
    header = _header_symbols(repo_root)
    for s in NEW:
        assert s in header and s in fdgs.ABI_SYMBOLS and hasattr(lib, s)
    assert set(header) == set(fdgs.ABI_SYMBOLS)
    assert lib.fdgs_version() == 2


def test_scratch_bytes():
    lib = _lib()
    # 27 float partials per block of 128 Gaussians per view, plus the 128-byte alignment slack
    assert lib.fdgs_camera_grad_scratch_bytes(0, 1) == 128
    assert lib.fdgs_camera_grad_scratch_bytes(1, 1) == 27 * 4 + 128
    assert lib.fdgs_camera_grad_scratch_bytes(129, 3) == 27 * 4 * 2 * 3 + 128
    assert lib.fdgs_camera_grad_scratch_bytes(2000000, 4) == 27 * 4 * 15625 * 4 + 128


def _buf(size):
    return ctypes.create_string_buffer(size)


def test_bad_arguments_are_rejected_before_gpu_work():
    from test_gpu_ctypes_abi import BwdArgs

    class _BatchArgs(ctypes.Structure):
        """include/fdgs.h: fdgs_backward_batch_args"""
        _fields_ = [("view", BwdArgs), ("B", ctypes.c_int), ("bg_image", F), ("bg_views", ctypes.c_int),
                    ("dL_dbg_image", F), ("scratch", ctypes.c_char_p)]

    lib = _lib()
    single = lambda args, cam: lib.fdgs_backward_camera(args, None, None, 0, cam, None)   # noqa: E731
    batch = lambda args, cam: lib.fdgs_backward_batch_camera(args, cam, None)            # noqa: E731
    a = BwdArgs(P=10, width=32, height=24)
    b = _BatchArgs(view=BwdArgs(P=10, width=32, height=24), B=2)
    for fn, args in ((single, ctypes.byref(a)), (batch, ctypes.byref(b))):
        assert fn(args, None) == 1 and b"camera gradient outputs" in lib.fdgs_last_error()
        for field in ("dL_dviewmatrix", "dL_dprojmatrix", "dL_dcampos", "scratch"):
            assert fn(args, ctypes.byref(_cam(**{field: None}))) == 1, field
            assert b"camera gradient outputs" in lib.fdgs_last_error()
        assert fn(None, ctypes.byref(_cam())) == 1 and b"null" in lib.fdgs_last_error()
    for B in (0, -1, 70000):
        b.B = B
        assert batch(ctypes.byref(b), ctypes.byref(_cam())) == 1 and b"view count" in lib.fdgs_last_error(), B


def test_extension_binds_the_camera_backward():
    import fdgs
    C = fdgs.ext()
    assert hasattr(C, "rasterize_gaussians_backward_camera") and hasattr(C, "rasterize_gaussians_backward_batch_camera")
