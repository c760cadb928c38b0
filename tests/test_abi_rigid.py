"""CPU: the rigidity / motion regulariser entry points of the C-ABI are declared, exported and listed; null pointers,
n <= 0, k outside [1, 32] and a backward without the forward's velocity are rejected before any GPU work; the
extension bindings check dtype, layout, shape and device first; non-rot_4d models are refused."""
import ctypes

import pytest
import torch

from test_abi_and_host import _header_symbols

NEW = ("fdgs_rigid_scratch_bytes", "fdgs_rigid_neighbours", "fdgs_rigid_forward", "fdgs_rigid_backward")
F = ctypes.POINTER(ctypes.c_float)
I = ctypes.POINTER(ctypes.c_int)


class RigidArgs(ctypes.Structure):     # include/fdgs.h fdgs_rigid_args
    _fields_ = [("n", ctypes.c_int), ("k", ctypes.c_int)] + \
               [(a, F) for a in ("t", "scaling", "scaling_t", "rotation", "rotation_r")] + \
               [("idx", I), ("weight", F), ("in_offsets", I), ("in_edges", I), ("velocity", F)]


@pytest.fixture(autouse=True)
def _clear_last_error():
    yield
    import fdgs
    assert fdgs.lib().fdgs_reset_opacity(ctypes.c_longlong(0), None, None, None, None) == 0    # a call that succeeds clears it


def _lib():
    import fdgs
    lib = fdgs.lib()
    for n in NEW[1:]:
        getattr(lib, n).restype = ctypes.c_int
    return lib


def _fake(ptr=F, n=4):
    """A non-null host address: the checks must fail before anything dereferences it."""
    base = ctypes.c_float if ptr is F else ctypes.c_int
    return ctypes.cast(ctypes.pointer((base * n)()), ptr)


def _valid():
    a = RigidArgs()
    a.n, a.k = 10, 4
    for f in ("t", "scaling", "scaling_t", "rotation", "rotation_r", "weight", "velocity"):
        setattr(a, f, _fake())
    for f in ("idx", "in_offsets", "in_edges"):
        setattr(a, f, _fake(I))
    return a


def test_symbols_declared_exported_and_listed(repo_root):
    import fdgs
    lib = fdgs.lib()
    for s in NEW:
        assert s in _header_symbols(repo_root)
        assert s in fdgs.ABI_SYMBOLS
        assert hasattr(lib, s)
    assert lib.fdgs_version() == 2
    assert lib.fdgs_rigid_scratch_bytes(1000, 20) > 0
    assert lib.fdgs_rigid_scratch_bytes(0, 20) == 0 and lib.fdgs_rigid_scratch_bytes(10, 33) == 0


def test_forward_and_backward_reject_bad_arguments():
    lib = _lib()
    scratch = ctypes.cast(_fake(), ctypes.c_char_p)
    loss = _fake()
    assert lib.fdgs_rigid_forward(None, scratch, loss, loss, None) == 1
    assert b"null" in lib.fdgs_last_error()
    cases = []
    a = _valid(); a.n = 0; cases.append((a, b"n / k"))
    a = _valid(); a.n = -3; cases.append((a, b"n / k"))
    a = _valid(); a.k = 0; cases.append((a, b"n / k"))
    a = _valid(); a.k = 33; cases.append((a, b"n / k"))
    a = _valid(); a.n = 200_000_000; a.k = 20; cases.append((a, b"2^31"))
    a = _valid(); a.scaling_t = None; cases.append((a, b"null"))
    a = _valid(); a.rotation_r = None; cases.append((a, b"null"))
    a = _valid(); a.weight = None; cases.append((a, b"idx / weight"))
    a = _valid(); a.velocity = None; cases.append((a, b"velocity"))
    for args, msg in cases:
        assert lib.fdgs_rigid_forward(ctypes.byref(args), scratch, loss, loss, None) == 1
        assert msg in lib.fdgs_last_error(), (msg, lib.fdgs_last_error())
    a = _valid()
    assert lib.fdgs_rigid_forward(ctypes.byref(a), None, loss, None, None) == 1           # no scratch
    assert b"scratch" in lib.fdgs_last_error()
    g = _fake()
    outs = [_fake() for _ in range(4)]
    bwd_cases = []
    a = _valid(); a.velocity = None; bwd_cases.append((a, g, g, outs, b"velocity"))        # no saved velocity
    a = _valid(); a.in_edges = None; bwd_cases.append((a, g, None, outs, b"in_offsets / in_edges"))
    a = _valid(); a.idx = None; bwd_cases.append((a, g, None, outs, b"idx / weight"))
    a = _valid(); a.k = 40; bwd_cases.append((a, None, g, outs, b"n / k"))
    a = _valid(); bwd_cases.append((a, g, g, [outs[0], None, outs[2], outs[3]], b"gradient outputs"))
    for args, gr, gm, o, msg in bwd_cases:
        assert lib.fdgs_rigid_backward(ctypes.byref(args), gr, gm, *o, None) == 1
        assert msg in lib.fdgs_last_error(), (msg, lib.fdgs_last_error())
    assert lib.fdgs_rigid_backward(None, g, g, *outs, None) == 1
    i, d = _fake(I), _fake()
    w, off, e = _fake(), _fake(I), _fake(I)
    assert lib.fdgs_rigid_neighbours(0, 20, i, d, scratch, w, off, e, None) == 1
    assert lib.fdgs_rigid_neighbours(10, 0, i, d, scratch, w, off, e, None) == 1
    assert lib.fdgs_rigid_neighbours(10, 4, i, d, None, w, off, e, None) == 1
    assert b"null" in lib.fdgs_last_error()
    assert lib.fdgs_rigid_neighbours(10, 4, i, d, scratch, w, off, None, None) == 1


def _params(n, dtype=torch.float32):
    return [torch.zeros(n, 1, dtype=dtype), torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 1, dtype=dtype),
            torch.zeros(n, 4, dtype=dtype), torch.zeros(n, 4, dtype=dtype)]


def test_extension_rejects_wrong_dtype_layout_shape_and_device_before_gpu_work():
    import fdgs
    C = fdgs.ext()
    n, k = 8, 4
    idx, w = torch.zeros(n, k, dtype=torch.int32), torch.zeros(n, k)
    with pytest.raises(RuntimeError, match="Float"):
        C.rigid_forward(_params(n, torch.float64), k, idx, w, True, True)
    p = _params(n)
    p[1] = torch.zeros(3, n).t()                                                        # non-contiguous scaling
    with pytest.raises(RuntimeError, match="contiguous"):
        C.rigid_forward(p, k, idx, w, True, True)
    p = _params(n)
    p[3] = torch.zeros(n, 3)                                                            # rotation rows of 3
    with pytest.raises(RuntimeError, match="shape"):
        C.rigid_forward(p, k, idx, w, True, True)
    with pytest.raises(RuntimeError, match="Int"):
        C.rigid_forward(_params(n), k, idx.long(), w, True, True)
    with pytest.raises(RuntimeError, match="shape"):
        C.rigid_forward(_params(n), k, idx[:, :2].contiguous(), w, True, True)
    with pytest.raises(RuntimeError, match="CUDA tensors"):                           # well-formed, but on the host
        C.rigid_forward(_params(n), k, idx, w, True, True)
    with pytest.raises(RuntimeError, match="velocity"):                               # the forward's velocity is required
        C.rigid_backward(_params(n), k, torch.empty(0), idx, w, torch.zeros(n + 1, dtype=torch.int32),
                         torch.zeros(n * k, dtype=torch.int32), torch.ones(()), torch.empty(0))
    with pytest.raises(RuntimeError, match="in_offsets"):
        C.rigid_backward(_params(n), k, torch.zeros(n, 3), idx, w, torch.zeros(n, dtype=torch.int32),
                         torch.zeros(n * k, dtype=torch.int32), torch.ones(()), torch.empty(0))
    with pytest.raises(RuntimeError, match="Float"):
        C.rigid_neighbours(idx, torch.zeros(n, k, dtype=torch.float64))
    with pytest.raises(RuntimeError, match="n / k"):
        C.rigid_neighbours(torch.zeros(n, 33, dtype=torch.int32), torch.zeros(n, 33))
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        C.rigid_neighbours(idx, w)


def test_models_without_rot_4d_are_refused():
    from fdgs import regularize as R

    class M:
        rot_4d = False
        gaussian_dim = 4

    with pytest.raises(ValueError, match="rot_4d"):
        R.rigidity_loss(M())
    with pytest.raises(ValueError, match="rot_4d"):
        R.motion_loss(M())
