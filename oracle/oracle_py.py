"""ctypes front-end of the CPU oracle (oracle/fdgs_oracle.c) + runner of the compiled reference.

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / reference arm.  The product package never imports this module.
"""
import ctypes
import importlib.util
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
BUILD = os.path.join(HERE, "_build")
LIB = os.path.join(BUILD, "libfdgs_oracle.so")
REF_SO = os.path.join(HERE, "_ref", "ref_rasterizer.so")

_lib = None


def build(force=False):
    """gcc -> oracle/_build/libfdgs_oracle.so  (-ffp-contract=off: every fmaf is explicit)."""
    src = os.path.join(HERE, "fdgs_oracle.c")
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) > os.path.getmtime(src):
        return LIB
    os.makedirs(BUILD, exist_ok=True)
    cmd = ["gcc", "-O2", "-std=c11", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-fPIC", "-shared",
           "-o", LIB, src, "-lm"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("oracle build failed:\n" + r.stdout)
    return LIB


class _Scene(ctypes.Structure):
    _fp = ctypes.POINTER(ctypes.c_float)
    _fields_ = [
        ("P", ctypes.c_int), ("D", ctypes.c_int), ("D_t", ctypes.c_int), ("M", ctypes.c_int),
        ("W", ctypes.c_int), ("H", ctypes.c_int),
        ("background", _fp), ("means3D", _fp), ("shs", _fp), ("colors_precomp", _fp), ("flows", _fp),
        ("opacities", _fp), ("ts", _fp), ("scales", _fp), ("scales_t", _fp), ("scale_modifier", ctypes.c_float),
        ("rotations", _fp), ("rotations_r", _fp), ("cov3D_precomp", _fp), ("prefilter_var", ctypes.c_float),
        ("viewmatrix", _fp), ("projmatrix", _fp), ("cam_pos", _fp),
        ("timestamp", ctypes.c_float), ("time_duration", ctypes.c_float),
        ("rot_4d", ctypes.c_int), ("gaussian_dim", ctypes.c_int), ("force_sh_3d", ctypes.c_int),
        ("tan_fovx", ctypes.c_float), ("tan_fovy", ctypes.c_float),
    ]


class _Geom(ctypes.Structure):
    _fields_ = [
        ("out_means3D", ctypes.POINTER(ctypes.c_float)), ("radii", ctypes.POINTER(ctypes.c_int)),
        ("depths", ctypes.POINTER(ctypes.c_float)), ("means2D", ctypes.POINTER(ctypes.c_float)),
        ("cov3D", ctypes.POINTER(ctypes.c_float)), ("conic_opacity", ctypes.POINTER(ctypes.c_float)),
        ("rgb", ctypes.POINTER(ctypes.c_float)), ("clamped", ctypes.POINTER(ctypes.c_uint8)),
        ("tiles_touched", ctypes.POINTER(ctypes.c_uint32)),
    ]


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(LIB)
        _lib.oracle_preprocess.restype = ctypes.c_int
        _lib.oracle_count_instances.restype = ctypes.c_int64
        _lib.oracle_bin.restype = ctypes.c_int
        _lib.oracle_num_threads.restype = ctypes.c_int
    return _lib


def _f(a):
    return None if a is None else a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def _np(t, dtype=np.float32):
    """torch tensor / array / None -> contiguous numpy array (or None if empty)."""
    if t is None:
        return None
    if hasattr(t, "detach"):
        t = t.detach().cpu().numpy()
    a = np.ascontiguousarray(t, dtype=dtype)
    return a if a.size else None


class OracleInputs:
    """Holds numpy copies of one forward call's inputs (same fields as the C-ABI fdgs_forward_args)."""

    def __init__(self, settings, means3D, opacities, shs=None, colors_precomp=None, flow_2d=None, ts=None, scales=None,
                 scales_t=None, rotations=None, rotations_r=None, cov3D_precomp=None, prefilter_var=-1.0):
        s = settings
        self.keep = dict(
            background=_np(s["bg"]), means3D=_np(means3D), shs=_np(shs), colors_precomp=_np(colors_precomp),
            flows=_np(flow_2d), opacities=_np(opacities), ts=_np(ts), scales=_np(scales), scales_t=_np(scales_t),
            rotations=_np(rotations), rotations_r=_np(rotations_r), cov3D_precomp=_np(cov3D_precomp),
            viewmatrix=_np(s["viewmatrix"]), projmatrix=_np(s["projmatrix"]), cam_pos=_np(s["campos"]))
        k = self.keep
        self.P = k["means3D"].shape[0]
        if k["flows"] is None:
            k["flows"] = np.zeros((self.P, 2), np.float32)
        self.M = 0 if k["shs"] is None else k["shs"].shape[1]
        self.W, self.H = int(s["image_width"]), int(s["image_height"])
        self.c = _Scene(
            P=self.P, D=int(s["sh_degree"]), D_t=int(s["sh_degree_t"]), M=self.M, W=self.W, H=self.H,
            background=_f(k["background"]), means3D=_f(k["means3D"]), shs=_f(k["shs"]),
            colors_precomp=_f(k["colors_precomp"]), flows=_f(k["flows"]), opacities=_f(k["opacities"]), ts=_f(k["ts"]),
            scales=_f(k["scales"]), scales_t=_f(k["scales_t"]), scale_modifier=float(s["scale_modifier"]),
            rotations=_f(k["rotations"]), rotations_r=_f(k["rotations_r"]), cov3D_precomp=_f(k["cov3D_precomp"]),
            prefilter_var=float(prefilter_var), viewmatrix=_f(k["viewmatrix"]), projmatrix=_f(k["projmatrix"]),
            cam_pos=_f(k["cam_pos"]), timestamp=float(s["timestamp"]), time_duration=float(s["time_duration"]),
            rot_4d=int(bool(s["rot_4d"])), gaussian_dim=int(s["gaussian_dim"]), force_sh_3d=int(bool(s["force_sh_3d"])),
            tan_fovx=float(s["tanfovx"]), tan_fovy=float(s["tanfovy"]))


def forward(inp: OracleInputs, stages=("preprocess", "bin", "render")):
    """Runs the oracle forward.  Returns a dict of numpy arrays named like the reference's state."""
    L = lib()
    P, W, H = inp.P, inp.W, inp.H
    out = dict(
        out_means3D=np.zeros((P, 3), np.float32), radii=np.zeros(P, np.int32), depths=np.zeros(P, np.float32),
        means2D=np.zeros((P, 2), np.float32), cov3D=np.zeros((P, 6), np.float32),
        conic_opacity=np.zeros((P, 4), np.float32), rgb=np.zeros((P, 3), np.float32),
        clamped=np.zeros((P, 3), np.uint8), tiles_touched=np.zeros(P, np.uint32))
    g = _Geom(out_means3D=_f(out["out_means3D"]), radii=out["radii"].ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
              depths=_f(out["depths"]), means2D=_f(out["means2D"]), cov3D=_f(out["cov3D"]),
              conic_opacity=_f(out["conic_opacity"]), rgb=_f(out["rgb"]),
              clamped=out["clamped"].ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)),
              tiles_touched=out["tiles_touched"].ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)))
    out["_geom"] = g
    out["num_visible"] = L.oracle_preprocess(ctypes.byref(inp.c), ctypes.byref(g))
    if "bin" not in stages:
        return out
    R = int(L.oracle_count_instances(ctypes.byref(g), P))
    gx, gy = (W + 15) // 16, (H + 15) // 16
    out["num_rendered"] = R
    out["point_list"] = np.zeros(max(R, 1), np.uint32)
    out["ranges"] = np.zeros((gx * gy, 2), np.uint32)
    rc = L.oracle_bin(P, W, H, ctypes.byref(g), ctypes.c_int64(R),
                      out["point_list"].ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)),
                      out["ranges"].ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)))
    if rc != 0:
        raise RuntimeError("oracle_bin failed: %d" % rc)
    out["point_list"] = out["point_list"][:R]
    if "render" not in stages:
        return out
    feats = inp.keep["colors_precomp"] if inp.keep["colors_precomp"] is not None else out["rgb"]
    out["final_T"] = np.zeros((H, W), np.float32)
    out["n_contrib"] = np.zeros((H, W), np.uint32)
    out["color"] = np.zeros((3, H, W), np.float32)
    out["flow"] = np.zeros((2, H, W), np.float32)
    out["depth"] = np.zeros((1, H, W), np.float32)
    u32p = ctypes.POINTER(ctypes.c_uint32)
    L.oracle_render_forward(W, H, out["ranges"].ctypes.data_as(u32p), out["point_list"].ctypes.data_as(u32p),
                            _f(out["means2D"]), _f(feats), _f(inp.keep["flows"]), _f(out["depths"]),
                            _f(out["conic_opacity"]), _f(inp.keep["background"]), _f(out["final_T"]),
                            out["n_contrib"].ctypes.data_as(u32p), _f(out["color"]), _f(out["flow"]), _f(out["depth"]))
    out["alpha"] = (1.0 - out["final_T"])[None]
    return out


def backward(inp: OracleInputs, fwd, grad_color, grad_depth, grad_alpha, grad_flow):
    """Oracle backward given the dict returned by forward().  Returns the 12 gradients as numpy arrays,
    named like the return tuple of _C.rasterize_gaussians_backward."""
    L = lib()
    P, W, H, M = inp.P, inp.W, inp.H, inp.M
    gc, gd, ga, gf = _np(grad_color), _np(grad_depth), _np(grad_alpha), _np(grad_flow)
    z = lambda *s: np.zeros(s, np.float32)
    g = dict(dL_dmeans2D=z(P, 3), dL_dcolors=z(P, 3), dL_dopacity=z(P, 1), dL_dmeans3D=z(P, 3), dL_dcov3D=z(P, 6),
             dL_dsh=z(P, max(M, 0), 3), dL_dflows=z(P, 2), dL_dts=z(P, 1), dL_dscales=z(P, 3), dL_dscales_t=z(P, 1),
             dL_drotations=z(P, 4), dL_drotations_r=z(P, 4), dL_dconic=z(P, 4))
    feats = inp.keep["colors_precomp"] if inp.keep["colors_precomp"] is not None else fwd["rgb"]
    u32p = ctypes.POINTER(ctypes.c_uint32)
    L.oracle_render_backward(W, H, fwd["ranges"].ctypes.data_as(u32p), fwd["point_list"].ctypes.data_as(u32p),
                             _f(inp.keep["background"]), _f(fwd["means2D"]), _f(fwd["conic_opacity"]), _f(feats),
                             _f(fwd["depths"]), _f(inp.keep["flows"]), _f(fwd["final_T"]),
                             fwd["n_contrib"].ctypes.data_as(u32p), _f(gc), _f(gd), _f(ga), _f(gf),
                             _f(g["dL_dmeans2D"]), _f(g["dL_dconic"]), _f(g["dL_dopacity"]), _f(g["dL_dcolors"]),
                             _f(g["dL_dflows"]))
    cov = inp.keep["cov3D_precomp"] if inp.keep["cov3D_precomp"] is not None else fwd["cov3D"]
    L.oracle_preprocess_backward(ctypes.byref(inp.c), _f(fwd["out_means3D"]),
                                 fwd["radii"].ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                                 fwd["clamped"].ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)),
                                 fwd["tiles_touched"].ctypes.data_as(u32p), _f(cov), _f(g["dL_dmeans2D"]),
                                 _f(g["dL_dconic"]), _f(g["dL_dopacity"]), _f(g["dL_dcolors"]), _f(g["dL_dmeans3D"]),
                                 _f(g["dL_dcov3D"]), _f(g["dL_dsh"]), _f(g["dL_dts"]), _f(g["dL_dscales"]),
                                 _f(g["dL_dscales_t"]), _f(g["dL_drotations"]), _f(g["dL_drotations_r"]))
    return g


def camera_terms(inp: OracleInputs, fwd, grads):
    """The camera's 27 per-row gradient terms [P,27] (oracle_camera_terms, zero on the rows not rendered), from the
    forward's dict and the dict backward() returned (its blend gradients dL_dmeans2D, dL_dconic and dL_dcolors)."""
    L = lib()
    u32p = ctypes.POINTER(ctypes.c_uint32)
    terms = np.zeros((inp.P, 27), np.float32)
    cov = inp.keep["cov3D_precomp"] if inp.keep["cov3D_precomp"] is not None else fwd["cov3D"]
    L.oracle_camera_terms(ctypes.byref(inp.c), _f(fwd["out_means3D"]),
                          fwd["radii"].ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                          fwd["clamped"].ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)),
                          fwd["tiles_touched"].ctypes.data_as(u32p), _f(cov), _f(grads["dL_dmeans2D"]),
                          _f(grads["dL_dconic"]), _f(grads["dL_dcolors"]), _f(terms))
    return terms


def num_threads():
    return int(lib().oracle_num_threads())


def set_num_threads(n):
    """n <= 0: back to all host cores"""
    lib().oracle_set_num_threads(int(n))


# ---- the compiled, unmodified reference (oracle/_ref) ----------------------------------------------
_ref = None


REF_VARIANT = ""      # "nofma": the -fmad=false build (oracle/_ref/nofma), for tools/capture_reference.py


def ref_available():
    """the module exists and was compiled with oracle/build_ref.py's current flags (not, e.g., for another GPU)"""
    import build_ref
    return build_ref.current(REF_VARIANT)


def ref_module():
    """The reference's own extension module (rasterize_gaussians / _backward / mark_visible),
    built from /root/reference by oracle/build_ref.py.  GPU only."""
    global _ref
    if _ref is None:
        if not ref_available():
            raise ImportError("oracle/_ref/ref_rasterizer.so not built (oracle/build_ref.py)")
        import torch  # noqa: F401
        spec = importlib.util.spec_from_file_location(
            "ref_rasterizer", os.path.join(HERE, "_ref", REF_VARIANT, "ref_rasterizer.so") if REF_VARIANT else REF_SO)
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        _ref = m
    return _ref


def ref_geom_views(geom_buffer, P):
    """Views into the reference's geomBuffer, carved exactly like GeometryState::fromChunk
    (reference: rasterizer_impl.cu:156-171; 128-byte aligned sub-arrays, rasterizer_impl.h:21-27):
    depths f32[P], clamped bool[3P], internal_radii i32[P], means2D f32[2P], cov3D f32[6P],
    conic_opacity f32[4P], rgb f32[3P], tiles_touched u32[P]."""
    import torch
    base = geom_buffer.data_ptr()
    off = 0
    views = {}

    def take(name, nbytes, dtype, shape):
        nonlocal off
        addr = (base + off + 127) & ~127
        off = addr - base
        views[name] = geom_buffer[off:off + nbytes].view(dtype).view(*shape)
        off += nbytes

    take("depths", 4 * P, torch.float32, (P,))
    take("clamped", 3 * P, torch.uint8, (P, 3))
    take("internal_radii", 4 * P, torch.int32, (P,))
    take("means2D", 8 * P, torch.float32, (P, 2))
    take("cov3D", 24 * P, torch.float32, (P, 6))
    take("conic_opacity", 16 * P, torch.float32, (P, 4))
    take("rgb", 12 * P, torch.float32, (P, 3))
    take("tiles_touched", 4 * P, torch.int32, (P,))
    return views


def ref_binning_point_list(binning_buffer, R):
    """point_list u32[R] is the first array of BinningState (rasterizer_impl.cu:182-195)."""
    import torch
    base = binning_buffer.data_ptr()
    off = ((base + 127) & ~127) - base
    return binning_buffer[off:off + 4 * R].view(torch.int32)


def ref_image_views(img_buffer, N):
    """accum_alpha f32[N], n_contrib u32[N], ranges uint2[N] (rasterizer_impl.cu:173-180)."""
    import torch
    base = img_buffer.data_ptr()
    off = 0
    views = {}
    for name, nbytes, dtype in (("accum_alpha", 4 * N, torch.float32), ("n_contrib", 4 * N, torch.int32),
                                ("ranges", 8 * N, torch.int32)):
        addr = (base + off + 127) & ~127
        off = addr - base
        views[name] = img_buffer[off:off + nbytes].view(dtype)
        off += nbytes
    views["ranges"] = views["ranges"].view(-1, 2)
    return views
