"""fdgs -- loader for the H100-native 4D Gaussian rasterizer libraries.

`fdgs.C` is the torch extension module (`fdgs_C.so`) exposing the reference's
`_C.rasterize_gaussians / rasterize_gaussians_backward / mark_visible`
(reference: diff-gaussian-rasterization/ext.cpp:15-19), the extended pair
`rasterize_gaussians_ext / rasterize_gaussians_backward_ext` (raw parameters, per-pixel background,
view-parallel colour factors), the batched pair `rasterize_gaussians_batch / rasterize_gaussians_backward_batch` (B views
of the same Gaussians per call) and the training-step bindings; `fdgs.lib()` is the raw C-ABI
(`libfdgs.so`, include/fdgs.h) through ctypes.

There is NO fallback: if the CUDA libraries have not been built (run
`python -c "import __graft_entry__ as g; g.build()"` at the repo root) importing the extension
raises, it never silently degrades to PyTorch or CPU code.
"""
import ctypes
import importlib.util
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_DIR = os.path.join(_HERE, "lib")
LIBFDGS_PATH = os.path.join(LIB_DIR, "libfdgs.so")
EXT_PATH = os.path.join(LIB_DIR, "fdgs_C.so")

# Symbols include/fdgs.h declares (checked by tests/test_abi.py).
ABI_SYMBOLS = (
    "fdgs_version", "fdgs_last_error", "fdgs_geom_bytes", "fdgs_image_bytes", "fdgs_binning_bytes",
    "fdgs_forward", "fdgs_backward", "fdgs_mark_visible", "fdgs_debug_export_geom", "fdgs_debug_export_binning",
    "fdgs_profile_enable", "fdgs_profile_read", "fdgs_launch_count", "fdgs_pack_rows", "fdgs_unpack_rows",
    "fdgs_sh_outer_sum", "fdgs_check_rows_zero", "fdgs_l1_ssim_forward", "fdgs_l1_ssim_backward", "fdgs_adam_step",
    "fdgs_knn_scratch_bytes", "fdgs_knn", "fdgs_debug_activate", "fdgs_union_maps", "fdgs_set_tile_cull", "fdgs_view_stats",
    "fdgs_forward_bg", "fdgs_backward_bg", "fdgs_sky_forward", "fdgs_sky_backward",
    "fdgs_densify_scratch_bytes", "fdgs_densify_plan", "fdgs_densify_apply", "fdgs_reset_opacity", "fdgs_densify_stats",
    "fdgs_rigid_scratch_bytes", "fdgs_rigid_neighbours", "fdgs_rigid_forward", "fdgs_rigid_backward",
    "fdgs_metrics_scratch_bytes", "fdgs_image_metrics",
    "fdgs_geom_batch_bytes", "fdgs_image_batch_bytes", "fdgs_backward_batch_scratch_bytes", "fdgs_forward_batch",
    "fdgs_backward_batch", "fdgs_debug_export_binning_view", "fdgs_forward_zero_sh", "fdgs_backward_zero_sh",
    "fdgs_forward_batch_capacity", "fdgs_densify_stats_status", "fdgs_adam_scalars", "fdgs_adam_step_staged",
    "fdgs_sky_forward_batch", "fdgs_sky_backward_batch",
    "fdgs_camera_grad_scratch_bytes", "fdgs_backward_camera", "fdgs_backward_batch_camera",
)

STAGE_NAMES = ("preprocess_fwd", "bin_count_scan", "bin_scatter", "tile_sort_pack", "reserved", "blend_fwd", "blend_bwd",
               "preprocess_bwd")

_lib = None
_ext = None


class FdgsNotBuilt(ImportError):
    pass


def lib():
    """ctypes handle of libfdgs.so (raises FdgsNotBuilt if it has not been compiled)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIBFDGS_PATH):
            raise FdgsNotBuilt("libfdgs.so not found at %s -- run __graft_entry__.build()" % LIBFDGS_PATH)
        _lib = ctypes.CDLL(LIBFDGS_PATH, mode=ctypes.RTLD_GLOBAL)
        _lib.fdgs_version.restype = ctypes.c_int
        _lib.fdgs_last_error.restype = ctypes.c_char_p
        for n in ("fdgs_geom_bytes", "fdgs_image_bytes", "fdgs_binning_bytes"):
            getattr(_lib, n).restype = ctypes.c_size_t
        _lib.fdgs_launch_count.restype = ctypes.c_longlong
        _lib.fdgs_densify_scratch_bytes.restype = ctypes.c_size_t
        _lib.fdgs_rigid_scratch_bytes.restype = ctypes.c_size_t
        _lib.fdgs_metrics_scratch_bytes.restype = ctypes.c_size_t
    return _lib


def ext():
    """The torch extension module (the drop-in for the reference's `_C`)."""
    global _ext
    if _ext is None:
        if not os.path.exists(EXT_PATH):
            raise FdgsNotBuilt("fdgs_C.so not found at %s -- run __graft_entry__.build()" % EXT_PATH)
        import torch  # noqa: F401  (libtorch must be loaded before the extension)
        lib()  # resolve libfdgs.so first (also found through the extension's $ORIGIN rpath)
        spec = importlib.util.spec_from_file_location("fdgs_C", EXT_PATH)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        _ext = mod
    return _ext


def profile_enable(on=True):
    """Per-stage CUDA-event timing inside the library (bench.py)."""
    lib().fdgs_profile_enable(1 if on else 0)


def profile_read():
    """{stage name: (milliseconds, calls)} accumulated since the previous read."""
    ms = (ctypes.c_double * len(STAGE_NAMES))()
    calls = (ctypes.c_longlong * len(STAGE_NAMES))()
    lib().fdgs_profile_read(ms, calls)
    return {n: (ms[i], calls[i]) for i, n in enumerate(STAGE_NAMES)}


def set_tile_cull(mode) -> int:
    """1 (default): tile lists hold only the instances a pixel can blend; 0: the reference's lists exactly
    (include/fdgs.h: fdgs_set_tile_cull).  Returns the previous mode."""
    return int(lib().fdgs_set_tile_cull(1 if mode else 0))


class tile_cull:
    """Context manager: `with fdgs.tile_cull(0): ...` renders with the reference's tile lists."""

    def __init__(self, mode):
        self.mode = mode

    def __enter__(self):
        self.prev = set_tile_cull(self.mode)
        return self

    def __exit__(self, *exc):
        set_tile_cull(self.prev)
        return False


def launch_count():
    return int(lib().fdgs_launch_count())


def __getattr__(name):
    if name == "C":
        return ext()
    raise AttributeError(name)
