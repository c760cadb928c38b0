"""Autograd boundary of the H100-native 4D Gaussian rasterizer.

Keeps the public surface of the reference's `gaussian_renderer/diff_gaussian_rasterization.py`
(reference: gaussian_renderer/diff_gaussian_rasterization.py:34-318) -- the names
`GaussianRasterizationSettings` (18 fields, same order), `GaussianRasterizer` (`forward`,
`markVisible`), `rasterize_gaussians`, the argument order, the validation errors, the 6-tuple
that comes back and the `debug` snapshot files -- so that `gaussian_renderer.render()` and the
reference's `train.py` run unchanged.

What differs is underneath: the reference JIT-compiles diff-gaussian-rasterization at import
(`:17-28`); here `_C` is the prebuilt sm_90a extension `fdgs_C.so` sitting on the C-ABI of
include/fdgs.h.  Importing this module fails loudly when that library has not been built --
there is no PyTorch or CPU fallback path.  Both entries (`GaussianRasterizer.forward` and the
raw-parameter `forward_raw`) run through one autograd Function, which calls `_C.rasterize_gaussians_ext`
and `_C.rasterize_gaussians_backward_ext`: the reference's 30 / 37 positional arguments followed by
the extensions.  So under `debug` a failing call's snapshot holds that extended argument tuple; its
first 30 (forward) or 37 (backward) entries are the reference's layout.

The camera tensors of the settings (viewmatrix, projmatrix, campos) are inputs of both autograd Functions.  When one of
them requires a gradient, the backward calls `_C.rasterize_gaussians_backward_camera` (batched:
`_C.rasterize_gaussians_backward_batch_camera`), which returns the same gradients plus the camera's
(include/fdgs.h: fdgs_backward_camera); otherwise it calls exactly what it calls without them.
"""
from typing import NamedTuple

import torch
from torch import nn

import fdgs

_C = fdgs.ext()

# an empty tensor is "not provided" (a null pointer in C) everywhere in _C; never given a gradient or written to
_NONE = torch.Tensor([])

_SNAPSHOT_MSG = {
    "snapshot_fw.dump": "\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.",
    "snapshot_bw.dump": "\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n",
}


def cpu_deep_copy_tuple(input_tuple):
    """CPU clones of every tensor in a tuple (reference: :30-32)."""
    return tuple(x.cpu().clone() if isinstance(x, torch.Tensor) else x for x in input_tuple)


def _invoke(fn, args, debug, dump_name):
    """Call into the extension; under `debug` dump the arguments on failure (reference: :122-131, :193-206)."""
    if not debug:
        return fn(*args)
    saved = cpu_deep_copy_tuple(args)  # copy before a failing kernel can corrupt them
    try:
        return fn(*args)
    except Exception:
        torch.save(saved, dump_name)
        print(_SNAPSHOT_MSG[dump_name])
        raise


def _check_bg_image(bg_image, settings, means3D):
    """A per-pixel background image must be a float32 [3, image_height, image_width] tensor on the device of the
    Gaussians; None means the constant background `settings.bg` alone."""
    if bg_image is None:
        return
    if not isinstance(bg_image, torch.Tensor):
        raise TypeError("bg_image must be a torch.Tensor, got %s" % type(bg_image).__name__)
    shape = (3, int(settings.image_height), int(settings.image_width))
    if tuple(bg_image.shape) != shape:
        raise ValueError("bg_image must have shape %s (3, image_height, image_width), got %s" % (shape, tuple(bg_image.shape)))
    if bg_image.dtype != torch.float32:
        raise ValueError("bg_image must be float32, got %s" % bg_image.dtype)
    if bg_image.device != means3D.device:
        raise ValueError("bg_image is on %s but the Gaussians are on %s" % (bg_image.device, means3D.device))


def _notify_forward(radii):
    """View-parallel step (fdgs/dist.py): the radii of a view are known after its forward -- lets the step build the
    union of rendered Gaussians behind the backward pass."""
    from fdgs.dist import ViewParallelStep
    step = ViewParallelStep.current()
    if step is not None:
        step.on_forward(radii)


def _wants_factors(sh, cov3Ds_precomp):
    """The view-parallel step (fdgs/dist.py) takes this view's SH gradient as colour factors, not dense rows."""
    from fdgs.dist import ViewParallelStep
    step = ViewParallelStep.current()
    return step is not None and step.wants_factors(sh, cov3Ds_precomp)


def _grad_sh(*sh):
    """Whether autograd will ask for the SH gradient of a call made now (inside Function.forward grad mode is off)."""
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in sh)


class GaussianRasterizationSettings(NamedTuple):
    """Per-view constants (reference: :227-245; names and order are the contract)."""
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    sh_degree_t: int
    campos: torch.Tensor
    timestamp: float
    time_duration: float
    rot_4d: bool
    gaussian_dim: int
    force_sh_3d: bool
    prefiltered: bool
    debug: bool


class _RasterizeGaussians(torch.autograd.Function):
    """reference: :67-225.  Inputs, in order: means3D, means2D, sh, sh_rest, colors_precomp, flow_2d, opacities, ts,
    scales, scales_t, rotations, rotations_r, cov3Ds_precomp, prefilter_var, raster_settings, raw, bg_image, grad_sh,
    viewmatrix, projmatrix, campos.

    raw: the raw-parameter entry (no reference counterpart; SURVEY.md section 8(f) row 1).  The inputs are then the
    optimiser's RAW parameters -- log-scales, un-normalised quaternions, opacity logits, and the SH row as the two tensors
    sh = features_dc [P,1,3] / sh_rest = features_rest [P,M-1,3] -- and the gradients come back w.r.t. exactly those, so
    the exp / F.normalize x2 / sigmoid kernels and the 1.15 GB torch.cat of the reference's getters
    (scene/gaussian_model.py:179-219), with their autograd mirror images, disappear from the frame.  Otherwise sh_rest is
    empty.  bg_image: a per-pixel background [3,H,W] behind the Gaussians, or None.  grad_sh: the caller runs under grad
    mode and the SH input requires a gradient -- the forward then allocates the dense SH gradient and its blend writes
    the zero rows of the Gaussians this view does not render, so that the backward writes only the rendered rows.
    viewmatrix, projmatrix, campos: the settings' camera tensors, passed again as inputs so that they can receive a
    gradient (the forward reads them from the settings)."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, sh_rest, colors_precomp, flow_2d, opacities, ts, scales, scales_t,
                rotations, rotations_r, cov3Ds_precomp, prefilter_var, raster_settings, raw, bg_image, grad_sh,
                viewmatrix, projmatrix, campos):
        s = raster_settings
        g_sh = g_sh_rest = _NONE
        if grad_sh and sh.numel() > 0 and colors_precomp.numel() == 0 and not _wants_factors(sh, cov3Ds_precomp):
            P = means3D.shape[0]
            g_sh = torch.empty((P, sh.shape[1], 3), dtype=torch.float32, device=means3D.device)
            if sh_rest.numel() > 0:
                g_sh_rest = torch.empty((P, sh_rest.shape[1], 3), dtype=torch.float32, device=means3D.device)
        # _C.rasterize_gaussians' positional layout (reference: :88-119, rasterize_points.h:18-49) + the extensions
        args = (s.bg, means3D, colors_precomp, flow_2d, opacities, ts, scales, scales_t, rotations, rotations_r,
                s.scale_modifier, cov3Ds_precomp, prefilter_var, s.viewmatrix, s.projmatrix, s.tanfovx, s.tanfovy,
                s.image_height, s.image_width, sh, s.sh_degree, s.sh_degree_t, s.campos, s.timestamp,
                s.time_duration, s.rot_4d, s.gaussian_dim, s.force_sh_3d, s.prefiltered, s.debug,
                sh_rest, raw, _NONE if bg_image is None else bg_image, g_sh, g_sh_rest)
        (num_rendered, color, flow, depth, T, radii, geom_buf, binning_buf, img_buf, covs_com,
         out_means3D) = _invoke(_C.rasterize_gaussians_ext, args, s.debug, "snapshot_fw.dump")

        _notify_forward(radii)
        ctx.bg_image = bg_image
        ctx.raw = raw
        ctx.raster_settings = s
        ctx.num_rendered = num_rendered
        ctx.prefilter_var = prefilter_var
        ctx.save_for_backward(colors_precomp, means3D, out_means3D, scales, rotations, cov3Ds_precomp, radii, sh, sh_rest,
                              flow_2d, opacities, ts, scales_t, rotations_r, geom_buf, binning_buf, img_buf)
        # outputs of this call, written once more by the backward: kept out of save_for_backward's version checks
        ctx.g_sh = (g_sh, g_sh_rest)
        ctx.mark_non_differentiable(radii)
        # outputs the loss does not touch arrive as None in backward() instead of zero images; the
        # library then skips their recurrences (the reference always blends all seven channels back)
        ctx.set_materialize_grads(False)
        ctx.image_shape = tuple(color.shape)
        # alpha = 1 - T (reference: :140)
        return color, radii, depth, 1 - T, flow, covs_com

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth, grad_alpha, grad_flow, grad_covs_com):
        s = ctx.raster_settings
        (colors_precomp, means3D, out_means3D, scales, rotations, cov3Ds_precomp, radii, sh, sh_rest, flow_2d, opacities,
         ts, scales_t, rotations_r, geom_buf, binning_buf, img_buf) = ctx.saved_tensors
        if grad_out_color is None:
            grad_out_color = torch.zeros(ctx.image_shape, dtype=torch.float32, device=means3D.device)
        none = torch.empty(0, dtype=torch.float32, device=means3D.device)   # "no gradient" placeholder
        grad_depth = none if grad_depth is None else grad_depth
        grad_alpha = none if grad_alpha is None else grad_alpha
        grad_flow = none if grad_flow is None else grad_flow
        # View-parallel step (fdgs/dist.py, multi-GPU): the dense dL_dsh of this view is not produced; the backward
        # emits the [P,3] colour factor of its rank-one rows and the step rebuilds / sums the rows of all views after
        # the exchange.  No reference counterpart (its views are sequential on one GPU, train.py:104-166).
        from fdgs.dist import ViewParallelStep
        step = ViewParallelStep.current()
        factors = (step is not None and step.wants_factors(sh, cov3Ds_precomp)
                   and (ctx.needs_input_grad[2] or ctx.needs_input_grad[3]))
        zeroed_sh, zeroed_sh_rest = (_NONE, _NONE) if factors else ctx.g_sh
        # once returned, the tensors belong to autograd: a second backward (retain_graph) allocates its own
        ctx.g_sh = (_NONE, _NONE)
        want_bg = ctx.needs_input_grad[16]
        want_cam = any(ctx.needs_input_grad[18:21])
        # _C.rasterize_gaussians_backward's positional layout (reference: :154-190, rasterize_points.h:51-89) + the
        # extensions
        args = (s.bg, means3D, out_means3D, radii, colors_precomp, flow_2d, opacities, ts, scales, scales_t,
                rotations, rotations_r, s.scale_modifier, cov3Ds_precomp, ctx.prefilter_var, s.viewmatrix,
                s.projmatrix, s.tanfovx, s.tanfovy, grad_out_color, grad_depth, grad_alpha, grad_flow, sh,
                s.sh_degree, s.sh_degree_t, s.campos, s.timestamp, s.time_duration, s.rot_4d, s.gaussian_dim,
                s.force_sh_3d, geom_buf, ctx.num_rendered, binning_buf, img_buf, s.debug,
                sh_rest, ctx.raw, _NONE if ctx.bg_image is None else ctx.bg_image, bool(factors), bool(want_bg),
                zeroed_sh, zeroed_sh_rest)
        g_cam = (None, None, None)
        if want_cam:
            out = _invoke(_C.rasterize_gaussians_backward_camera, args, s.debug, "snapshot_bw.dump")
            g_cam = tuple(g if need else None for g, need in zip(out[15:], ctx.needs_input_grad[18:21]))
        else:
            out = _invoke(_C.rasterize_gaussians_backward_ext, args, s.debug, "snapshot_bw.dump")
        (g_means2D, g_colors, g_opacities, g_means3D, g_cov3D, g_sh, g_flows, g_ts, g_scales, g_scales_t, g_rot, g_rot_r,
         sh_factors, g_sh_rest, g_bg) = out[:15]
        if factors:
            inputs = dict(means3D=means3D, ts=ts, scales=scales, scales_t=scales_t, rotations=rotations,
                          rotations_r=rotations_r)
            if ctx.raw:
                inputs["raw"] = True
            step.record_view(sh_factors, s, inputs)
            g_sh = g_sh_rest = None

        def for_input(grad, inp):
            # inputs passed as the empty "not provided" placeholder take no gradient
            return grad if (inp.numel() > 0 and grad is not None) else None

        # one entry per forward input (reference: :208-223); prefilter_var / settings / raw / grad_sh get None
        return (g_means3D, g_means2D, for_input(g_sh, sh), for_input(g_sh_rest, sh_rest), for_input(g_colors, colors_precomp),
                for_input(g_flows, flow_2d), g_opacities, for_input(g_ts, ts), for_input(g_scales, scales),
                for_input(g_scales_t, scales_t), for_input(g_rot, rotations), for_input(g_rot_r, rotations_r),
                for_input(g_cov3D, cov3Ds_precomp), None, None, None, g_bg if want_bg else None, None) + g_cam


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, flow_2d, opacities, ts, scales, scales_t,
                        rotations, rotations_r, cov3Ds_precomp, prefilter_var, raster_settings, bg_image=None):
    """Functional entry point (reference: :34-65).  bg_image: optional per-pixel background [3,H,W] (float32, on the
    Gaussians' device) behind the Gaussians; the image is then `rendered + (1 - alpha) * bg_image`, bit for bit, and
    bg_image receives a gradient when it requires one.  So do raster_settings.viewmatrix / projmatrix / campos: their
    gradients have their shapes (see include/fdgs.h: fdgs_backward_camera)."""
    _check_bg_image(bg_image, raster_settings, means3D)
    s = raster_settings
    return _RasterizeGaussians.apply(means3D, means2D, sh, _NONE, colors_precomp, flow_2d, opacities, ts, scales,
                                     scales_t, rotations, rotations_r, cov3Ds_precomp, prefilter_var,
                                     raster_settings, False, bg_image, _grad_sh(sh), s.viewmatrix, s.projmatrix, s.campos)


class GaussianRasterizer(nn.Module):
    """reference: :247-318"""

    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        """bool[P]: view-space z > 0.2 (reference: :252-261, auxiliary.h:140-163)."""
        with torch.no_grad():
            return _C.mark_visible(positions, self.raster_settings.viewmatrix, self.raster_settings.projmatrix)

    def forward_raw(self, means3D, means2D, opacity_logits, features_dc, features_rest, log_scales, rotations_raw,
                    flow_2d=None, ts=None, log_scales_t=None, rotations_r_raw=None, prefilter_var=-1.0, bg_image=None):
        """Same 6-tuple as forward(), from the optimiser's RAW parameters (see _RasterizeGaussians): activations and
        the SH concatenation happen inside the kernels, gradients arrive at the raw leaves directly.  bg_image: as in
        rasterize_gaussians."""
        if self.raster_settings.rot_4d and (rotations_r_raw is None or log_scales_t is None or ts is None):
            raise Exception(
                'Please provide exactly rotations_r and scales_t and ts if rot_4d and cov3D_precomp is None!')

        def opt(t):
            return torch.Tensor([]) if t is None else t

        _check_bg_image(bg_image, self.raster_settings, means3D)
        s = self.raster_settings
        return _RasterizeGaussians.apply(means3D, means2D, features_dc, opt(features_rest), _NONE, opt(flow_2d),
                                         opacity_logits, opt(ts), log_scales, opt(log_scales_t), rotations_raw,
                                         opt(rotations_r_raw), _NONE, prefilter_var, self.raster_settings, True, bg_image,
                                         _grad_sh(features_dc, features_rest), s.viewmatrix, s.projmatrix, s.campos)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, flow_2d=None, ts=None,
                scales=None, scales_t=None, rotations=None, rotations_r=None, cov3D_precomp=None,
                prefilter_var=-1.0, bg_image=None):
        """The reference's 6-tuple (color, radii, depth, alpha, flow, covs_com).  bg_image: optional per-pixel
        background behind the Gaussians (see rasterize_gaussians)."""
        # the three argument checks of the reference (:271-280), same messages
        if (shs is None) == (colors_precomp is None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        have_sr = scales is not None and rotations is not None
        any_sr = scales is not None or rotations is not None
        if (not have_sr and cov3D_precomp is None) or (any_sr and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        if self.raster_settings.rot_4d and cov3D_precomp is None and (
                rotations_r is None or scales_t is None or ts is None):
            raise Exception(
                'Please provide exactly rotations_r and scales_t and ts if rot_4d and cov3D_precomp is None!')

        # "not provided" travels as an empty CPU tensor, i.e. a null pointer in C (reference: :282-300)
        def opt(t):
            return torch.Tensor([]) if t is None else t

        return rasterize_gaussians(means3D, means2D, opt(shs), opt(colors_precomp), opt(flow_2d), opacities,
                                   opt(ts), opt(scales), opt(scales_t), opt(rotations), opt(rotations_r),
                                   opt(cov3D_precomp), prefilter_var, self.raster_settings, bg_image)


class BatchRasterizationSettings(NamedTuple):
    """What B views of one batch share, plus their per-view cameras: viewmatrix / projmatrix [B,4,4] and campos [B,3]
    CUDA tensors, tanfovx / tanfovy / timestamp sequences of B floats."""
    image_height: int
    image_width: int
    tanfovx: tuple
    tanfovy: tuple
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    sh_degree_t: int
    campos: torch.Tensor
    timestamp: tuple
    time_duration: float
    rot_4d: bool
    gaussian_dim: int
    force_sh_3d: bool
    prefiltered: bool
    debug: bool


class _RasterizeGaussiansBatch(torch.autograd.Function):
    """B views of the same Gaussians in one forward and one backward (include/fdgs.h: fdgs_forward_batch).  Inputs, in
    order: means3D, means2D [B,P,3], sh, sh_rest, flow_2d, opacities, ts, scales, scales_t, rotations, rotations_r,
    prefilter_var, settings (BatchRasterizationSettings), raw, bg_image ([B,3,H,W] or None), capacity, viewmatrix,
    projmatrix, campos.  raw and sh / sh_rest as in
    _RasterizeGaussians.  Returns color [B,3,H,W], radii [B,P], depth [B,1,H,W], alpha [B,1,H,W], flow [B,2,H,W].
    Every per-Gaussian gradient is the sum of the views' gradients in view order; means2D's gradient stays per view.

    capacity (an int >= 0) selects the entry sized by an instance capacity (_C.rasterize_gaussians_batch_capacity), which
    never synchronises with the host and can be captured in a CUDA graph: settings.timestamp / tanfovx / tanfovy are then
    float32 CUDA tensors [B], and a sixth output, status (int32 [4] on the device: R, largest tile, overflow, wrap),
    follows the five images.  On overflow the views render as if no Gaussian were listed, and the gradients are zero.

    viewmatrix, projmatrix, campos: the settings' camera tables, passed again as inputs so that they can receive a
    gradient, each view its own (rasterize_gaussians_backward_batch_camera)."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, sh_rest, flow_2d, opacities, ts, scales, scales_t, rotations, rotations_r,
                prefilter_var, settings, raw, bg_image, capacity, viewmatrix, projmatrix, campos):
        s = settings
        if capacity is None:
            cams = (s.viewmatrix, s.projmatrix, s.campos) + tuple(
                torch.tensor(list(v), dtype=torch.float32) for v in (s.timestamp, s.tanfovx, s.tanfovy))
        else:
            cams = (s.viewmatrix, s.projmatrix, s.campos, s.timestamp, s.tanfovx, s.tanfovy)
        args = (s.bg, means3D, flow_2d, opacities, ts, scales, scales_t, rotations, rotations_r, s.scale_modifier,
                prefilter_var) + cams + (s.image_height, s.image_width, sh, sh_rest, s.sh_degree, s.sh_degree_t,
                                         s.time_duration, s.rot_4d, s.gaussian_dim, s.force_sh_3d, s.prefiltered, s.debug,
                                         raw, _NONE if bg_image is None else bg_image)
        if capacity is None:
            (num_rendered, color, flow, depth, T, radii, geom_buf, binning_buf, img_buf,
             out_means3D) = _invoke(_C.rasterize_gaussians_batch, args, s.debug, "snapshot_fw.dump")
        else:
            (status, color, flow, depth, T, radii, geom_buf, binning_buf, img_buf,
             out_means3D) = _invoke(_C.rasterize_gaussians_batch_capacity, args + (int(capacity),), s.debug,
                                    "snapshot_fw.dump")
            # the backward reads the per-view scalars from the forward's geometry buffer; its binding still takes host
            # tables of the right shape
            cams = cams[:3] + (_host_placeholder(int(s.viewmatrix.shape[0])),) * 3
            num_rendered = int(capacity)
        ctx.cams = cams
        ctx.settings = s
        ctx.raw = raw
        ctx.bg_image = bg_image
        ctx.num_rendered = num_rendered
        ctx.capacity = capacity is not None
        ctx.prefilter_var = prefilter_var
        ctx.save_for_backward(means3D, out_means3D, radii, sh, sh_rest, flow_2d, opacities, ts, scales, scales_t,
                              rotations, rotations_r, geom_buf, binning_buf, img_buf)
        ctx.mark_non_differentiable(radii)
        ctx.set_materialize_grads(False)
        ctx.image_shape = tuple(color.shape)
        if capacity is None:
            return color, radii, depth, 1 - T, flow
        ctx.mark_non_differentiable(status)
        return color, radii, depth, 1 - T, flow, status

    @staticmethod
    def backward(ctx, grad_color, grad_radii, grad_depth, grad_alpha, grad_flow, grad_status=None):
        s = ctx.settings
        (means3D, out_means3D, radii, sh, sh_rest, flow_2d, opacities, ts, scales, scales_t, rotations, rotations_r,
         geom_buf, binning_buf, img_buf) = ctx.saved_tensors
        if grad_color is None:
            grad_color = torch.zeros(ctx.image_shape, dtype=torch.float32, device=means3D.device)
        none = torch.empty(0, dtype=torch.float32, device=means3D.device)   # "no gradient": the colour-only blend backward
        grad_depth = none if grad_depth is None else grad_depth
        grad_alpha = none if grad_alpha is None else grad_alpha
        grad_flow = none if grad_flow is None else grad_flow
        want_bg = ctx.needs_input_grad[14]
        want_cam = any(ctx.needs_input_grad[16:19])
        args = (s.bg, means3D, out_means3D, radii, flow_2d, opacities, ts, scales, scales_t, rotations, rotations_r,
                s.scale_modifier, ctx.prefilter_var) + ctx.cams + (
            grad_color, grad_depth, grad_alpha, grad_flow, sh, sh_rest, s.sh_degree, s.sh_degree_t, s.time_duration,
            s.rot_4d, s.gaussian_dim, s.force_sh_3d, geom_buf, ctx.num_rendered, binning_buf, img_buf, s.debug, ctx.raw,
            _NONE if ctx.bg_image is None else ctx.bg_image, bool(want_bg))
        g_cam = (None, None, None)
        if want_cam:
            out = _invoke(_C.rasterize_gaussians_backward_batch_camera, args, s.debug, "snapshot_bw.dump")
            g_cam = tuple(g if need else None for g, need in zip(out[11:], ctx.needs_input_grad[16:19]))
        else:
            out = _invoke(_C.rasterize_gaussians_backward_batch, args, s.debug, "snapshot_bw.dump")
        (g_means2D, g_opacities, g_means3D, g_sh, g_sh_rest, g_ts, g_scales, g_scales_t, g_rot, g_rot_r, g_bg) = out[:11]

        def for_input(grad, inp):
            return grad if inp.numel() > 0 else None

        return (g_means3D, g_means2D, g_sh, for_input(g_sh_rest, sh_rest), None, g_opacities, for_input(g_ts, ts),
                g_scales, for_input(g_scales_t, scales_t), g_rot, for_input(g_rot_r, rotations_r), None, None, None,
                g_bg if want_bg else None, None) + g_cam


_HOST_PLACEHOLDERS = {}


def _host_placeholder(B):
    """A float32 CPU tensor [B], built once per B: what the backward binding's host camera tables are given in capacity
    mode (the values are not read)."""
    t = _HOST_PLACEHOLDERS.get(B)
    if t is None:
        t = _HOST_PLACEHOLDERS[B] = torch.zeros(B, dtype=torch.float32)
    return t


def rasterize_gaussians_batch(means3D, means2D, opacities, sh, scales, rotations, settings, sh_rest=None, flow_2d=None,
                              ts=None, scales_t=None, rotations_r=None, prefilter_var=-1.0, raw=False, bg_image=None,
                              capacity=None):
    """Rasterize B views of the same Gaussians in one call (see _RasterizeGaussiansBatch).  raw: the inputs are the
    optimiser's raw parameters (forward_raw's convention: sh = features_dc, sh_rest = features_rest).  bg_image: per-view
    background images [B,3,H,W] behind the Gaussians, or None.  capacity: None, or the instance capacity of the entry
    that does not synchronise (the per-view scalars of `settings` are then CUDA tensors [B] and a sixth output, the
    device status, is returned).  settings.viewmatrix / projmatrix / campos receive their gradients, one per view, when
    they require them."""
    B = int(settings.viewmatrix.shape[0])
    P = int(means3D.shape[0])
    if tuple(means2D.shape) != (B, P, 3):
        raise ValueError("means2D must have shape (B, P, 3) = %s, got %s" % ((B, P, 3), tuple(means2D.shape)))
    for name in ("tanfovx", "tanfovy", "timestamp"):
        if len(getattr(settings, name)) != B:
            raise ValueError("settings.%s must hold one value per view (%d), got %d" % (name, B, len(getattr(settings, name))))
    if bg_image is not None:
        shape = (B, 3, int(settings.image_height), int(settings.image_width))
        if not isinstance(bg_image, torch.Tensor) or tuple(bg_image.shape) != shape:
            raise ValueError("bg_image must be a tensor of shape %s (B, 3, image_height, image_width)" % (shape,))
    if settings.rot_4d and (rotations_r is None or scales_t is None or ts is None):
        raise Exception('Please provide exactly rotations_r and scales_t and ts if rot_4d and cov3D_precomp is None!')

    def opt(t):
        return _NONE if t is None else t

    return _RasterizeGaussiansBatch.apply(means3D, means2D, sh, opt(sh_rest), opt(flow_2d), opacities, opt(ts), scales,
                                          opt(scales_t), rotations, opt(rotations_r), prefilter_var, settings, raw,
                                          bg_image, None if capacity is None else int(capacity), settings.viewmatrix,
                                          settings.projmatrix, settings.campos)
