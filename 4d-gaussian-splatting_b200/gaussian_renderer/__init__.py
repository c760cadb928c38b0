"""`gaussian_renderer` -- drop-in replacement for the reference package of the same name.

Put `4d-gaussian-splatting_b200/` ahead of the reference checkout on PYTHONPATH and the
reference's `train.py` (`from gaussian_renderer import render`, train.py:17) picks up this
module: `render()` keeps the reference's signature and returns the same 7-key dict
(reference: gaussian_renderer/__init__.py:19-194), but rasterizes through the H100-native
CUDA library (fdgs) instead of diff-gaussian-rasterization.

`render()` only duck-types its arguments (camera / Gaussian model / pipeline flags); it does not
import the reference's `scene` or `utils` packages, so it also works stand-alone (tests, bench).
"""
import math

import torch
from torch.nn import functional as F

from .diff_gaussian_rasterization import (BatchRasterizationSettings, GaussianRasterizationSettings, GaussianRasterizer,
                                          rasterize_gaussians_batch)
from . import pyprep
from fdgs.sky import sample_sky, sample_sky_batch

__all__ = ["render", "render_batch", "GaussianRasterizationSettings", "GaussianRasterizer"]


def _select(mask, *tensors):
    return tuple(None if t is None else t[mask] for t in tensors)


def _fused_prologue_ok(pc, pipe, override_color):
    """Can this frame take the raw-parameter entry (GaussianRasterizer.forward_raw)?  Yes when the model is the
    reference's GaussianModel in its all-CUDA configuration: raw parameter tensors present, the standard activations
    (scene/gaussian_model.py:44-60: exp / sigmoid / F.normalize) and no python-side preprocessing or colour override.
    Then exp, F.normalize x2, sigmoid and the torch.cat of get_features run inside the kernels.
    pipe.fused_prologue = False forces the getter path."""
    if not getattr(pipe, "fused_prologue", True):
        return False
    if override_color is not None or pipe.compute_cov3D_python or pipe.convert_SHs_python:
        return False
    need = ["_xyz", "_scaling", "_rotation", "_opacity", "_features_dc", "_features_rest"]
    if pc.gaussian_dim == 4:
        need += ["_t", "_scaling_t"]
    if pc.rot_4d:
        need += ["_rotation_r"]
    if not all(isinstance(getattr(pc, n, None), torch.Tensor) for n in need):
        return False
    return (getattr(pc, "scaling_activation", None) is torch.exp and getattr(pc, "opacity_activation", None) is torch.sigmoid
            and getattr(pc, "rotation_activation", None) is F.normalize
            and pc._features_dc.dim() == 3 and pc._features_dc.shape[1] == 1)


def _check_sky_camera(cams):
    """The sky sampler has no camera gradient: with an environment map, a camera tensor that requires a gradient would
    receive only the rasterizer's share of it, so it is refused (ValueError)."""
    if not torch.is_grad_enabled():
        return
    for c in cams:
        for name in ("world_view_transform", "full_proj_transform", "camera_center"):
            t = getattr(c, name, None)
            if isinstance(t, torch.Tensor) and t.requires_grad:
                raise ValueError("camera %s requires a gradient, but the environment-map sky has no camera gradient: "
                                 "render without env_map_res, or detach the camera" % name)


def render(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None):
    """Render the scene from `viewpoint_camera` (background tensor must live on the GPU).

    Same contract as the reference's render(): returns {"render", "viewspace_points",
    "visibility_filter", "radii", "depth", "alpha", "flow"}.

    The camera's world_view_transform, full_proj_transform and camera_center receive gradients when they require them
    (pose refinement, INTEGRATION.md), except with an environment map (pipe.env_map_res): its sky has no camera
    gradient, and such a call raises ValueError.
    """
    xyz = pc.get_xyz
    dev = xyz.device
    # zero tensor whose .grad receives dL/d(screen-space mean) (reference: :27-31)
    screenspace_points = torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device=dev) + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass

    env_map_res = getattr(pipe, "env_map_res", 0)
    if env_map_res:
        _check_sky_camera([viewpoint_camera])
    duration = pc.time_duration[1] - pc.time_duration[0]
    settings = GaussianRasterizationSettings(
        image_height=int(viewpoint_camera.image_height),
        image_width=int(viewpoint_camera.image_width),
        tanfovx=math.tan(viewpoint_camera.FoVx * 0.5),
        tanfovy=math.tan(viewpoint_camera.FoVy * 0.5),
        bg=bg_color if not env_map_res else torch.zeros(3, device=dev),
        scale_modifier=scaling_modifier,
        viewmatrix=viewpoint_camera.world_view_transform,
        projmatrix=viewpoint_camera.full_proj_transform,
        sh_degree=pc.active_sh_degree,
        sh_degree_t=pc.active_sh_degree_t,
        campos=viewpoint_camera.camera_center,
        timestamp=viewpoint_camera.timestamp,
        time_duration=duration,
        rot_4d=pc.rot_4d,
        gaussian_dim=pc.gaussian_dim,
        force_sh_3d=pc.force_sh_3d,
        prefiltered=False,
        debug=pipe.debug,
    )
    rasterizer = GaussianRasterizer(raster_settings=settings)

    # environment-map sky (reference: :165-178): sampled by its own kernel, composed as `rendered + (1 - alpha) * sky`
    # inside the rasterizer; a ray that misses the sphere is reported once the rasterizer's forward has synchronised
    sky = sky_miss = None
    if env_map_res:
        assert pc.env_map is not None
        sky, sky_miss = sample_sky(pc.env_map, viewpoint_camera)

    if _fused_prologue_ok(pc, pipe, override_color):
        # raw-parameter entry: no activation kernels, no SH concatenation (reference: :83-91,113-119 and the getters of
        # scene/gaussian_model.py:179-219)
        four_d = pc.gaussian_dim == 4
        rendered_image, radii, depth, alpha, flow, _covs = rasterizer.forward_raw(
            means3D=xyz, means2D=screenspace_points, opacity_logits=pc._opacity, features_dc=pc._features_dc,
            features_rest=pc._features_rest if pc._features_rest.numel() else None, log_scales=pc._scaling,
            rotations_raw=pc._rotation, flow_2d=torch.zeros_like(xyz[:, :2]), ts=pc._t if four_d else None,
            log_scales_t=pc._scaling_t if four_d else None, rotations_r_raw=pc._rotation_r if pc.rot_4d else None,
            prefilter_var=pc.prefilter_var if (four_d and pc.prefilter_var > 0.0) else -1.0, bg_image=sky)
        if sky_miss is not None:
            sky_miss.check()
        return {"render": rendered_image, "viewspace_points": screenspace_points, "visibility_filter": radii > 0,
                "radii": radii, "depth": depth, "alpha": alpha, "flow": flow}

    means3D, means2D, opacity = xyz, screenspace_points, pc.get_opacity
    scales = scales_t = rotations = rotations_r = ts = cov3D_precomp = None
    prefilter_var = -1.0
    four_d = pc.gaussian_dim == 4
    py_cov = bool(pipe.compute_cov3D_python)
    marginal = None

    if py_cov:
        # covariance / mean shift / marginal in PyTorch (reference: :73-81)
        if pc.rot_4d:
            cov3D_precomp, delta_mean = pc.get_current_covariance_and_mean_offset(scaling_modifier,
                                                                                  viewpoint_camera.timestamp)
            means3D = means3D + delta_mean
        else:
            cov3D_precomp = pc.get_covariance(scaling_modifier)
        if four_d:
            marginal = pc.get_marginal_t(viewpoint_camera.timestamp)
            opacity = opacity * marginal
    else:
        # the rasterizer slices the 4D covariance itself (reference: :82-91)
        scales, rotations = pc.get_scaling, pc.get_rotation
        if four_d:
            scales_t, ts = pc.get_scaling_t, pc.get_t
            if pc.rot_4d:
                rotations_r = pc.get_rotation_r
            if pc.prefilter_var > 0.0:
                prefilter_var = pc.prefilter_var

    shs = colors_precomp = None
    if override_color is not None:
        colors_precomp = override_color
    elif pipe.convert_SHs_python:
        # SH -> RGB in PyTorch (reference: :98-111)
        feats = pc.get_features
        shs_view = feats.transpose(1, 2).view(-1, 3, pc.get_max_sh_channels)
        if py_cov:
            centres = means3D
        else:
            _, delta_mean = pc.get_current_covariance_and_mean_offset(scaling_modifier, viewpoint_camera.timestamp)
            centres = means3D + delta_mean
        dirs = (centres - viewpoint_camera.camera_center.repeat(feats.shape[0], 1)).detach()
        dirs = dirs / dirs.norm(dim=1, keepdim=True)
        if pc.gaussian_dim == 3 or pc.force_sh_3d:
            sh2rgb = pyprep.eval_sh(pc.active_sh_degree, shs_view, dirs)
        else:
            dir_t = (pc.get_t - viewpoint_camera.timestamp).detach()
            sh2rgb = pyprep.eval_shfs_4d(pc.active_sh_degree, pc.active_sh_degree_t, shs_view, dirs, dir_t, duration)
        colors_precomp = torch.clamp_min(sh2rgb + 0.5, 0.0)
    else:
        shs = pc.get_features
        if four_d and ts is None:
            ts = pc.get_t

    flow_2d = torch.zeros_like(xyz[:, :2])

    # python-side temporal prefilter (reference: :122-147)
    mask = None
    if py_cov and four_d:
        mask = marginal[:, 0] > 0.05
        (means2D, means3D, ts, shs, colors_precomp, opacity, scales, scales_t, rotations, rotations_r,
         cov3D_precomp, flow_2d) = _select(mask, means2D, means3D, ts, shs, colors_precomp, opacity, scales,
                                           scales_t, rotations, rotations_r, cov3D_precomp, flow_2d)

    rendered_image, radii, depth, alpha, flow, _covs = rasterizer(
        means3D=means3D, means2D=means2D, shs=shs, colors_precomp=colors_precomp, flow_2d=flow_2d,
        opacities=opacity, ts=ts, scales=scales, scales_t=scales_t, rotations=rotations,
        rotations_r=rotations_r, cov3D_precomp=cov3D_precomp, prefilter_var=prefilter_var, bg_image=sky)
    if sky_miss is not None:
        sky_miss.check()

    if mask is not None:
        radii_all = radii.new_zeros(mask.shape)
        radii_all[mask] = radii
    else:
        radii_all = radii

    # Gaussians that were culled or have zero radius are excluded from the densification statistics
    return {"render": rendered_image,
            "viewspace_points": screenspace_points,
            "visibility_filter": radii_all > 0,
            "radii": radii_all,
            "depth": depth,
            "alpha": alpha,
            "flow": flow}


def render_batch(viewpoint_cameras, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None):
    """Render B views of the scene in one rasterizer call per direction: one launch per stage and one host
    synchronisation for the whole batch instead of one per view.

    Returns render()'s seven keys, each stacked along a leading view dimension: "render" [B,3,H,W], "viewspace_points"
    [B,P,3] (its .grad receives every view's screen-space gradient), "visibility_filter" / "radii" [B,P], "depth" /
    "alpha" [B,1,H,W], "flow" [B,2,H,W].  View b's images and radii equal render(viewpoint_cameras[b], ...) bit for bit;
    each Gaussian's parameter gradient is the sum of the views' gradients in view order, as a sequential loop with one
    backward() per view would accumulate it.

    The views must share the image size; precomputed colours or covariances (override_color, compute_cov3D_python,
    convert_SHs_python) and a call inside an active ViewParallelStep are not supported (ValueError).

    `viewpoint_cameras` may also be an fdgs.graph.StaticViews: the cameras then come from its device tensors, the
    rasterizer is sized by its instance capacity and never synchronises with the host (the call can be captured in a CUDA
    graph), and the result has an eighth key, "status" (int32 [4] on the device: instances R, largest tile, overflow,
    wrap; on overflow every view renders as if no Gaussian were listed).  pipe.debug is not supported then (ValueError:
    it synchronises after every stage).  An environment map needs StaticViews(..., sky=True) (ValueError otherwise): the
    sky of every view is then sampled by one batched call on the views' device cameras (fdgs.sky.sample_sky_batch), and
    the result has a ninth key, "sky_miss" (int32 [1] on the device: 1 if a ray missed the sky sphere), which nothing
    here reads -- the caller asserts on it, as fdgs.graph.GraphedStep does.

    Camera tensors that require a gradient receive it as in render(): each camera's world_view_transform,
    full_proj_transform and camera_center get their view's gradient through the stack of the views' cameras (and, as
    there, not with an environment map: ValueError)."""
    from fdgs.graph import StaticViews
    views = viewpoint_cameras if isinstance(viewpoint_cameras, StaticViews) else None
    cams = None if views is not None else list(viewpoint_cameras)
    if views is None and not cams:
        raise ValueError("render_batch needs at least one camera")
    if override_color is not None:
        raise ValueError("render_batch does not take override_color (precomputed colours); use render()")
    if pipe.compute_cov3D_python:
        raise ValueError("render_batch does not support compute_cov3D_python (precomputed covariances); use render()")
    if pipe.convert_SHs_python:
        raise ValueError("render_batch does not support convert_SHs_python (precomputed colours); use render()")
    from fdgs.dist import ViewParallelStep
    if ViewParallelStep.current() is not None:
        raise ValueError("render_batch cannot run inside an active ViewParallelStep; render its views with render()")
    env_map_res = getattr(pipe, "env_map_res", 0)
    if views is not None:
        if env_map_res and getattr(views, "c2w", None) is None:
            raise ValueError("render_batch with an environment map needs StaticViews(..., sky=True): these views carry no "
                             "sky tables")
        if pipe.debug:
            raise ValueError("render_batch with StaticViews does not support pipe.debug (it synchronises after every stage)")
        B, H, W = views.B, views.H, views.W
    else:
        B, H, W = len(cams), int(cams[0].image_height), int(cams[0].image_width)
        for c in cams[1:]:
            if (int(c.image_height), int(c.image_width)) != (H, W):
                raise ValueError("render_batch views must share the image size: %dx%d and %dx%d"
                                 % (W, H, int(c.image_width), int(c.image_height)))
        if env_map_res:
            _check_sky_camera(cams)

    xyz = pc.get_xyz
    dev = xyz.device
    P = xyz.shape[0]
    screenspace_points = torch.zeros((B, P, 3), dtype=xyz.dtype, requires_grad=True, device=dev) + 0
    screenspace_points.retain_grad()

    if views is not None:
        cameras = dict(tanfovx=views.tanfovx, tanfovy=views.tanfovy, viewmatrix=views.viewmatrix,
                       projmatrix=views.projmatrix, campos=views.campos, timestamp=views.timestamp)
    else:
        cameras = dict(tanfovx=tuple(math.tan(c.FoVx * 0.5) for c in cams),
                       tanfovy=tuple(math.tan(c.FoVy * 0.5) for c in cams),
                       viewmatrix=torch.stack([c.world_view_transform for c in cams]),
                       projmatrix=torch.stack([c.full_proj_transform for c in cams]),
                       campos=torch.stack([c.camera_center for c in cams]),
                       timestamp=tuple(float(c.timestamp) for c in cams))
    settings = BatchRasterizationSettings(
        image_height=H, image_width=W,
        bg=bg_color if not env_map_res else torch.zeros(3, device=dev),
        scale_modifier=scaling_modifier,
        sh_degree=pc.active_sh_degree, sh_degree_t=pc.active_sh_degree_t,
        time_duration=pc.time_duration[1] - pc.time_duration[0],
        rot_4d=pc.rot_4d, gaussian_dim=pc.gaussian_dim, force_sh_3d=pc.force_sh_3d,
        prefiltered=False, debug=pipe.debug, **cameras)
    capacity = None if views is None else views.capacity

    sky = sky_miss = None
    misses = []
    if env_map_res and views is not None:
        assert pc.env_map is not None
        sky, sky_miss = sample_sky_batch(pc.env_map, views)
    elif env_map_res:
        assert pc.env_map is not None
        skies = []
        for c in cams:
            s, miss = sample_sky(pc.env_map, c)
            skies.append(s)
            misses.append(miss)
        sky = torch.stack(skies)

    four_d = pc.gaussian_dim == 4
    if _fused_prologue_ok(pc, pipe, None):
        out = rasterize_gaussians_batch(
            xyz, screenspace_points, pc._opacity, pc._features_dc, pc._scaling, pc._rotation, settings,
            sh_rest=pc._features_rest if pc._features_rest.numel() else None, flow_2d=torch.zeros_like(xyz[:, :2]),
            ts=pc._t if four_d else None, scales_t=pc._scaling_t if four_d else None,
            rotations_r=pc._rotation_r if pc.rot_4d else None,
            prefilter_var=pc.prefilter_var if (four_d and pc.prefilter_var > 0.0) else -1.0, raw=True, bg_image=sky,
            capacity=capacity)
    else:
        out = rasterize_gaussians_batch(
            xyz, screenspace_points, pc.get_opacity, pc.get_features, pc.get_scaling, pc.get_rotation, settings,
            flow_2d=torch.zeros_like(xyz[:, :2]), ts=pc.get_t if four_d else None,
            scales_t=pc.get_scaling_t if four_d else None, rotations_r=pc.get_rotation_r if pc.rot_4d else None,
            prefilter_var=pc.prefilter_var if (four_d and pc.prefilter_var > 0.0) else -1.0, bg_image=sky,
            capacity=capacity)
    for miss in misses:
        miss.check()
    color, radii, depth, alpha, flow = out[:5]
    pkg = {"render": color, "viewspace_points": screenspace_points, "visibility_filter": radii > 0, "radii": radii,
           "depth": depth, "alpha": alpha, "flow": flow}
    if views is not None:
        pkg["status"] = out[5]
        if sky_miss is not None:
            pkg["sky_miss"] = sky_miss
    return pkg
