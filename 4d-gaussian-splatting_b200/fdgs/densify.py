"""Native densification: clone, split and prune as one compaction pass over the parameters and their Adam moments
(csrc/densify.cu over the C-ABI).

Drop-in for the reference's `GaussianModel.densify_and_prune` (scene/gaussian_model.py:557-577), `reset_opacity`
(:371-374) and `add_densification_stats` (:579-589, with the batch rescale and max-radius update of
train.py:168-183, 233-237).  Each function takes the model (the reference's attribute names: `_xyz`,
`_features_dc`, `_features_rest`, `_opacity`, `_scaling`, `_rotation`, `_t`, `_scaling_t`, `_rotation_r`,
`optimizer`, `xyz_gradient_accum`, `t_gradient_accum`, `denom`, `max_radii2D`, `percent_dense`, `gaussian_dim`,
`rot_4d`), finds the parameter groups by the optimiser's group names, replaces every group's leaf with a new
`nn.Parameter` and re-keys the optimiser state, like the reference.  It works with `fdgs.optim.FusedAdam` and with
`torch.optim.Adam` (whose per-parameter "step" entry is kept).

The result equals the reference's surgery bit for bit except the split children's positions and times, which are
evaluated in double and rounded once (the reference's come out of a cuBLAS bmm).  The split's normal samples are
drawn here with `torch.randn` in the reference's shapes and order, from `generator` (default: the device's default
generator, which the reference's `torch.normal` uses): the same generator state gives the reference's samples, and
ranks that share a seeded generator stay identical.  The only host synchronisation is one 16-byte read of the plan's
totals.  CUDA only.
"""
import math
from typing import Optional

import torch
from torch import nn

import fdgs

_ATTR = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
         "scaling": "_scaling", "rotation": "_rotation", "t": "_t", "scaling_t": "_scaling_t",
         "rotation_r": "_rotation_r"}
# include/fdgs.h FDGS_DENSIFY_*
COPY, MOMENT, XYZ, T, SCALING, SCALING_T = range(6)
_KIND = {"xyz": XYZ, "t": T, "scaling": SCALING, "scaling_t": SCALING_T}


def _groups(gaussians):
    out = {}
    for g in gaussians.optimizer.param_groups:
        name = g.get("name")
        if name in _ATTR:
            if len(g["params"]) != 1:
                raise ValueError("parameter group %r must hold exactly one tensor" % name)
            out[name] = g
    for name in ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation"):
        if name not in out:
            raise ValueError("the optimiser has no %r parameter group" % name)
    return out


def _rebind(gaussians, group, new_param, new_m=None, new_v=None):
    """Replace the group's leaf by `new_param` and move its optimiser state (moments replaced when given)."""
    opt = gaussians.optimizer
    old = group["params"][0]
    st = opt.state.pop(old, None)
    group["params"][0] = new_param
    if st is not None:
        if new_m is not None:
            st["exp_avg"], st["exp_avg_sq"] = new_m, new_v
        opt.state[new_param] = st
    setattr(gaussians, _ATTR[group["name"]], new_param)


def _flat(t: torch.Tensor) -> torch.Tensor:
    """[P, ...] -> [P, width] view (the kernels take row tensors)."""
    return t.view(t.shape[0], math.prod(t.shape[1:]))


def _geometry(gaussians, groups):
    def get(name):
        g = groups.get(name)
        return g["params"][0].detach() if g is not None else torch.empty(0)
    return [get("xyz"), get("t"), get("scaling"), get("scaling_t"), get("rotation"), get("rotation_r"), get("opacity")]


@torch.no_grad()
def densify_and_prune(gaussians, max_grad, min_opacity, extent, max_screen_size, max_grad_t=None, prune_only=False,
                      N: int = 2, generator: Optional[torch.Generator] = None):
    """`GaussianModel.densify_and_prune` (+ the `densify_and_clone` / `densify_and_split` / `prune_points` it calls).
    `max_grad_t` is accepted and ignored, as in the reference.  Returns the number of Gaussians after the call."""
    groups = _groups(gaussians)
    dim = int(getattr(gaussians, "gaussian_dim", 4 if "t" in groups else 3))
    rot_4d = bool(getattr(gaussians, "rot_4d", "rotation_r" in groups))
    geo = _geometry(gaussians, groups)
    P = geo[2].shape[0]
    use_screen = bool(max_screen_size)
    t_acc = getattr(gaussians, "t_gradient_accum", None) if dim == 4 else None
    stats = [gaussians.xyz_gradient_accum, gaussians.denom, gaussians.max_radii2D]
    thr = [float(max_grad), float(min_opacity), float(gaussians.percent_dense * extent), float(0.1 * extent),
           float(max_screen_size) if use_screen else 0.0]
    flags = [int(N), dim, int(rot_4d), int(bool(prune_only)), int(use_screen)]
    if prune_only:
        stats[0] = stats[1] = torch.empty(0)
    C = fdgs.ext()
    scratch, totals_d = C.densify_plan(geo, stats, thr, flags)
    totals = [int(x) for x in totals_d.cpu()]                 # the one host synchronisation
    kept, clones, S, kids = totals
    P_new = kept + clones + N * kids
    dev = geo[2].device

    samples = samples_t = torch.empty(0, device=dev)
    if not prune_only:
        # the reference's torch.normal calls (normal_(0, 1), then * std + 0), same shapes, same order
        if rot_4d:
            samples = torch.randn((S * N, 4), device=dev, generator=generator)
        else:
            samples = torch.randn((S * N, 3), device=dev, generator=generator)
            if dim == 4:
                samples_t = torch.randn((S * N, 1), device=dev, generator=generator)

    opt = gaussians.optimizer
    srcs, dsts, kinds, plan = [], [], [], []
    for name, g in groups.items():
        p = g["params"][0]
        new_p = torch.empty((P_new,) + tuple(p.shape[1:]), dtype=p.dtype, device=dev)
        srcs.append(_flat(p.detach())); dsts.append(_flat(new_p)); kinds.append(_KIND.get(name, COPY))
        st = opt.state.get(p)
        m = v = None
        if st is not None and "exp_avg" in st:
            m, v = torch.empty_like(new_p), torch.empty_like(new_p)
            for old, new in ((st["exp_avg"], m), (st["exp_avg_sq"], v)):
                srcs.append(_flat(old)); dsts.append(_flat(new)); kinds.append(MOMENT)
        plan.append((g, new_p, m, v))
    stat_names = ["xyz_gradient_accum", "denom", "max_radii2D"] + (["t_gradient_accum"] if t_acc is not None else [])
    new_stats = {}
    for name in stat_names:
        old = getattr(gaussians, name)
        if prune_only:                                        # gathered with the surviving rows
            new_stats[name] = torch.empty((P_new,) + tuple(old.shape[1:]), dtype=old.dtype, device=dev)
            srcs.append(_flat(old)); dsts.append(_flat(new_stats[name])); kinds.append(MOMENT)
        else:                                                 # densification_postfix: zeros of the new size
            new_stats[name] = torch.zeros((P_new,) + tuple(old.shape[1:]), dtype=old.dtype, device=dev)
    C.densify_apply(geo, stats, thr, flags, srcs, dsts, kinds, scratch, totals, samples, samples_t)

    for g, new_p, m, v in plan:
        _rebind(gaussians, g, nn.Parameter(new_p.requires_grad_(True)), m, v)
    for name, t in new_stats.items():
        setattr(gaussians, name, t)
    return P_new


@torch.no_grad()
def reset_opacity(gaussians):
    """`GaussianModel.reset_opacity`: opacity = inverse_sigmoid(min(sigmoid(opacity), 0.01)) and both of its Adam
    moments zeroed, in place, then the leaf replaced like the reference's replace_tensor_to_optimizer."""
    g = _groups(gaussians)["opacity"]
    p = g["params"][0]
    st = gaussians.optimizer.state.get(p)
    new_p = p.detach().clone()
    m = v = torch.empty(0)
    if st is not None and "exp_avg" in st:
        m, v = st["exp_avg"], st["exp_avg_sq"]
    fdgs.ext().reset_opacity(_flat(new_p), _flat(m) if m.numel() else m, _flat(v) if v.numel() else v)
    _rebind(gaussians, g, nn.Parameter(new_p.requires_grad_(True)))


@torch.no_grad()
def add_densification_stats(gaussians, viewspace_grad: Optional[torch.Tensor] = None, radii: Optional[torch.Tensor] = None,
                            t_grad: Optional[torch.Tensor] = None, batch_stats=None, batch_size: int = 1,
                            status: Optional[torch.Tensor] = None):
    """The densification statistics of one optimisation step in one kernel: train.py's max_radii2D update and
    `add_densification_stats` (one view: `viewspace_grad` = viewspace_points.grad, `radii` of the view) or
    `add_densification_stats_grad` with the batch rescale (`batch_stats` = fdgs.dist.ViewBatchStats of `batch_size`
    views).  `t_grad`: `_t.grad` for 4D Gaussians.  `status`: render_batch's pkg["status"] of a step sized by an
    instance capacity (fdgs.graph): when it reports an overflow nothing is accumulated."""
    C = fdgs.ext()
    dim = int(getattr(gaussians, "gaussian_dim", 3))
    t_acc = gaussians.t_gradient_accum if dim == 4 else torch.empty(0)
    tg = t_grad.reshape(-1) if (dim == 4 and t_grad is not None) else torch.empty(0)
    if dim == 4 and t_grad is None:
        raise ValueError("4D Gaussians need t_grad (the _t gradient)")
    status_arg = () if status is None else (status,)
    if batch_stats is not None:
        if batch_size < 2:
            raise ValueError("batch_stats needs batch_size >= 2")
        C.densify_stats(batch_size, batch_stats.grad_norm_sum.reshape(-1), batch_stats.visibility_count.reshape(-1),
                        batch_stats.max_radii.to(torch.int32).contiguous(), tg, gaussians.xyz_gradient_accum,
                        gaussians.denom, t_acc, gaussians.max_radii2D, *status_arg)
    else:
        if batch_size != 1 or viewspace_grad is None or radii is None:
            raise ValueError("one view needs viewspace_grad and radii (or pass batch_stats and batch_size)")
        # the reference's call passes the screen-space tensor itself and a bool visibility filter: refuse both
        if viewspace_grad.requires_grad:
            raise ValueError("viewspace_grad must be the gradient (viewspace_points.grad), not the screen-space tensor")
        if radii.dtype == torch.bool:
            raise ValueError("radii must be the view's integer radii, not the bool visibility filter")
        C.densify_stats(1, viewspace_grad, torch.empty(0), radii.to(torch.int32).contiguous(), tg,
                        gaussians.xyz_gradient_accum, gaussians.denom, t_acc, gaussians.max_radii2D, *status_arg)
