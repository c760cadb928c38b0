"""Native rigidity and motion regularisers (csrc/regularize.cu over the C-ABI).

Drop-ins for the two loss terms of the reference's train.py:132-159 (configs/dnerf/lego.yaml:58 `lambda_rigid`, and
`lambda_motion`):

    loss = loss + opt.lambda_rigid * rigidity_loss(gaussians)
    loss = loss + opt.lambda_motion * motion_loss(gaussians)

Both are autograd functions of the model's raw parameters `_scaling`, `_scaling_t`, `_rotation` and `_rotation_r`, so
they compose with render()'s loss in one `loss.backward()` and accumulate into the leaves' `.grad`.  `_xyz` gets no
gradient (the reference's kNN input is detached) and `_t` none either (the reference's is exactly zero).  Only
`rot_4d` models have a velocity; any other model raises ValueError.

`neighbours=None` recomputes the kNN on every call, as the reference does.  The positions only change at the
optimiser step, so a training loop can build the list once per iteration with `neighbours(gaussians.get_xyz)` and
pass it to every view of the batch.  The list is not cached here: the fused optimiser writes parameters in place
without bumping their version counter, so a cache keyed on the tensor could silently go stale.

The sums run in a fixed order in double precision: values and gradients are bit-identical run to run.  Nothing here
synchronises the host.  CUDA only.
"""
from typing import Optional, Tuple

import torch

import fdgs


class Neighbours:
    """The k nearest neighbours of every Gaussian centre (the point itself first): `idx` [n,k] int32, `dist2` [n,k]
    squared distances, `weight` = exp(-100 * dist2), and the transpose -- the incoming edges of row j are
    `in_edges[in_offsets[j]:in_offsets[j+1]]`, edge id = i * k + slot, ascending."""

    __slots__ = ("k", "idx", "dist2", "weight", "in_offsets", "in_edges")

    def __init__(self, k, idx, dist2, weight, in_offsets, in_edges):
        self.k, self.idx, self.dist2, self.weight, self.in_offsets, self.in_edges = k, idx, dist2, weight, in_offsets, in_edges

    @property
    def n(self) -> int:
        return self.idx.shape[0]


def neighbours(xyz: torch.Tensor, k: int = 20) -> Neighbours:
    """The neighbour list of the positions `xyz` [n,3] (detached), for every loss call until they change."""
    C = fdgs.ext()
    x = xyz.detach().contiguous()
    idx, d2 = C.knn(x, int(k), False)
    weight, in_offsets, in_edges = C.rigid_neighbours(idx, d2)
    return Neighbours(int(k), idx, d2, weight, in_offsets, in_edges)


_build_neighbours = neighbours     # the loss functions' `neighbours` argument shadows the name


def _params(gaussians):
    if not getattr(gaussians, "rot_4d", False):
        raise ValueError("the rigidity / motion regularisers need a rot_4d model (a 3D covariance has no velocity)")
    return [gaussians._t, gaussians._scaling, gaussians._scaling_t, gaussians._rotation, gaussians._rotation_r]


class _Regularisers(torch.autograd.Function):
    @staticmethod
    def forward(ctx, scaling, scaling_t, rotation, rotation_r, t, nb, k, want_rigid, want_motion):
        params = [t.detach(), scaling.detach(), scaling_t.detach(), rotation.detach(), rotation_r.detach()]
        empty = scaling.new_empty(0)
        idx, weight = (nb.idx, nb.weight) if want_rigid else (empty.int(), empty)
        velocity, lr, lm = fdgs.ext().rigid_forward(params, k, idx, weight, want_rigid, want_motion)
        ctx.save_for_backward(*params, velocity)
        ctx.nb, ctx.k, ctx.want_rigid, ctx.want_motion = nb, k, want_rigid, want_motion
        ctx.set_materialize_grads(False)
        return lr, lm

    @staticmethod
    def backward(ctx, g_rigid, g_motion):
        t, scaling, scaling_t, rotation, rotation_r, velocity = ctx.saved_tensors
        empty = scaling.new_empty(0)
        nb = ctx.nb
        # an unrequested term is a constant 0: no gradient flows through it
        g_rigid = g_rigid if ctx.want_rigid else None
        g_motion = g_motion if ctx.want_motion else None
        if g_rigid is None and g_motion is None:
            return (None,) * 9
        lists = (nb.idx, nb.weight, nb.in_offsets, nb.in_edges) if g_rigid is not None else (empty.int(), empty, empty.int(), empty.int())
        ds, dst, dr, drr = fdgs.ext().rigid_backward([t, scaling, scaling_t, rotation, rotation_r], ctx.k, velocity, *lists,
                                                     g_rigid.contiguous() if g_rigid is not None else empty,
                                                     g_motion.contiguous() if g_motion is not None else empty)
        return ds, dst, dr, drr, None, None, None, None, None


def rigidity_and_motion_loss(gaussians, k: int = 20, neighbours: Optional[Neighbours] = None, rigid: bool = True,
                             motion: bool = True) -> Tuple[torch.Tensor, torch.Tensor]:
    """(L_rigid, L_motion) from one velocity pass (an unrequested term comes back as a constant 0)."""
    t, scaling, scaling_t, rotation, rotation_r = _params(gaussians)
    nb = None
    if rigid:
        nb = neighbours if neighbours is not None else _build_neighbours(gaussians.get_xyz, k)
        if nb.k != k or nb.n != scaling.shape[0]:
            raise ValueError("neighbour list of %d rows x %d neighbours for %d Gaussians and k = %d"
                             % (nb.n, nb.k, scaling.shape[0], k))
    return _Regularisers.apply(scaling, scaling_t, rotation, rotation_r, t, nb, int(k), bool(rigid), bool(motion))


def rigidity_loss(gaussians, k: int = 20, neighbours: Optional[Neighbours] = None) -> torch.Tensor:
    """train.py:132-152: (sum_i sum_j exp(-100 d2_ij) ||v_j - v_i||) / k / n over the k nearest neighbours."""
    return rigidity_and_motion_loss(gaussians, k, neighbours, rigid=True, motion=False)[0]


def motion_loss(gaussians) -> torch.Tensor:
    """train.py:155-159: mean_i ||v_i||."""
    return rigidity_and_motion_loss(gaussians, rigid=False, motion=True)[1]
