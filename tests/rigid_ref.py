"""The reference's rigidity and motion regularisers (train.py:132-159) restated in plain PyTorch, device-agnostic, in
float32 (what the reference computes) or float64 (the checker's precise evaluation of the same semantics).

    velocity = get_current_covariance_and_mean_offset(1.0, get_t + 0.1)[1]     scene/gaussian_model.py:34-47, 247-251
    L_rigid  = (exp(-100 * dist) * ||velocity[idx] - velocity[i]||).sum() / k / n
    L_motion = velocity.norm(p=2, dim=1).mean()

Spelled op for op like the reference: torch.norm-based rotation without an eps clamp (utils/general_utils.py:113-145),
the 4D covariance as L @ L^T, the `velocity[idx]` gather.  dt = (t + 0.1) - t is the reference's fp32 value in both
precisions: the timestamp t + 0.1 is an fp32 tensor there, so dt differs from 0.1 by the rounding of t + 0.1, and that
difference is part of the semantics (float64 gets the fp32 dt, promoted).  TEST INFRASTRUCTURE."""
import torch


def build_rotation_4d(l, r):
    """utils/general_utils.py:113-135"""
    l_norm = torch.norm(l, dim=-1, keepdim=True)
    r_norm = torch.norm(r, dim=-1, keepdim=True)
    q_l = l / l_norm
    q_r = r / r_norm
    a, b, c, d = q_l.unbind(-1)
    p, q, r, s = q_r.unbind(-1)
    M_l = torch.stack([a, -b, -c, -d,
                       b, a, -d, c,
                       c, d, a, -b,
                       d, -c, b, a]).view(4, 4, -1).permute(2, 0, 1)
    M_r = torch.stack([p, q, r, s,
                       -q, p, -s, r,
                       -r, s, p, -q,
                       -s, -r, q, p]).view(4, 4, -1).permute(2, 0, 1)
    A = M_l @ M_r
    return A.flip(1, 2)


def build_scaling_rotation_4d(s, l, r):
    """utils/general_utils.py:137-145"""
    L = torch.zeros((s.shape[0], 4, 4), dtype=s.dtype, device=s.device)
    R = build_rotation_4d(l, r)
    L[:, 0, 0] = s[:, 0]
    L[:, 1, 1] = s[:, 1]
    L[:, 2, 2] = s[:, 2]
    L[:, 3, 3] = s[:, 3]
    return R @ L


def reference_dt(t):
    """(t + 0.1) - t evaluated in fp32 like the reference, in t's dtype"""
    t32 = t.detach().float()
    return ((t32 + 0.1) - t32).to(t.dtype)


def velocity(scaling, scaling_t, rotation, rotation_r, t):
    """get_current_covariance_and_mean_offset(1.0, get_t + 0.1)[1] of a rot_4d model from its raw parameters
    (scaling [n,3] and scaling_t [n,1] log-scales, un-normalised quaternions [n,4], t [n,1])."""
    s = 1.0 * torch.exp(torch.cat([scaling, scaling_t], dim=1))      # scaling_modifier * get_scaling_xyzt
    L = build_scaling_rotation_4d(s, rotation, rotation_r)
    cov = L @ L.transpose(1, 2)
    cov_12 = cov[:, 0:3, 3:4]
    cov_t = cov[:, 3:4, 3:4]
    if t.dtype == torch.float32:
        dt = (t + 0.1) - t              # autograd: +g - g, an exact zero gradient for t, as in the reference
    else:
        dt = reference_dt(t) + (t - t)
    return cov_12.squeeze(-1) / cov_t.squeeze(-1) * dt


def rigid_from_velocity(vel, idx, dist, k):
    weight = torch.exp(-100 * dist)
    vel_dist = torch.norm(vel[idx] - vel[:, None], p=2, dim=-1)
    return (weight * vel_dist).sum() / k / vel.shape[0]


def motion_from_velocity(vel):
    return vel.norm(p=2, dim=1).mean()


def rigid_loss(scaling, scaling_t, rotation, rotation_r, t, idx, dist, k=20):
    """train.py:132-152 given the kNN result (idx [n,k] int64, dist [n,k] squared distances)"""
    return rigid_from_velocity(velocity(scaling, scaling_t, rotation, rotation_r, t), idx, dist.to(scaling.dtype), k)


def motion_loss(scaling, scaling_t, rotation, rotation_r, t):
    """train.py:155-159"""
    return motion_from_velocity(velocity(scaling, scaling_t, rotation, rotation_r, t))


def knn_reference(xyz, k):
    """The reference's kNN semantics (pointops2 knnquery) by brute force on the host: squared distances in fp32
    (dx*dx + dy*dy + dz*dz), ascending by (distance, index), padded with (0, 1e10) when n < k."""
    x = xyz.detach().float().cpu()
    n = x.shape[0]
    d = x[:, None, :] - x[None, :, :]
    d2 = d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2]
    order = torch.argsort(d2, dim=1, stable=True)[:, :min(k, n)]
    dist = torch.gather(d2, 1, order)
    if n < k:
        order = torch.cat([order, order.new_zeros(n, k - n)], 1)
        dist = torch.cat([dist, dist.new_full((n, k - n), 1e10)], 1)
    return order.long(), dist
