"""CPU: the rigidity / motion restatement (tests/rigid_ref.py) against an independent numpy float64 evaluation with a
brute-force kNN, for the values and (gradcheck) the gradients; t gets an exact zero gradient."""
import numpy as np
import pytest
import torch

import rigid_ref


def _scene(n, seed, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    p = dict(scaling=torch.log(0.02 * (0.5 + torch.rand(n, 3, generator=g))),
             scaling_t=-0.8 + 0.1 * torch.randn(n, 1, generator=g),
             rotation=torch.randn(n, 4, generator=g), rotation_r=torch.randn(n, 4, generator=g),
             t=torch.rand(n, 1, generator=g))
    xyz = (torch.rand(n, 3, generator=g) * 0.4 - 0.2)
    return {k: v.to(dtype) for k, v in p.items()}, xyz


def _numpy_velocity(p):
    """v = Sigma[0:3,3] / Sigma[3,3] * dt from the left / right quaternion matrices of the 4D rotation"""
    s = np.exp(np.concatenate([p["scaling"], p["scaling_t"]], 1))
    ql = p["rotation"] / np.sqrt((p["rotation"] ** 2).sum(1, keepdims=True))
    qr = p["rotation_r"] / np.sqrt((p["rotation_r"] ** 2).sum(1, keepdims=True))
    a, b, c, d = ql.T
    pp, q, r, ss = qr.T
    Ml = np.stack([np.stack([a, -b, -c, -d], -1), np.stack([b, a, -d, c], -1),
                   np.stack([c, d, a, -b], -1), np.stack([d, -c, b, a], -1)], 1)
    Mr = np.stack([np.stack([pp, q, r, ss], -1), np.stack([-q, pp, -ss, r], -1),
                   np.stack([-r, ss, pp, -q], -1), np.stack([-ss, -r, q, pp], -1)], 1)
    A = (Ml @ Mr)[:, ::-1, ::-1]
    assert np.allclose(A @ A.transpose(0, 2, 1), np.eye(4), atol=1e-12)        # a rotation
    sigma = np.einsum("nij,nj,nkj->nik", A, s * s, A)
    t32 = p["t"].astype(np.float32)
    dt = ((t32 + np.float32(0.1)) - t32).astype(np.float64)
    return sigma[:, 0:3, 3] / sigma[:, 3:4, 3] * dt


def _numpy_knn(xyz, k):
    x = xyz.astype(np.float32)
    d = x[:, None, :] - x[None, :, :]
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2]).astype(np.float32)
    idx = np.argsort(d2, axis=1, kind="stable")[:, :k]
    return idx, np.take_along_axis(d2, idx, 1)


@pytest.mark.parametrize("n,k", [(40, 20), (64, 8), (7, 20)])
def test_values_match_numpy_float64(n, k):
    p, xyz = _scene(n, seed=n)
    pn = {a: v.numpy() for a, v in p.items()}
    v_np = _numpy_velocity(pn)
    idx_t, dist_t = rigid_ref.knn_reference(xyz, k)
    if n >= k:
        idx_np, d_np = _numpy_knn(xyz.numpy(), k)
        assert np.array_equal(idx_t.numpy(), idx_np) and np.array_equal(dist_t.numpy(), d_np)
    idx_np, d_np = idx_t.numpy(), dist_t.numpy().astype(np.float64)
    w = np.exp(-100.0 * d_np)
    rigid_np = (w * np.linalg.norm(v_np[idx_np] - v_np[:, None], axis=-1)).sum() / k / n
    motion_np = np.linalg.norm(v_np, axis=1).mean()
    v = rigid_ref.velocity(p["scaling"], p["scaling_t"], p["rotation"], p["rotation_r"], p["t"])
    assert np.allclose(v.numpy(), v_np, rtol=1e-12, atol=1e-15)
    r = rigid_ref.rigid_loss(**p, idx=idx_t, dist=dist_t, k=k).item()
    m = rigid_ref.motion_loss(**p).item()
    assert abs(r - rigid_np) <= 1e-12 * abs(rigid_np) and abs(m - motion_np) <= 1e-12 * motion_np
    # float32: the reference's own precision, close to float64
    p32 = {a: b.float() for a, b in p.items()}
    r32 = rigid_ref.rigid_loss(**p32, idx=idx_t, dist=dist_t, k=k).item()
    assert abs(r32 - rigid_np) <= 1e-5 * abs(rigid_np)
    if n < k:     # padded entries weigh exactly 0
        assert (w[:, n:] == 0).all()


def test_gradients_gradcheck_and_zero_t_gradient():
    n, k = 24, 6
    p, xyz = _scene(n, seed=5)
    idx, dist = rigid_ref.knn_reference(xyz, k)
    leaves = [p[a].clone().requires_grad_(True) for a in ("scaling", "scaling_t", "rotation", "rotation_r")]

    def f(s, st, q, qr):
        return (rigid_ref.rigid_loss(s, st, q, qr, p["t"], idx, dist, k)
                + 0.1 * rigid_ref.motion_loss(s, st, q, qr, p["t"]))

    assert torch.autograd.gradcheck(f, leaves, eps=1e-7, atol=1e-9, rtol=1e-6)
    for dtype in (torch.float32, torch.float64):
        q = {a: v.to(dtype).clone().requires_grad_(True) for a, v in p.items()}
        loss = rigid_ref.rigid_loss(**q, idx=idx, dist=dist, k=k) + rigid_ref.motion_loss(**q)
        loss.backward()
        assert torch.equal(q["t"].grad, torch.zeros_like(q["t"]))      # +g - g: exactly zero
        assert all(q[a].grad.abs().sum() > 0 for a in ("scaling", "scaling_t", "rotation", "rotation_r"))
