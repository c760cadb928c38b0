"""H100: the rigidity and motion regularisers inside a lego-shaped training loop.

30 iterations, batch of 2 views, render() through the raw-parameter entry + L1 + lambda_rigid = 1 * L_rigid +
lambda_motion = 0.1 * L_motion, one `loss.backward()` per view.  At every iteration both arms start from the same state:
  - native: one neighbour list per iteration (fdgs.regularize.neighbours), shared by both views;
  - reference: the restatement of train.py:132-159 (tests/rigid_ref.py) with the kNN recomputed for every view by the
    reference's brute-force algorithm.
The regularisers' losses and gradients are held to the float64 bars of tests/test_gpu_rigid.py, the composed losses and
every leaf's .grad are compared between the arms, and the step is taken on the native gradients (FusedAdam, dense).
"""
import pytest
import torch

import densify_ref as DR
import rigid_ref
from test_gpu_densify_train import _Pipe, _lego_model
from test_gpu_rigid import NAMES, _native, _restated, _within_bars

pytestmark = pytest.mark.gpu
LAMBDA_RIGID, LAMBDA_MOTION, BATCH, K = 1.0, 0.1, 2, 20


def _grads(m):
    return {n: getattr(m, DR.ATTR[n]).grad.detach().clone() for n in m.group_names()}


def test_training_loop_with_native_regularisers():
    from gaussian_renderer import render
    from fdgs import regularize as R
    from fdgs.knn import knn
    dev = "cuda:0"
    m, cams, gts = _lego_model(20_000, 256, 256, dev, seed=6)
    bg = torch.zeros(3, device=dev)
    losses = []
    for it in range(1, 31):
        views = [(it * BATCH + b) % len(cams) for b in range(BATCH)]
        # native arm: one neighbour list for the iteration
        nb = R.neighbours(m.get_xyz, K)
        m.optimizer.zero_grad(set_to_none=True)
        total_nat = 0.0
        for c in views:
            img = render(cams[c], m, _Pipe(), bg)["render"]
            lr, lm = R.rigidity_and_motion_loss(m, K, nb)
            loss = ((img - gts[c]).abs().mean() + LAMBDA_RIGID * lr + LAMBDA_MOTION * lm) / BATCH
            loss.backward()
            total_nat += float(loss.detach())
        g_nat = _grads(m)
        # reference arm from the same state: the kNN recomputed per view
        m.optimizer.zero_grad(set_to_none=True)
        total_ref = 0.0
        for c in views:
            img = render(cams[c], m, _Pipe(), bg)["render"]
            xyz = m.get_xyz
            idx, dist = knn(xyz[None].contiguous().detach(), xyz[None].contiguous().detach(), K, brute_force=True)
            assert torch.equal(idx[0].int(), nb.idx) and torch.equal(dist[0], nb.dist2)
            args = (m._scaling, m._scaling_t, m._rotation, m._rotation_r, m._t)
            lr_ref = rigid_ref.rigid_loss(*args, idx[0], dist[0], K)
            lm_ref = rigid_ref.motion_loss(*args)
            loss = ((img - gts[c]).abs().mean() + LAMBDA_RIGID * lr_ref + LAMBDA_MOTION * lm_ref) / BATCH
            loss.backward()
            total_ref += float(loss.detach())
        g_ref = _grads(m)
        assert abs(total_nat - total_ref) <= 1e-5 * abs(total_ref), (it, total_nat, total_ref)
        # the regularisers alone (deterministic): value and gradients against float64, upstream lambda / batch
        p = {a: getattr(m, a).detach() for a in ("_xyz", "_t") + NAMES}
        reg_lr, reg_lm, reg_g = _native(p, nb, K)
        v32, r32, m32, g32 = _restated(p, idx[0], dist[0], torch.float32, K)
        v64, r64, m64, g64 = _restated(p, idx[0], dist[0], torch.float64, K)
        _within_bars("L_rigid", reg_lr, r32, r64)
        _within_bars("L_motion", reg_lm, m32, m64)
        for a in NAMES:
            _within_bars(a, reg_g[a], g32[a], g64[a])
        # every leaf's .grad: the arms differ by the regularisers' rounding and by the order of the blend backward's
        # float atomics (up to ~1e-4 of a gradient with cancellations, like _t's); the regulariser's share of a
        # gradient (x batch views) must be present in the native .grad
        for name, g in g_ref.items():
            d = float((g_nat[name] - g).norm())
            reg = BATCH * float(reg_g["_" + name].norm()) if "_" + name in NAMES else 0.0
            assert d <= 1e-2 * reg + 1e-3 * float(g.norm()), (it, name, d, reg, float(g.norm()))
        # step on the native gradients
        for n in m.group_names():
            getattr(m, DR.ATTR[n]).grad = g_nat[n]
        m.optimizer.step()
        losses.append(total_nat)
    assert losses[-1] < losses[0], losses
