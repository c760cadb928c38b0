"""H100: densification inside training.

  1. A short training loop on tests/lego.py's scene (batch of 2 views, FusedAdam dense and sparse steps, native
     statistics update every iteration, densify every 50 iterations, reset_opacity once): at every densification point
     the native result equals the reference's surgery run on a copy of the same state (bit for bit, split positions
     against float64), the statistics equal the reference formulas every iteration, and training continues on the
     native result.
  2. Two NCCL ranks (skipped below two GPUs): views spread over the ranks with ViewParallelStep, statistics through
     ViewBatchStats -> add_densification_stats, densify with a generator seeded identically on every rank: the
     replicas stay bit-identical.  The same loop on one rank runs everywhere.
"""
import os
import socket

import pytest
import torch
from torch import nn

import densify_ref as R
from test_gpu_densify import _compare, _check_positions

pytestmark = pytest.mark.gpu


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False
    env_map_res = 0
    fused_prologue = True


class _TrainModel(R.Model):
    """The reference's GaussianModel over raw parameters (getters of scene/gaussian_model.py:179-219), trained with
    FusedAdam under the reference's group names."""
    get_xyz = property(lambda s: s._xyz)
    get_t = property(lambda s: s._t)
    get_scaling = property(lambda s: torch.exp(s._scaling))
    get_scaling_t = property(lambda s: torch.exp(s._scaling_t))
    get_rotation = property(lambda s: nn.functional.normalize(s._rotation))
    get_rotation_r = property(lambda s: nn.functional.normalize(s._rotation_r))
    get_opacity = property(lambda s: torch.sigmoid(s._opacity))
    get_features = property(lambda s: torch.cat((s._features_dc, s._features_rest), dim=1))


def _lego_model(P, W, H, device, seed=4):
    from fdgs.optim import FusedAdam
    from lego import lego_setup, LegoModel, lego_render
    cams, init, teacher = lego_setup(P, W, H, seed=seed)
    cams = [c.to(device) for c in cams]
    with torch.no_grad():
        tm = LegoModel({k: v.to(device) for k, v in teacher.items()})
        import lego
        old = lego.DEV
        lego.DEV = device
        try:
            gts = [lego_render(tm, c, "ours").clone() for c in cams]
        finally:
            lego.DEV = old
    m = _TrainModel()
    m.scaling_activation, m.opacity_activation, m.rotation_activation = torch.exp, torch.sigmoid, nn.functional.normalize
    m.active_sh_degree, m.active_sh_degree_t, m.time_duration = 3, 2, [0.0, 1.0]
    m.gaussian_dim, m.rot_4d, m.force_sh_3d, m.prefilter_var, m.get_max_sh_channels = 4, True, False, -1.0, 48
    m.env_map, m.percent_dense = None, 0.01
    src = dict(xyz=init["xyz"], t=init["t"], scaling=init["log_s"], scaling_t=init["log_st"], rotation=init["rot"],
               rotation_r=init["rot_r"], opacity=init["op"], f_dc=init["sh"][:, :1], f_rest=init["sh"][:, 1:])
    for n in m.group_names():
        setattr(m, R.ATTR[n], nn.Parameter(src[n].contiguous().to(device).requires_grad_(True)))
    lr = dict(xyz=1.6e-4, t=1.6e-4, f_dc=2.5e-3, f_rest=2.5e-3 / 20, opacity=5e-2, scaling=5e-3, scaling_t=5e-3,
              rotation=1e-3, rotation_r=1e-3)                       # configs/dnerf/lego.yaml:36-44
    m.optimizer = FusedAdam([{"params": [getattr(m, R.ATTR[n])], "lr": lr[n], "name": n} for n in m.group_names()],
                            lr=0.0, eps=1e-15)
    Pn = m._xyz.shape[0]
    m.xyz_gradient_accum = torch.zeros((Pn, 1), device=device)
    m.t_gradient_accum = torch.zeros((Pn, 1), device=device)
    m.denom = torch.zeros((Pn, 1), device=device)
    m.max_radii2D = torch.zeros((Pn,), device=device)
    return m, cams, gts


def _max_grad(m):
    """A gradient threshold that selects about 5 % of the seen rows (the scene's gradients are not the reference's)."""
    g = (m.xyz_gradient_accum / m.denom)[m.denom > 0]
    return float(torch.quantile(g.float(), 0.95)) if g.numel() else 1.0


class _Stats:
    """The statistics tensors alone, updated by the reference formulas (densify_ref.ref_stats)."""

    def __init__(self, m):
        self.gaussian_dim = m.gaussian_dim
        for s in ("xyz_gradient_accum", "t_gradient_accum", "denom", "max_radii2D"):
            setattr(self, s, getattr(m, s).clone())


def test_training_loop_with_native_densification():
    from gaussian_renderer import render
    from fdgs import densify as D
    from fdgs.dist import ViewBatchStats
    dev = "cuda:0"
    m, cams, gts = _lego_model(20_000, 256, 256, dev)
    bg = torch.zeros(3, device=dev)
    extent, batch, losses, points = 1.2, 2, [], []     # percent_dense * extent in the scene's scale range
    for it in range(1, 151):
        grads, radii, total = [], [], 0.0
        for b in range(batch):
            k = (it * batch + b) % len(cams)
            pkg = render(cams[k], m, _Pipe(), bg)
            loss = (pkg["render"] - gts[k]).abs().mean() / batch
            loss.backward()
            total += float(loss.detach())
            grads.append(pkg["viewspace_points"].grad.detach().clone())
            radii.append(pkg["radii"].int())
        losses.append(total)
        # statistics: native kernel against the reference formulas (train.py:168-183, 233-237)
        ref = _Stats(m)
        with torch.no_grad():
            gsum = R.ref_stats(ref, grads, radii, m._t.grad)
        st = ViewBatchStats(m._xyz.shape[0], dev)
        st.grad_norm_sum = gsum.unsqueeze(1).contiguous()
        st.visibility_count = torch.stack([r > 0 for r in radii], 1).sum(1).float().unsqueeze(1)
        st.max_radii = torch.stack(radii, 1).max(1)[0].int()
        D.add_densification_stats(m, t_grad=m._t.grad, batch_stats=st, batch_size=batch)
        for s in ("xyz_gradient_accum", "t_gradient_accum", "denom", "max_radii2D"):
            assert torch.equal(getattr(m, s), getattr(ref, s)), (it, s)
        if it % 50 == 0:
            args = (_max_grad(m), 0.005, extent, 20 if it > 50 else None)
            copy = R.clone_model(m)
            state = torch.cuda.get_rng_state()
            rec = {}
            with torch.no_grad():
                R.ref_densify_and_prune(copy, *args, record=rec)
            torch.cuda.set_rng_state(state)
            P_before = m._xyz.shape[0]
            D.densify_and_prune(m, *args)
            kids = _compare(m, copy, rec, label=("iteration", it))
            assert kids > 0 and int(rec["samples"].shape[0]) > 0, it
            torch.cuda.set_rng_state(state)
            S = rec["samples"].shape[0]
            raw = torch.randn((S, 4), device=dev)
            _check_positions(m, copy, rec, raw, None, kids, ("iteration", it))
            points.append((P_before, m._xyz.shape[0]))
        if it == 100:
            copy = R.clone_model(m)
            with torch.no_grad():
                R.ref_reset_opacity(copy)
            D.reset_opacity(m)
            _compare(m, copy, label="reset_opacity")
        # optimiser step: dense, and on every third iteration sparse over the rendered rows
        rows = torch.nonzero(m.max_radii2D > 0).squeeze(1) if it % 3 == 0 else None
        m.optimizer.step(rows=rows)
        m.optimizer.zero_grad(set_to_none=True)
    assert len(points) == 3 and all(b != a for a, b in points), points
    assert all(x == x and x < float("inf") for x in losses)
    # the opacity reset at iteration 100 throws the fit back; the loop recovers on the native result
    assert sum(losses[-10:]) < sum(losses[100:110]), "training does not continue on the densified model"
    print("densification points (P before, after):", points, "loss %.4f -> %.4f" % (losses[0], losses[-1]))


# ---- replicas across ranks -------------------------------------------------------------------------------------------
def _view_parallel_train(dev, rank, world, iters=12, nviews=4, seed=21):
    """ViewParallelStep + native statistics + densify every 4 iterations with a seeded generator; returns the model."""
    from gaussian_renderer import render
    from fdgs import densify as D
    from fdgs.dist import ViewParallelStep, shard_views
    m, cams, gts = _lego_model(8_000, 160, 160, dev)
    gen = torch.Generator(device=dev).manual_seed(seed)
    bg = torch.zeros(3, device=dev)
    splits = 0
    for it in range(1, iters + 1):
        step = ViewParallelStep(m._xyz.shape[0], dev)
        with step:
            for k in shard_views(nviews, rank, world):
                pkg = render(cams[k % len(cams)], m, _Pipe(), bg)
                ((pkg["render"] - gts[k % len(cams)]).abs().mean() / nviews).backward()
                step.add_view_stats(pkg["viewspace_points"].grad, pkg["radii"])
        stats = step.finish([m._xyz, m._t, m._scaling, m._scaling_t, m._rotation, m._rotation_r, m._opacity],
                            [m._features_dc, m._features_rest])
        D.add_densification_stats(m, t_grad=m._t.grad, batch_stats=stats, batch_size=nviews)
        if it % 4 == 0:
            P0 = m._xyz.shape[0]
            D.densify_and_prune(m, _max_grad(m), 0.005, 1.2, None, generator=gen)
            splits += int(m._xyz.shape[0] != P0)
        m.optimizer.step()
        m.optimizer.zero_grad(set_to_none=True)
    torch.cuda.synchronize(dev)
    return m, splits


def _state(m):
    out = {n: getattr(m, R.ATTR[n]).detach().cpu() for n in m.group_names()}
    for n in m.group_names():
        st = m.optimizer.state[getattr(m, R.ATTR[n])]
        out[n + ".exp_avg"], out[n + ".exp_avg_sq"] = st["exp_avg"].cpu(), st["exp_avg_sq"].cpu()
    for s in ("xyz_gradient_accum", "t_gradient_accum", "denom", "max_radii2D"):
        out[s] = getattr(m, s).cpu()
    return out


def test_view_parallel_densify_one_rank():
    m, changed = _view_parallel_train("cuda:0", 0, 1)
    assert changed > 0
    assert all(torch.isfinite(v).all() for v in _state(m).values())


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _nccl_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = "cuda:%d" % rank
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        m, changed = _view_parallel_train(dev, rank, world)
        out[rank] = (changed, _state(m))
    finally:
        dist.destroy_process_group()


def test_nccl_replicas_stay_identical_through_densification():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    world = 2
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_nccl_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    assert len(out) == world
    (c0, s0), (c1, s1) = out[0], out[1]
    assert c0 > 0 and c0 == c1
    for k in s0:
        assert torch.equal(s0[k], s1[k]), k
