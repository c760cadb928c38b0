"""GPU (-m gpu): the camera gradients of the rasterizer backward (include/fdgs.h: fdgs_backward_camera).

  1. translation identity: sum_i dL/dmeans3D[i] + dL/dcampos = Wt[:3,:] @ dL/dWt[3,:] + Pt[:3,:] @ dL/dPt[3,:] on every
     call: 3D and 4D rot_4d scenes with SH degree 3 / D_t = 2, activated and raw entries, colour-only and AUX (depth +
     alpha), both tile-list modes, a per-pixel background, and the batched entry (both sides summed over the views);
  2. float64: on the 3D twin of a scene (camera_f64, ambiguous pixels masked, frustum-clamped rows removed), each
     matrix gradient against the restatement, normwise, within K times the same call's normwise error of dL_dmeans2D;
  3. batch: each view's gradients equal the single-view call on that camera within the blend backward's run-to-run
     spread;
  4. off means off: camera tensors that need no gradient run the existing backward (same launches, no camera gradient);
  5. refusals: an environment map with a camera that requires a gradient raises ValueError; with precomputed colours
     campos gets exactly 0;
  6. pose recovery: a 2 degree / 2 % perturbation of the camera is undone by Adam on a 6-DoF delta through render() and
     render_batch() with an L1 loss."""
import math

import numpy as np
import pytest
import torch

import camera_f64 as CF
import helpers
import regimes
from test_gpu_batch import _inputs
from test_gpu_view_parallel import DEV, _Model, _env, _pipe, _views

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -24


def _rast_settings(st, **kw):
    from gaussian_renderer import GaussianRasterizationSettings
    d = dict(st)
    d.update(kw)
    return GaussianRasterizationSettings(**{k: d[k] for k in GaussianRasterizationSettings._fields})


def _leaf(t):
    return t.detach().clone().requires_grad_(True)


def _loss(cfg, color, depth, alpha, aux):
    gc, gd, ga, _ = helpers.pixel_grads(cfg, device=DEV)
    L = (color * gc.reshape(color.shape[-3:])).sum()
    if aux:
        L = L + (depth * gd.reshape(depth.shape[-3:])).sum() + (alpha * ga.reshape(alpha.shape[-3:])).sum()
    return L


def _single(name, raw=False, aux=False, bgi=False, colors=False):
    """one render + backward with learnable camera tensors; returns the gradients (float64 CPU) and the camera"""
    from gaussian_renderer import GaussianRasterizer
    cfg, cam, sc, st = helpers.build(name, device=DEV)
    V, Pm, c = _leaf(st["viewmatrix"]), _leaf(st["projmatrix"]), _leaf(st["campos"])
    rast = GaussianRasterizer(_rast_settings(st, viewmatrix=V, projmatrix=Pm, campos=c))
    means = _leaf(sc.means3D)
    m2 = torch.zeros_like(means, requires_grad=True)
    bg_image = torch.rand(3, cfg["H"], cfg["W"], generator=torch.Generator().manual_seed(4)).to(DEV) if bgi else None
    four = sc.gaussian_dim == 4
    if raw:
        g = _inputs(sc, True, True)
        out = rast.forward_raw(means, m2, g["opacity"], g["sh"], g["sh_rest"], g["scales"], g["rotations"],
                               flow_2d=sc.flow_2d, ts=sc.ts if four else None, log_scales_t=g["scales_t"] if four else None,
                               rotations_r_raw=g["rotations_r"] if sc.rot_4d else None, bg_image=bg_image)
    else:
        kw = dict(colors_precomp=torch.rand(sc.P, 3, generator=torch.Generator().manual_seed(5)).to(DEV)) if colors \
            else dict(shs=sc.shs)
        out = rast(means, m2, sc.opacities, flow_2d=sc.flow_2d, ts=sc.ts, scales=sc.scales,
                   scales_t=sc.scales_t if four else None, rotations=sc.rotations,
                   rotations_r=sc.rotations_r if sc.rot_4d else None, bg_image=bg_image, **kw)
    color, radii, depth, alpha = out[:4]
    _loss(cfg, color, depth, alpha, aux).backward()
    d = lambda t: t.detach().double().cpu()
    return dict(means3D=d(means.grad), V=d(V), P=d(Pm), dV=d(V.grad), dP=d(Pm.grad), dc=d(c.grad), means2D=d(m2.grad))


def _identity(gs):
    """both sides of the translation identity summed over the calls in gs, and the scale of their terms"""
    lhs = sum(g["means3D"].sum(0) + g["dc"] for g in gs)
    rhs = sum(g["V"][:3, :] @ g["dV"][3, :] + g["P"][:3, :] @ g["dP"][3, :] for g in gs)
    scale = sum(g["means3D"].abs().sum(0) + g["dc"].abs() + g["V"][:3, :].abs() @ g["dV"][3, :].abs()
                + g["P"][:3, :].abs() @ g["dP"][3, :].abs() for g in gs)
    return lhs, rhs, scale


def _check_identity(label, gs, K=64):
    lhs, rhs, scale = _identity(gs)
    err = (lhs - rhs).abs()
    print("%-28s identity err / (eps * sum|terms|): %s" % (label, (err / (EPS * scale)).numpy().round(2)))
    assert torch.all(err <= K * EPS * scale), (label, lhs, rhs, scale)
    for g in gs:
        assert torch.all(g["dV"][:, 3] == 0) and torch.all(g["dP"][:, 2] == 0)


@pytest.mark.parametrize("name", ["small", "dim3", "rotcam"])
@pytest.mark.parametrize("raw", [False, True])
@pytest.mark.parametrize("aux", [False, True])
def test_translation_identity(name, raw, aux):
    _check_identity("%s raw=%d aux=%d" % (name, raw, aux), [_single(name, raw=raw, aux=aux)])


@pytest.mark.parametrize("cull", [0, 1])
def test_translation_identity_tile_modes_and_background(cull):
    import fdgs
    lib = fdgs.lib()
    old = lib.fdgs_set_tile_cull(cull)
    try:
        _check_identity("tile_cull=%d bg_image" % cull, [_single("flowbg", aux=True, bgi=True)])
    finally:
        lib.fdgs_set_tile_cull(old)


def _batch(name, n=3, raw=False, grad=True):
    """rasterize_gaussians_batch over n views with learnable stacked cameras"""
    from gaussian_renderer import BatchRasterizationSettings, rasterize_gaussians_batch
    from fdgs import synth
    cfg, _, sc, _ = helpers.build(name, device=DEV)
    cams = _views(cfg, n, DEV)
    sts = [synth.raster_settings(c, sc, bg=torch.zeros(3), device=DEV) for c in cams]
    V = torch.stack([s["viewmatrix"] for s in sts]).requires_grad_(grad)
    Pm = torch.stack([s["projmatrix"] for s in sts]).requires_grad_(grad)
    c = torch.stack([s["campos"] for s in sts]).requires_grad_(grad)
    st = sts[0]
    settings = BatchRasterizationSettings(
        image_height=st["image_height"], image_width=st["image_width"], tanfovx=tuple(s["tanfovx"] for s in sts),
        tanfovy=tuple(s["tanfovy"] for s in sts), bg=st["bg"], scale_modifier=1.0, viewmatrix=V, projmatrix=Pm,
        sh_degree=st["sh_degree"], sh_degree_t=st["sh_degree_t"], campos=c, timestamp=tuple(s["timestamp"] for s in sts),
        time_duration=st["time_duration"], rot_4d=st["rot_4d"], gaussian_dim=st["gaussian_dim"],
        force_sh_3d=st["force_sh_3d"], prefiltered=False, debug=False)
    g = _inputs(sc, raw, raw)
    means = _leaf(sc.means3D)
    m2 = torch.zeros(n, sc.P, 3, device=DEV, requires_grad=True)
    four = sc.gaussian_dim == 4
    color, radii, depth, alpha, flow = rasterize_gaussians_batch(
        means, m2, g["opacity"], g["sh"], g["scales"], g["rotations"], settings,
        sh_rest=g["sh_rest"] if raw else None, flow_2d=sc.flow_2d, ts=sc.ts if four else None,
        scales_t=g["scales_t"] if four else None, rotations_r=g["rotations_r"] if sc.rot_4d else None, raw=raw)
    _loss(cfg, color, depth, alpha, True).backward()
    d = lambda t: None if t is None else t.detach().double().cpu()
    return cams, sts, dict(means3D=d(means.grad), V=d(V), P=d(Pm), dV=d(V.grad), dP=d(Pm.grad), dc=d(c.grad))


@pytest.mark.parametrize("raw", [False, True])
def test_translation_identity_batched(raw):
    _, _, g = _batch("small", raw=raw)
    gs = [dict(means3D=g["means3D"] if b == 0 else torch.zeros_like(g["means3D"]), dc=g["dc"][b], V=g["V"][b],
               dV=g["dV"][b], P=g["P"][b], dP=g["dP"][b]) for b in range(g["V"].shape[0])]
    _check_identity("batch raw=%d" % raw, gs)


def test_batched_views_match_the_single_view_call():
    from gaussian_renderer import GaussianRasterizer
    cams, sts, gb = _batch("small", n=3)
    cfg, _, sc, _ = helpers.build("small", device=DEV)
    for b, st in enumerate(sts):
        runs = []
        for _ in range(2):    # the blend backward's run-to-run spread (atomic accumulation order)
            V, Pm, c = _leaf(st["viewmatrix"]), _leaf(st["projmatrix"]), _leaf(st["campos"])
            rast = GaussianRasterizer(_rast_settings(st, viewmatrix=V, projmatrix=Pm, campos=c))
            color, radii, depth, alpha = rast(_leaf(sc.means3D), torch.zeros_like(sc.means3D, requires_grad=True),
                                              sc.opacities, shs=sc.shs, flow_2d=sc.flow_2d, ts=sc.ts, scales=sc.scales,
                                              scales_t=sc.scales_t, rotations=sc.rotations, rotations_r=sc.rotations_r)[:4]
            gc, gd, ga, _ = helpers.pixel_grads(cfg, device=DEV)
            ((color * gc).sum() + (depth * gd).sum() + (alpha * ga).sum()).backward()
            runs.append([t.grad.detach().double().cpu() for t in (V, Pm, c)])
        for k, name in enumerate(("dV", "dP", "dc")):
            spread = (runs[0][k] - runs[1][k]).abs().max().item()
            tol = max(4 * spread, 1e-5 * runs[0][k].abs().max().item())
            diff = (gb[name][b] - runs[0][k]).abs().max().item()
            assert diff <= tol, (b, name, diff, spread)


def test_float64_restatement_on_the_3d_twin():
    import fdgs
    import oracle_py
    C = fdgs.ext()
    cfg, cam, sc, st = helpers.build("tiny")
    f = oracle_py.forward(helpers.oracle_inputs(st, sc, cfg))
    _, st3, t = regimes.twin(cfg, sc, st, f)
    V0, P0 = torch.as_tensor(st3["viewmatrix"]).double(), torch.as_tensor(st3["projmatrix"]).double()
    clamp = CF.project(st3, torch.as_tensor(t["means3D"]).double(), torch.as_tensor(t["cov3D"]).double(), V0, P0)[4].numpy()
    t = {k: np.ascontiguousarray(v[~clamp]) for k, v in t.items()}
    fw = C.rasterize_gaussians(*regimes.twin_args(st3, t, DEV))
    pl, ranges, _ = C.debug_export_binning(fw[7], fw[8], fw[0], cfg["W"], cfg["H"])
    lists = dict(ranges=helpers.to_np(ranges), point_list=helpers.to_np(pl))
    grads = [helpers.to_np(g) for g in helpers.pixel_grads(cfg)]
    _, _, amb = CF.loss(st3, lists, t, grads, V0, P0)
    grads = [g * (~amb).astype(np.float32) for g in grads]
    ref = CF.camera_grads(st3, lists, t, grads)
    import blend_f64
    ref2d = blend_f64.forward_backward(st3, lists, t, grads, mask_ambiguous=False)["grads"]["dL_dmeans2D"]
    e = torch.Tensor([]).to(DEV)
    bw = C.rasterize_gaussians_backward_camera(*regimes.twin_bwd_args(st3, t, DEV, fw, [torch.from_numpy(g).to(DEV) for g in grads]),
                                               e, False, e, False, False, e, e)
    got2d = helpers.to_np(bw[0]).astype(np.float64)
    # the call's own fp32 error, normwise, on the per-Gaussian screen-space gradient the camera terms are built from
    eps = max(np.abs(got2d[:, :2] - ref2d[:, :2]).max() / np.abs(ref2d[:, :2]).max(), EPS)
    for key, k in (("view", 15), ("proj", 16)):
        got = helpers.to_np(bw[k]).astype(np.float64).reshape(4, 4)
        rel = np.abs(got - ref[key]).max() / np.abs(ref[key]).max()
        print("dL/d%s: normwise error %.3e, dL_dmeans2D's %.3e" % (key, rel, eps))
        assert rel <= 64 * eps, (key, rel, eps)
    assert helpers.to_np(bw[17]).tolist() == [0.0, 0.0, 0.0]     # colours precomputed: no view direction


def test_off_means_off_and_one_more_launch():
    import fdgs
    counts = []
    for grad in (False, True):
        n0 = fdgs.launch_count()
        _, _, g = _batch("tiny", n=2, grad=grad)
        counts.append(fdgs.launch_count() - n0)
        assert (g["dV"] is None) == (not grad)
    assert counts[1] == counts[0] + 1, counts
    counts = []
    from gaussian_renderer import GaussianRasterizer
    cfg, cam, sc, st = helpers.build("tiny", device=DEV)
    for grad in (False, True):
        V = st["viewmatrix"].clone().requires_grad_(grad)
        rast = GaussianRasterizer(_rast_settings(st, viewmatrix=V))
        n0 = fdgs.launch_count()
        color = rast(_leaf(sc.means3D), torch.zeros_like(sc.means3D, requires_grad=True), sc.opacities, shs=sc.shs,
                     flow_2d=sc.flow_2d, ts=sc.ts, scales=sc.scales, scales_t=sc.scales_t, rotations=sc.rotations,
                     rotations_r=sc.rotations_r)[0]
        color.sum().backward()
        counts.append(fdgs.launch_count() - n0)
        assert (V.grad is None) == (not grad)
    assert counts[1] == counts[0] + 1, counts


def test_refusals():
    g = _single("tiny", colors=True)
    assert g["dc"].tolist() == [0.0, 0.0, 0.0]
    from gaussian_renderer import render, render_batch
    cfg, cam, sc, _ = helpers.build("tiny", device=DEV)
    pc = _Model(sc, env=_env())
    cams = _views(cfg, 2, DEV)
    cams[1].world_view_transform = cams[1].world_view_transform.clone().requires_grad_(True)
    with pytest.raises(ValueError, match="environment-map"):
        render(cams[1], pc, _pipe(pc), torch.zeros(3, device=DEV))
    with pytest.raises(ValueError, match="environment-map"):
        render_batch(cams, pc, _pipe(pc), torch.zeros(3, device=DEV))


# ---- pose recovery ----------------------------------------------------------------------------------------------------
def _twist(xi):
    """4x4 rigid transform exp([omega]x, v) of xi = (omega, v)"""
    A = torch.zeros(4, 4, dtype=xi.dtype, device=xi.device)
    w, v = xi[:3], xi[3:]
    A[0, 1], A[0, 2], A[1, 2] = -w[2], w[1], -w[0]
    A[1, 0], A[2, 0], A[2, 1] = w[2], -w[1], w[0]
    A[:3, 3] = v
    return torch.linalg.matrix_exp(A)


class _PoseCam:
    """a camera whose world_view_transform is the base's composed with a camera-space se(3) delta D: Wt = Wt0 @ D^T,
    full_proj_transform = Wt @ proj, camera_center from the inverse"""

    def __init__(self, base, D):
        for k in ("image_height", "image_width", "FoVx", "FoVy", "timestamp"):
            setattr(self, k, getattr(base, k))
        W0 = base.world_view_transform
        proj = torch.linalg.inv(W0) @ base.full_proj_transform
        self.world_view_transform = W0 @ D.t()
        self.full_proj_transform = self.world_view_transform @ proj
        self.camera_center = torch.linalg.inv(self.world_view_transform)[3, :3]


def _errors(D):
    R = D[:3, :3]
    ang = math.degrees(math.acos(max(-1.0, min(1.0, (torch.trace(R).item() - 1) / 2))))
    return ang, D[:3, 3].norm().item()


def _recover(batch):
    from gaussian_renderer import render, render_batch
    cfg, _, sc, _ = helpers.build(dict(P=10000, W=256, H=256, seed=4242))
    sc = sc.to(DEV)
    pc = _Model(sc)
    pipe = _pipe(pc)
    bg = torch.zeros(3, device=DEV)
    cams = _views(cfg, 4 if batch else 1, DEV)
    for c in cams:
        c.world_view_transform, c.full_proj_transform, c.camera_center = (
            c.world_view_transform.to(DEV), c.full_proj_transform.to(DEV), c.camera_center.to(DEV))
    with torch.no_grad():
        gt = [render(c, pc, pipe, bg)["render"] for c in cams]
    dist = [(c.camera_center - sc.means3D.mean(0)).norm().item() for c in cams]
    gen = torch.Generator().manual_seed(7)
    D0, xis = [], []
    for d in dist:
        axis = torch.randn(3, generator=gen, dtype=torch.float64)
        tdir = torch.randn(3, generator=gen, dtype=torch.float64)
        xi0 = torch.cat([axis / axis.norm() * math.radians(2.0), tdir / tdir.norm() * 0.02 * d])
        D0.append(_twist(xi0).to(DEV).float())
        xis.append(torch.zeros(6, device=DEV, requires_grad=True))
    init = [_errors((D).double().cpu()) for D in D0]
    scale = torch.tensor([1.0, 1.0, 1.0] + [0.0] * 3, device=DEV)
    opt = torch.optim.Adam(xis, lr=2e-3)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, 0.99)
    for it in range(400):
        opt.zero_grad()
        posed = [_PoseCam(c, _twist(xi * scale + xi * (1 - scale) * d) @ D) for c, xi, D, d in zip(cams, xis, D0, dist)]
        if batch:
            img = render_batch(posed, pc, pipe, bg)["render"]
            loss = (img - torch.stack(gt)).abs().mean()
        else:
            loss = (render(posed[0], pc, pipe, bg)["render"] - gt[0]).abs().mean()
        loss.backward()
        opt.step()
        sched.step()
    with torch.no_grad():
        final = [_errors((_twist(xi * scale + xi * (1 - scale) * d) @ D).double().cpu())
                 for xi, D, d in zip(xis, D0, dist)]
    print("pose recovery (batch=%d): initial %s final %s" % (batch, init, final))
    for (a0, t0), (a1, t1) in zip(init, final):
        assert a1 < 0.1 * a0 and t1 < 0.1 * t0, (init, final)


def test_pose_recovery_through_render():
    _recover(False)


def test_pose_recovery_through_render_batch():
    _recover(True)
