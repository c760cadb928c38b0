"""GPU (-m gpu): batched views -- B cameras of the same Gaussians through one forward and one backward call
(rasterize_gaussians_batch, render_batch).

  1. forward, bit for bit per view: every output of the batched call equals the single-view call on that camera,
     including the private tile lists (view b's lists are one contiguous stretch of the batched point_list);
  2. backward against the sequential loop (render + backward per view, autograd accumulating), with the bars of
     test_gpu_view_parallel.py::_cmp;
  3. launches: a batch of 8 launches no more kernels than a batch of 1 plus the sort's second size class, and no
     host synchronisation happens on the PyTorch side;
  4. training: a lego-shaped loop whose steps are taken on the batched gradients tracks the sequential loop (the
     covariance-chain leaves within max(1e-3, 4 x the loop's own run-to-run distance at that iteration)).
"""
import copy
import ctypes

import pytest
import torch

import helpers
import regimes
from test_gpu_view_parallel import DEV, _Model, _cmp, _env, _pipe, _views

pytestmark = pytest.mark.gpu


def _C():
    import fdgs
    return fdgs.ext()


def _settings(cams, sc, cfg):
    from fdgs import synth
    bg = torch.tensor(cfg.get("bg", (0.0, 0.0, 0.0)), dtype=torch.float32)
    return [synth.raster_settings(c, sc, bg=bg, scale_modifier=cfg.get("scale_modifier", 1.0), device=DEV) for c in cams]


def _inputs(sc, raw, split):
    """Gaussian inputs of either entry: activated parameters, or the raw ones (log-scales, logits, un-normalised
    quaternions) that activate to the same values; SH as one tensor or split like features_dc / features_rest."""
    e = torch.Tensor([])
    four_d = sc.gaussian_dim == 4
    scales, scales_t, op, rot, rot_r = sc.scales, sc.scales_t, sc.opacities, sc.rotations, sc.rotations_r
    if raw:
        scales, scales_t, op = scales.log(), scales_t.log(), torch.logit(op)
        rot, rot_r = 2.0 * rot, 3.0 * rot_r
    sh, sh_rest = (sc.shs[:, :1].contiguous(), sc.shs[:, 1:].contiguous()) if split else (sc.shs, e)
    return dict(opacity=op, ts=sc.ts if four_d else e, scales=scales, scales_t=scales_t if four_d else e, rotations=rot,
                rotations_r=rot_r if sc.rot_4d else e, sh=sh, sh_rest=sh_rest)


def _single(st, sc, cfg, g, raw, bg_image):
    e = torch.Tensor([])
    return _C().rasterize_gaussians_ext(
        st["bg"], sc.means3D, e, sc.flow_2d, g["opacity"], g["ts"], g["scales"], g["scales_t"], g["rotations"],
        g["rotations_r"], st["scale_modifier"], e, cfg.get("prefilter_var", -1.0), st["viewmatrix"], st["projmatrix"],
        st["tanfovx"], st["tanfovy"], st["image_height"], st["image_width"], g["sh"], st["sh_degree"], st["sh_degree_t"],
        st["campos"], st["timestamp"], st["time_duration"], st["rot_4d"], st["gaussian_dim"], st["force_sh_3d"],
        st["prefiltered"], False, g["sh_rest"], raw, e if bg_image is None else bg_image)


def _batch(sts, sc, cfg, g, raw, bg_image):
    e = torch.Tensor([])
    st = sts[0]
    f32 = lambda k: torch.tensor([s[k] for s in sts], dtype=torch.float32)
    return _C().rasterize_gaussians_batch(
        st["bg"], sc.means3D, sc.flow_2d, g["opacity"], g["ts"], g["scales"], g["scales_t"], g["rotations"],
        g["rotations_r"], st["scale_modifier"], cfg.get("prefilter_var", -1.0),
        torch.stack([s["viewmatrix"] for s in sts]), torch.stack([s["projmatrix"] for s in sts]),
        torch.stack([s["campos"] for s in sts]), f32("timestamp"), f32("tanfovx"), f32("tanfovy"), st["image_height"],
        st["image_width"], g["sh"], g["sh_rest"], st["sh_degree"], st["sh_degree_t"], st["time_duration"], st["rot_4d"],
        st["gaussian_dim"], st["force_sh_3d"], st["prefiltered"], False, raw, e if bg_image is None else bg_image)


def _check_forward(cfg, sc, cams, raw=False, split=False, sky=False):
    sts = _settings(cams, sc, cfg)
    B, H, W = len(cams), cfg["H"], cfg["W"]
    g = _inputs(sc, raw, split)
    bgs = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(3)).to(DEV) if sky else None
    R_b, color, flow, depth, T, radii, geom_b, bin_b, img_b, means_b = _batch(sts, sc, cfg, g, raw, bgs)
    pl_all = _C().debug_export_binning(bin_b, img_b, R_b, W, H)[0]
    total = 0
    for v in range(B):
        one = _single(sts[v], sc, cfg, g, raw, None if bgs is None else bgs[v])
        R, c1, f1, d1, T1, r1, _, bin1, img1, _, m1 = one
        for a, b in ((color[v], c1), (flow[v], f1), (depth[v], d1), (T[v], T1), (radii[v], r1), (means_b[v], m1)):
            assert torch.equal(a, b), v
        pl, rg, nc = _C().debug_export_binning(bin1, img1, R, W, H)
        rg_v, nc_v = _C().debug_export_binning_view(img_b, W, H, B, v)
        assert torch.equal(nc_v, nc), v
        full = rg[:, 1] > rg[:, 0]
        assert torch.equal(rg_v[:, 1] > rg_v[:, 0], full), v
        start = int(rg_v[full, 0].min()) if R > 0 else 0
        assert torch.equal(rg_v[full] - start, rg[full]) and int(rg_v[~full].abs().sum()) == 0, v
        assert torch.equal(pl_all[start:start + R], pl), v
        total += R
    assert total == R_b
    return radii


GOLDEN = ["small", "dur10", "n3v", "rotcam", "sh3d", "deg1", "norot4d", "dim3", "flowbg", "ragged", "smod2", "prefilter"]


@pytest.mark.parametrize("B", [1, 2, 5])
@pytest.mark.parametrize("name", GOLDEN)
def test_forward_is_the_single_view_call_bit_for_bit(name, B):
    cfg, _, sc, _ = helpers.build(name, device=DEV)
    _check_forward(cfg, sc, _views(cfg, B, DEV))


@pytest.mark.parametrize("tile_cull", [0, 1])
@pytest.mark.parametrize("raw,split,sky", [(False, False, False), (True, True, False), (False, True, True),
                                           (True, False, True)])
def test_forward_entries_and_tile_modes(tile_cull, raw, split, sky):
    import fdgs
    old = fdgs.lib().fdgs_set_tile_cull(tile_cull)
    try:
        cfg, _, sc, _ = helpers.build("n3v", device=DEV)
        _check_forward(cfg, sc, _views(cfg, 3, DEV), raw=raw, split=split, sky=sky)
    finally:
        fdgs.lib().fdgs_set_tile_cull(old)


@pytest.mark.parametrize("regime", ["opaque", "huge", "deep"])
def test_forward_regimes(regime):
    cfg, cam, sc, _ = getattr(regimes, regime)()
    sc = sc.to(DEV)
    _check_forward(cfg, sc, [cam.to(DEV)] + _views(cfg, 2, DEV))


def test_forward_with_an_empty_view_and_no_gaussians():
    from fdgs import synth
    cfg, _, sc, _ = helpers.build("small", device=DEV)
    cams = _views(cfg, 2, DEV)
    R, T = synth.pose_from_euler(0.0, 180.0, 0.0, 0.0, 0.0, 0.0)    # looking away from every Gaussian
    cams.insert(1, synth.make_camera(cfg["W"], cfg["H"], timestamp=0.5, R=R, T=T).to(DEV))
    radii = _check_forward(cfg, sc, cams, sky=True)
    assert int(radii[1].abs().sum()) == 0 and int(radii[0].abs().sum()) > 0
    empty = copy.copy(sc)
    for k, v in sc.tensors().items():
        setattr(empty, k, v[:0].contiguous())
    assert empty.P == 0
    _check_forward(cfg, empty, cams, sky=True)


@pytest.mark.parametrize("cfg,B", [(dict(P=100000, W=800, H=800, seed=7), 8), (helpers.CONFIGS["cfg5"], 4)],
                         ids=["lego-800-B8", "cfg5-B4"])
def test_forward_at_training_shapes(cfg, B):
    cfg, _, sc, _ = helpers.build(cfg, device=DEV)
    _check_forward(cfg, sc, _views(cfg, B, DEV))


# ---- 2. backward against the sequential loop --------------------------------------------------------------------
def _loss(pkg_img, cfg, k, n, aux, depth=None, alpha=None):
    g = torch.Generator(device="cpu").manual_seed(1000 + k)
    G = torch.randn(3, cfg["H"], cfg["W"], generator=g).to(DEV)
    loss = (pkg_img * G).sum()
    if aux:
        Gd = torch.randn(1, cfg["H"], cfg["W"], generator=g).to(DEV)
        loss = loss + 0.1 * (depth * Gd).sum() + 0.3 * (alpha * Gd).sum()
    return loss / n


def _sequential(cfg, sc, cams, split, env, aux):
    from gaussian_renderer import render
    from fdgs.dist import ViewBatchStats
    pc = _Model(sc, split, env)
    stats = ViewBatchStats(sc.P, DEV)
    bg = torch.zeros(3, device=DEV)
    for k, cam in enumerate(cams):
        pkg = render(cam, pc, _pipe(pc), bg)
        _loss(pkg["render"], cfg, k, len(cams), aux, pkg["depth"], pkg["alpha"]).backward()
        stats.add_view(pkg["viewspace_points"].grad, pkg["radii"])
    return pc, stats


def _batched(cfg, sc, cams, split, env, aux):
    from gaussian_renderer import render_batch
    from fdgs.dist import ViewBatchStats
    pc = _Model(sc, split, env)
    stats = ViewBatchStats(sc.P, DEV)
    pkg = render_batch(cams, pc, _pipe(pc), torch.zeros(3, device=DEV))
    sum(_loss(pkg["render"][k], cfg, k, len(cams), aux, pkg["depth"][k], pkg["alpha"][k]) for k in range(len(cams))).backward()
    for k in range(len(cams)):
        stats.add_view(pkg["viewspace_points"].grad[k], pkg["radii"][k])
    return pc, stats


BWD = [("small", 3, False, False, False), ("n3v", 4, True, False, False), ("dur10", 3, False, False, True),
       ("rotcam", 2, True, False, True), ("sh3d", 2, False, False, False), ("mid", 3, True, False, False),
       ("small", 2, False, True, False), ("mid", 3, True, True, True)]


@pytest.mark.parametrize("name,nviews,split,sky,aux", BWD,
                         ids=["%s-%d%s%s%s" % (n, v, "-split" if s else "", "-sky" if k else "", "-aux" if a else "")
                              for n, v, s, k, a in BWD])
def test_backward_matches_the_sequential_loop(name, nviews, split, sky, aux):
    cfg, _, sc, _ = helpers.build(name, device=DEV)
    cams = _views(cfg, nviews, DEV, sky)
    env = _env() if sky else None
    ref, rs = _sequential(cfg, sc, cams, split, env, aux)
    got, gs = _batched(cfg, sc, cams, split, env, aux)
    _cmp(got, ref, gs, rs, tol_sh=2e-6, tol_geo=1e-4, tol_chain=1e-3 if cfg["P"] < 50000 else 5e-3)
    sh_got = torch.cat([p.grad for p in got.sh_leaves], 1)
    assert float(sh_got[rs.max_radii <= 0].abs().sum()) == 0.0
    assert float(sh_got.abs().max()) > 0


# ---- 3. launches and host synchronisation -----------------------------------------------------------------------
def test_one_launch_per_stage_and_no_torch_side_sync():
    import fdgs
    from gaussian_renderer import render, render_batch
    lib = fdgs.lib()
    lib.fdgs_launch_count.restype = ctypes.c_longlong
    cfg, _, sc, _ = helpers.build("mid", device=DEV)
    cams = _views(cfg, 8, DEV)
    pc = _Model(sc)
    bg = torch.zeros(3, device=DEV)

    def launches(fn):
        torch.cuda.synchronize()
        n0 = lib.fdgs_launch_count()
        fn()
        torch.cuda.synchronize()
        return lib.fdgs_launch_count() - n0

    def batch(cs):
        return lambda: render_batch(cs, pc, _Pipe(), bg)["render"].sum().backward()

    def loop():
        for c in cams:
            render(c, pc, _Pipe(), bg)["render"].sum().backward()

    one, eight, seq = launches(batch(cams[:1])), launches(batch(cams)), launches(loop)
    assert eight <= one + 1, (one, eight)     # + the large-tile sort instantiation
    assert eight < seq, (eight, seq)
    torch.cuda.set_sync_debug_mode("error")
    try:
        batch(cams)()
    finally:
        torch.cuda.set_sync_debug_mode(0)


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False
    env_map_res = 0


# ---- 4. training ----------------------------------------------------------------------------------------------------
def test_training_loop_on_batched_gradients():
    from test_gpu_densify_train import _lego_model, _Pipe as TrainPipe
    from gaussian_renderer import render, render_batch
    from fdgs.dist import ViewBatchStats
    m, cams, gts = _lego_model(20000, 400, 400, DEV)
    params = [p for g in m.optimizer.param_groups for p in g["params"]]
    bg = torch.zeros(3, device=DEV)
    P = params[0].shape[0]
    batch = 8
    chain = ("xyz", "t", "scaling", "scaling_t", "rotation", "rotation_r")

    def sequential(views):
        for p in params:
            p.grad = None
        stats = ViewBatchStats(P, DEV)
        total = 0.0
        for k in views:
            pkg = render(cams[k], m, TrainPipe(), bg)
            loss = (pkg["render"] - gts[k]).abs().mean()
            loss.backward()
            total += float(loss.detach())
            stats.add_view(pkg["viewspace_points"].grad, pkg["radii"])
        return [p.grad.clone() for p in params], stats, total

    for it in range(30):
        views = [(it * batch + k) % len(cams) for k in range(batch)]
        ref, rs, loss_seq = sequential(views)
        # the loop's own run-to-run distance: the blend backward's atomics add in a different order every run, and the
        # normalisation chain of the raw quaternions magnifies that rounding in the rotation gradients
        again = sequential(views)[0]
        # batched arm, from the same state
        for p in params:
            p.grad = None
        gs = ViewBatchStats(P, DEV)
        pkg = render_batch([cams[k] for k in views], m, TrainPipe(), bg)
        losses = [(pkg["render"][j] - gts[k]).abs().mean() for j, k in enumerate(views)]
        sum(losses).backward()
        for j in range(batch):
            gs.add_view(pkg["viewspace_points"].grad[j], pkg["radii"][j])
        loss_b = float(sum(losses).detach())
        assert abs(loss_b - loss_seq) <= 1e-5 * abs(loss_seq), (it, loss_b, loss_seq)
        for g, p, r, r2 in zip(m.optimizer.param_groups, params, ref, again):
            err = helpers.l2_rel(helpers.to_np(p.grad), helpers.to_np(r))
            if g["name"] in chain:
                tol = max(1e-3, 4 * helpers.l2_rel(helpers.to_np(r2), helpers.to_np(r)))
            else:
                tol = 2e-6 if g["name"] in ("f_dc", "f_rest") else 1e-4
            assert err <= tol, (it, g["name"], err, tol)
        assert helpers.l2_rel(helpers.to_np(gs.grad_norm_sum), helpers.to_np(rs.grad_norm_sum)) <= 1e-4
        assert torch.equal(gs.visibility_count, rs.visibility_count) and torch.equal(gs.max_radii, rs.max_radii)
        m.optimizer.step()
