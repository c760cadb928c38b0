"""GPU (-m gpu): the raw-parameter entry (SURVEY.md section 8(f) row 1) -- render() over a GaussianModel stand-in
with the activations and the SH concatenation fused into the kernels -- against the getter path (torch exp / sigmoid /
F.normalize / cat + autograd through them) and against the compiled reference rasterizer under the same torch prologue."""
import pytest
import torch

import helpers
from raw_model import RawModel, Pipe, PipeUnfused

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CHAIN = {"scaling", "scaling_t", "rotation", "rotation_r", "t"}


def _render_and_backward(model, cam, pipe, G, aux=None):
    from gaussian_renderer import render
    pkg = render(cam, model, pipe, torch.zeros(3, device=DEV))
    loss = (pkg["render"] * G).sum()
    if aux is not None:
        loss = loss + (pkg["depth"] * aux[0]).sum() + (pkg["alpha"] * aux[1]).sum()
    loss.backward()
    return pkg



def test_activations_bit_identical_to_torch():
    """The kernels' exp / sigmoid / quaternion normalisation (fdgs_common.cuh: act_exp, act_sigmoid, act_normalize) give
    torch.exp / torch.sigmoid / F.normalize word for word, so the raw entry activates exactly what the getters would."""
    import fdgs
    g = torch.Generator().manual_seed(1)
    n = 1 << 20
    log_s = (torch.randn(n, generator=g) * 1.5 - 4.0).to(DEV)
    logit = (torch.randn(n, generator=g) * 3.0).to(DEV)
    quat = torch.randn(n, 4, generator=g) * (0.2 + 2 * torch.rand(n, 1, generator=g))
    quat[0] = 0.0   # a zero quaternion: F.normalize divides by the 1e-12 floor
    quat = quat.to(DEV)
    s, o, q = fdgs.ext().debug_activate(log_s, logit, quat, 0)
    for name, got, want in (("exp", s, torch.exp(log_s)), ("sigmoid", o, torch.sigmoid(logit)),
                            ("normalize", q, torch.nn.functional.normalize(quat))):
        differing = int((got.view(torch.int32) != want.view(torch.int32)).sum())
        assert differing == 0, (name, differing)

@pytest.mark.parametrize("name,aux", [("small", False), ("rotcam", True), ("dur10", False), ("smod2", False), ("dim3", False),
                                      ("norot4d", False), ("deg1m4", False), ("mid", False)])
def test_fused_prologue_matches_getter_path(name, aux):
    cfg, cam, sc, st = helpers.build(name, device=DEV)
    cam = cam.to(DEV)
    gc, gd, ga, gf = helpers.pixel_grads(cfg, device=DEV)
    A = RawModel(sc, seed=1, requires_grad=True)
    B = RawModel(sc, seed=1, requires_grad=True)
    # scale_modifier / prefilter are per-call settings of render(); the configuration's modifier is applied to both
    pa = _render_and_backward(A, cam, PipeUnfused(), gc, (gd, ga) if aux else None)
    pb = _render_and_backward(B, cam, Pipe(), gc, (gd, ga) if aux else None)
    same_radii = (pa["radii"] == pb["radii"]).float().mean().item()
    assert same_radii > 0.9995, same_radii
    assert helpers.psnr(helpers.to_np(pb["render"]), helpers.to_np(pa["render"])) > 90.0
    assert helpers.max_rel(helpers.to_np(pb["depth"]), helpers.to_np(pa["depth"])) < 1e-4
    print("%s: image bit-identical: %s, radii identical: %.6f" % (name, torch.equal(pa["render"], pb["render"]), same_radii))
    for k, a in A.leaves().items():
        b = B.leaves()[k]
        if a.grad is None:
            assert b.grad is None or float(b.grad.abs().max()) == 0.0, k
            continue
        assert b.grad is not None and b.grad.shape == a.grad.shape, k
        err = helpers.l2_rel(helpers.to_np(b.grad), helpers.to_np(a.grad))
        # both sides run the same (non-deterministic) blend backward: blend-level tensors agree to its noise; the
        # covariance chain amplifies that noise (see test_gpu_parity.py) -- at 100k Gaussians up to a few 1e-4
        assert err < (2e-3 if (k in CHAIN and cfg["P"] >= 50000) else 1e-4), (k, err)
    assert helpers.l2_rel(helpers.to_np(pb["viewspace_points"].grad), helpers.to_np(pa["viewspace_points"].grad)) < 1e-4


def test_raw_entry_vs_reference_render_at_cfg3():
    """Gradients w.r.t. the RAW parameters against the reference rasterizer under the reference's own torch prologue
    (getters + autograd), at cfg3: the record of 3 reference runs and of its -fmad=false build on a fixed sample of rows
    (tests/golden/ref_raw_cfg3.npz).  Bar: 1e-4, or 4 x the reference's run-to-run spread or the distance of its other
    build, whichever is largest."""
    R = helpers.ref_record("raw_cfg3")
    cfg, cam, sc, st = helpers.build("cfg3", device=DEV)
    cam = cam.to(DEV)
    g = torch.Generator().manual_seed(77)
    G = torch.randn(3, cfg["H"], cfg["W"], generator=g).to(DEV)
    B = RawModel(sc, seed=2, requires_grad=True)
    pb = _render_and_backward(B, cam, Pipe(), G)
    img = helpers.get_summary(R, "image")
    ours_px = pb["render"].detach().reshape(3, -1).t()[torch.from_numpy(img["rows"]).to(DEV)]
    assert helpers.psnr(helpers.to_np(ours_px), img["mean"]) > 90.0
    for k, b in B.leaves().items():
        s = helpers.get_summary(R, k)
        rows, m = torch.from_numpy(s["rows"]).to(DEV), torch.from_numpy(s["mean"]).double()
        spread, l2b = float(s["stats"][3]), float(s["stats"][4])
        l2 = ((b.grad[rows].cpu().double() - m).norm() / m.norm()).item()
        assert l2 < max(1e-4, 4 * max(spread, l2b)), (k, l2, spread, l2b)
        print("raw grad %-13s vs reference render(): l2 %.2e (reference spread %.2e, other build %.2e)" % (k, l2, spread, l2b))


def test_view_parallel_step_with_raw_entry():
    """factor mode + raw entry on one GPU: 3 views, gradients at the raw leaves == sequential autograd accumulation,
    without and with an environment-map sky behind the Gaussians"""
    from fdgs.dist import ViewParallelStep
    from gaussian_renderer import render
    import test_gpu_view_parallel as vp
    from test_gpu_sky import SkyModel, SkyPipe
    cfg, cam, sc, st = helpers.build("n3v", device=DEV)
    bg = torch.zeros(3, device=DEV)
    Gs = [torch.randn(3, cfg["H"], cfg["W"], generator=torch.Generator().manual_seed(50 + k)).to(DEV) for k in range(3)]
    for sky in (False, True):
        cams = vp._views(cfg, 3, DEV, sky)
        if sky:
            A, B, pipe = SkyModel(sc, vp._env(), seed=4, requires_grad=True), SkyModel(sc, vp._env(), seed=4, requires_grad=True), SkyPipe()
        else:
            A, B, pipe = RawModel(sc, seed=4, requires_grad=True), RawModel(sc, seed=4, requires_grad=True), Pipe()
        for k, c in enumerate(cams):
            ((render(c, A, pipe, bg)["render"] * Gs[k]).sum() / 3).backward()
        step = ViewParallelStep(sc.P, DEV)
        with step:
            for k, c in enumerate(cams):
                pkg = render(c, B, pipe, bg)
                ((pkg["render"] * Gs[k]).sum() / 3).backward()
                step.add_view_stats(pkg["viewspace_points"].grad, pkg["radii"])
        lv = B.leaves()
        step.finish([lv[k] for k in ("xyz", "t", "scaling", "scaling_t", "rotation", "rotation_r", "opacity")],
                    [lv["features_dc"], lv["features_rest"]])
        for k, a in A.leaves().items():
            assert helpers.l2_rel(helpers.to_np(lv[k].grad), helpers.to_np(a.grad)) < (2e-6 if k.startswith("features") else 1e-4), (sky, k)
        if sky:
            assert helpers.l2_rel(helpers.to_np(B.env_map.grad), helpers.to_np(A.env_map.grad)) < 1e-4
