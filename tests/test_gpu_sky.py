"""GPU (-m gpu): the environment-map sky (csrc/sky.cu, fdgs/sky.py) against a float64 restatement of the reference's
sky, with the fp32 PyTorch composition's own error as the yardstick; and render() with an environment map -- the sky
composed inside the rasterizer -- against the PyTorch composition it replaces, on the raw, getter and python-covariance
paths."""
import numpy as np
import pytest
import torch

import helpers
import sky_ref
from fdgs import synth
from raw_model import RawModel, Pipe, PipeUnfused

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# camera poses (yaw, pitch, roll, eye): the default camera looks along +z, i.e. straight at a pole of the sphere, where
# acos is ill-conditioned; yaw -90 looks along -x, across the atan2 seam; the last is posed N3V-style off the origin
CAMERAS = {"pole": None, "seam": (-90.0, 7.3, 0.0, 0.0, 0.0, 0.0), "n3v": (-15.0, 8.0, -3.0, -0.5, 0.3, 0.8)}
MAPS = {"500sq": (500, 500), "300x700": (300, 700)}
IMAGES = {"101x67": (101, 67), "1352x1014": (1352, 1014)}


def _camera(pose, W, H):
    R = T = None
    if pose is not None:
        R, T = synth.pose_from_euler(*pose)
    return sky_ref.SkyCamera(W, H, R=R, T=T, device=DEV)


def _env(hw, seed=5):
    return torch.rand(3, *hw, generator=torch.Generator().manual_seed(seed)).to(DEV)


@pytest.mark.parametrize("img", list(IMAGES))
@pytest.mark.parametrize("emap", list(MAPS))
@pytest.mark.parametrize("camname", list(CAMERAS))
def test_sky_sampler_against_float64(camname, emap, img):
    from fdgs.sky import sky_background
    W, H = IMAGES[img]
    cam = _camera(CAMERAS[camname], W, H)
    env = _env(MAPS[emap]).requires_grad_(True)
    env_t = env.detach().clone().requires_grad_(True)
    g = torch.randn(3, H, W, generator=torch.Generator().manual_seed(9)).to(DEV)

    native = sky_background(env, cam)
    (native * g).sum().backward()
    torch_img = sky_ref.torch_sky(env_t, cam)
    (torch_img * g).sum().backward()
    ref = sky_ref.f64_sky(env, cam).numpy()
    ref_g = sky_ref.f64_sky_grad(env, cam, g).numpy()

    nat = native.detach().cpu().double().numpy()
    tor = torch_img.detach().cpu().double().numpy()
    assert np.isfinite(nat).all()
    ok = np.isfinite(tor)   # at a pole the fp32 composition can take acos of a value an ulp past 1
    e_nat, e_tor = np.abs(nat - ref)[ok], np.abs(tor - ref)[ok]
    print("%s %s %s: max |err| native %.3e torch-fp32 %.3e; mean %.3e / %.3e; non-finite torch pixels %d"
          % (camname, emap, img, e_nat.max(), e_tor.max(), e_nat.mean(), e_tor.mean(), int((~ok).sum())))
    assert e_nat.max() <= 2 * e_tor.max() + 1e-6
    assert e_nat.mean() <= 2 * e_tor.mean() + 1e-6

    if ok.all():
        l2n = helpers.l2_rel(helpers.to_np(env.grad), ref_g)
        l2t = helpers.l2_rel(helpers.to_np(env_t.grad), ref_g)
        print("   dL/denv rel-L2 native %.3e torch-fp32 %.3e" % (l2n, l2t))
        assert l2n <= 2 * l2t + 1e-6


# ---- render() with an environment map ---------------------------------------------------------------------------------
class SkyModel(RawModel):
    """RawModel with an environment-map parameter and the python-side covariance helpers of the reference's model."""

    def __init__(self, sc, env, **kw):
        super().__init__(sc, **kw)
        self.env_map = env.detach().clone().requires_grad_(True)

    def get_current_covariance_and_mean_offset(self, mod, timestamp):
        from gaussian_renderer import pyprep
        return pyprep.conditional_covariance_and_offset(torch.cat([self.get_scaling, self.get_scaling_t], 1), mod,
                                                        self.get_rotation, self.get_rotation_r, timestamp - self.get_t)

    def get_marginal_t(self, timestamp):
        from gaussian_renderer import pyprep
        return pyprep.marginal_t(torch.cat([self.get_scaling, self.get_scaling_t], 1), 1.0, self.get_rotation,
                                 self.get_rotation_r, self.get_t, timestamp)


class SkyPipe(Pipe):
    env_map_res = 500


class SkyPipeUnfused(PipeUnfused):
    env_map_res = 500


class SkyPipePyCov(PipeUnfused):
    env_map_res = 500
    compute_cov3D_python = True


def _torch_reference_render(cam, model, pipe):
    """render() with the sky composed the PyTorch way: rasterize without a sky, then rendered + (1 - alpha) * sky."""
    from gaussian_renderer import render

    class NoSky(pipe):
        env_map_res = 0

    pkg = render(cam, model, NoSky(), torch.zeros(3, device=DEV))
    sky = sky_ref.torch_sky(model.env_map, cam)
    pkg["render"] = sky_ref.torch_composition(pkg["render"], pkg["alpha"], sky)
    return pkg


@pytest.mark.parametrize("pipe", [SkyPipe, SkyPipeUnfused, SkyPipePyCov])
@pytest.mark.parametrize("name", ["n3v", "mid"])
def test_render_with_environment_map(name, pipe):
    from gaussian_renderer import render
    cfg, _, sc, st = helpers.build(name, device=DEV)
    pose = cfg.get("pose") or (0.0, 0.0, 0.0, 0.0, 0.0, 0.0)
    R, T = synth.pose_from_euler(*pose)
    cam = sky_ref.SkyCamera(cfg["W"], cfg["H"], R=R, T=T, timestamp=cfg.get("timestamp", 0.5), device=DEV)
    env = _env((500, 500))
    gc = helpers.pixel_grads(cfg, device=DEV)[0]
    A, B = SkyModel(sc, env, seed=1, requires_grad=True), SkyModel(sc, env, seed=1, requires_grad=True)
    pa = render(cam, A, pipe(), torch.zeros(3, device=DEV))
    (pa["render"] * gc).sum().backward()
    pb = _torch_reference_render(cam, B, pipe)
    (pb["render"] * gc).sum().backward()

    # the image: within the sky bar of the sampler (the sky differs by the fp32 rounding of the two samplers)
    ref = sky_ref.f64_sky(env, cam).numpy()
    alpha = pb["alpha"].detach().cpu().double().numpy()
    rendered_no_sky = pb["render"].detach().cpu().double().numpy() - (1 - alpha) * sky_ref.torch_sky(env, cam).cpu().double().numpy()
    want = rendered_no_sky + (1 - alpha) * ref
    e_nat = np.abs(pa["render"].detach().cpu().double().numpy() - want)
    e_tor = np.abs(pb["render"].detach().cpu().double().numpy() - want)
    assert e_nat.max() <= 2 * e_tor.max() + 1e-6 and e_nat.mean() <= 2 * e_tor.mean() + 1e-6
    assert torch.equal(pa["alpha"], pb["alpha"]) and torch.equal(pa["depth"], pb["depth"])

    # env_map.grad: both paths hand the sampler the same dL/dsky = (1 - alpha) g bit for bit, so they differ by their
    # samplers' fp32 rounding, and torch-fp32's own distance from the exact gradient is itself about 1e-4: the bar is
    # the sampler's (native within 2x of torch-fp32's distance from float64), with the distance to torch reported
    dsky = (1 - pb["alpha"].detach()) * gc
    ref_g = sky_ref.f64_sky_grad(env, cam, dsky).numpy()
    e_nat_g = helpers.l2_rel(helpers.to_np(A.env_map.grad), ref_g)
    e_tor_g = helpers.l2_rel(helpers.to_np(B.env_map.grad), ref_g)
    print("%s env_map.grad rel-L2: native vs torch %.2e; vs float64 native %.2e torch %.2e"
          % (name, helpers.l2_rel(helpers.to_np(A.env_map.grad), helpers.to_np(B.env_map.grad)), e_nat_g, e_tor_g))
    assert e_nat_g <= 2 * e_tor_g + 1e-6

    # the Gaussian leaves: the bars of the raw-entry tests, or 4x the distance between the two formulations of a
    # constant background (test_gpu_background.blend_kernel_floor) if larger
    cbg = float(ref.mean())

    def grads(native):
        M = SkyModel(sc, env, seed=1, requires_grad=True)
        nosky = type("NoSky", (pipe,), {"env_map_res": 0})()
        pkg = render(cam, M, nosky, torch.full((3,), cbg if native else 0.0, device=DEV))
        img = pkg["render"] if native else pkg["render"] + (1 - pkg["alpha"]) * cbg
        (img * gc).sum().backward()
        return dict({k: t.grad for k, t in M.leaves().items()}, viewspace_points=pkg["viewspace_points"].grad)
    from test_gpu_background import blend_kernel_floor
    floor = blend_kernel_floor(grads)
    chain = {"scaling", "scaling_t", "rotation", "rotation_r", "t"}
    for k in list(A.leaves()) + ["viewspace_points"]:
        a, b = (pa[k].grad, pb[k].grad) if k == "viewspace_points" else (A.leaves()[k].grad, B.leaves()[k].grad)
        e = helpers.l2_rel(helpers.to_np(a), helpers.to_np(b))
        # the chain leaves' bar at every size: the blend backward accumulates per Gaussian with atomics, and the chain
        # to scales and rotations amplifies that order's rounding -- the same native render run twice differs there by
        # up to 7e-5 (n3v, 3000 Gaussians) and 1.2e-4 (mid) rel-L2 on an H100, so a 1e-4 bar on the distance of two
        # such runs fails about half the time
        bar = max(2e-3 if k in chain else 1e-4, 4 * floor[k])
        print("%s %-17s rel-L2 %.2e (constant-background formulations %.2e, bar %.2e)" % (name, k, e, floor[k], bar))
        assert e <= bar, (k, e, floor[k])


def test_camera_outside_the_sky_sphere_raises():
    from gaussian_renderer import render
    cfg, _, sc, st = helpers.build("small", device=DEV)
    # eye 100 units out along -z, looking along +x: every ray's line passes at least 73 units from the origin
    R, T = synth.pose_from_euler(90.0, 0.0, 0.0, 0.0, 0.0, -100.0)
    cam = sky_ref.SkyCamera(cfg["W"], cfg["H"], R=R, T=T, device=DEV)
    model = SkyModel(sc, _env((500, 500)), seed=1)
    with pytest.raises(AssertionError):
        render(cam, model, SkyPipe(), torch.zeros(3, device=DEV))
