"""GPU (-m gpu): environment-map scenes in the captured training iteration -- the batched sky sampler on device cameras
(fdgs.sky.sample_sky_batch over StaticViews(..., sky=True)), the map's Adam step as the optimiser's "env_map" group and
the miss check that travels with the rasterizer's status.

  1. sky against float64: the batched dL/d env_map of pole, seam and N3V-posed cameras in one batch is within 2x the
     per-view sampler's distance from float64 (plus 1e-6), for 500^2 and 300x700 maps at 101x67 and 1352x1014;
  2. forward bit for bit: each view's sky equals sample_sky(env_map, camera) and the miss flags agree;
  3. render: render_batch(StaticViews(sky=True)) images and radii equal the eager render_batch(cameras) bit for bit;
     the gradients agree to the batch tests' bars;
  4. Adam: with the exact-loss trick (test_gpu_graph_iteration.py) and a deterministic term on env_map, the graphed
     iteration equals eager FusedAdam.step() bit for bit, env_map included, on plain iterations, with every Gaussian
     group held (the map steps), with the map held, and across an overflow and re-capture;
  5. miss: a camera outside the radius-60 sphere raises AssertionError with the eager message, in the warm-up and in a
     replay, and nothing has moved; the next call with valid cameras replays without a re-capture;
  6. synchronisation: with the map the status read is still the call's only host synchronisation;
  7. training: a coffee_martini-shaped loop (B = 4, a map optimised until mid-run, one densification, one opacity
     reset) tracks the eager loop run in the reference's order (statistics -> densify / reset -> Gaussian Adam -> env
     Adam).
"""
import copy
import math
import warnings

import pytest
import torch
from torch import nn

import helpers
import sky_ref
from test_gpu_graph_iteration import _assert_equal, _exact_loss, _gt, _rel, _state
from test_gpu_sky import CAMERAS, IMAGES, MAPS, _camera, _env

pytestmark = pytest.mark.gpu
DEV = "cuda"
MISS = "does not intersect the sky sphere"


def _static(cams, capacity=0):
    from fdgs.graph import StaticViews
    v = StaticViews(len(cams), int(cams[0].image_height), int(cams[0].image_width), DEV, sky=True)
    v.load(cams)
    v.capacity = capacity
    return v


def _outside(W, H):
    """eye 100 units out along -z, looking along +x: no ray meets the radius-60 sphere (test_gpu_sky.py)"""
    from fdgs import synth
    R, T = synth.pose_from_euler(90.0, 0.0, 0.0, 0.0, 0.0, -100.0)
    return sky_ref.SkyCamera(W, H, R=R, T=T, device=DEV)


# ---- 1. sky against float64 / 2. forward bit for bit ----------------------------------------------------------------
@pytest.mark.parametrize("img", list(IMAGES))
@pytest.mark.parametrize("emap", list(MAPS))
def test_batched_sky_against_float64_and_the_single_view_sampler(emap, img):
    from fdgs.sky import sample_sky, sample_sky_batch
    W, H = IMAGES[img]
    cams = [_camera(CAMERAS[n], W, H) for n in CAMERAS]
    env = _env(MAPS[emap]).requires_grad_(True)
    env_e = env.detach().clone().requires_grad_(True)
    g = torch.randn(len(cams), 3, H, W, generator=torch.Generator().manual_seed(9)).to(DEV)

    sky, miss = sample_sky_batch(env, _static(cams))
    (sky * g).sum().backward()
    for b, cam in enumerate(cams):
        s, flag = sample_sky(env_e, cam)
        assert torch.equal(sky[b], s), b                        # 2. the single view's sky, bit for bit
        (s * g[b]).sum().backward()
        flag.check()
    assert int(miss[0]) == 0

    ref = sum(sky_ref.f64_sky_grad(env, cam, g[b]).numpy() for b, cam in enumerate(cams))
    e_batch = helpers.l2_rel(helpers.to_np(env.grad), ref)
    e_eager = helpers.l2_rel(helpers.to_np(env_e.grad), ref)
    print("%s %s: dL/denv rel-L2 to float64, batched %.3e per-view %.3e" % (emap, img, e_batch, e_eager))
    assert e_batch <= 2 * e_eager + 1e-6


def test_batched_miss_flag_agrees_with_the_single_view_sampler():
    from fdgs.sky import MISS_MESSAGE, sample_sky, sample_sky_batch
    W, H = IMAGES["101x67"]
    env = _env(MAPS["500sq"])
    inside, outside = _camera(CAMERAS["n3v"], W, H), _outside(W, H)
    for cams in ([inside, inside], [inside, outside], [outside]):
        sky, miss = sample_sky_batch(env, _static(cams))
        flags = []
        for b, cam in enumerate(cams):
            s, flag = sample_sky(env, cam)
            assert torch.equal(sky[b], s), b
            flag.ready.synchronize()
            flags.append(int(flag.host[0]))
        assert int(miss[0]) == int(any(flags)), flags
    with pytest.raises(AssertionError, match=MISS):
        sample_sky(env, outside)[1].check()
    assert MISS in MISS_MESSAGE


# ---- 3. render ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,nviews,split", [("n3v", 4, True), ("mid", 3, False)])
def test_render_batch_with_sky_views_equals_the_eager_batch(name, nviews, split):
    from gaussian_renderer import render_batch
    from fdgs.dist import ViewBatchStats
    from test_gpu_batch import _loss
    from test_gpu_view_parallel import _Model, _cmp, _pipe, _views
    cfg, _, sc, _ = helpers.build(name, device=DEV)
    cams = _views(cfg, nviews, DEV, True)
    env = _env((500, 500))
    views = _static(cams)

    def run(cameras):
        pc = _Model(sc, split, env)
        pkg = render_batch(cameras, pc, _pipe(pc), torch.zeros(3, device=DEV))
        if "status" in pkg:
            assert int(pkg["status"][2]) == 0 and int(pkg["sky_miss"][0]) == 0
        sum(_loss(pkg["render"][k], cfg, k, nviews, False) for k in range(nviews)).backward()
        stats = ViewBatchStats(sc.P, DEV)
        for k in range(nviews):
            stats.add_view(pkg["viewspace_points"].grad[k], pkg["radii"][k])
        return pc, stats, pkg

    ref, rs, pr = run(cams)
    views.capacity = int(ref.get_xyz.shape[0]) * nviews * 64         # no overflow: far above the scene's instances
    got, gs, pg = run(views)
    for k in ("render", "radii", "depth", "alpha", "flow"):
        assert torch.equal(pg[k], pr[k]), k
    _cmp(got, ref, gs, rs, tol_sh=2e-6, tol_geo=1e-4, tol_chain=1e-3)


# ---- the lego scene with an environment map -----------------------------------------------------------------------
def _with_intrinsics(cam):
    """The camera with the reference Camera's pinhole intrinsics, which the sky sampler reads."""
    c = copy.copy(cam)
    W, H = int(cam.image_width), int(cam.image_height)
    c.fl_x, c.fl_y = W / (2 * math.tan(cam.FoVx * 0.5)), H / (2 * math.tan(cam.FoVy * 0.5))
    c.cx, c.cy = W / 2.0, H / 2.0
    return c


def _sky_lego(P=8000, W=128, H=128, env_hw=(64, 128)):
    """The lego model of test_gpu_densify_train.py with a learned map stepped as FusedAdam group "env_map" at the
    features' learning rate, as the reference's separate Adam([env_map], lr=feature_lr, eps=1e-15)."""
    from test_gpu_densify_train import _lego_model
    m, cams, gts = _lego_model(P, W, H, DEV)
    m.env_map = nn.Parameter(torch.rand(3, *env_hw, generator=torch.Generator().manual_seed(6)).to(DEV))
    m.optimizer.add_param_group({"params": [m.env_map], "lr": 2.5e-3, "name": "env_map"})
    return m, [_with_intrinsics(c) for c in cams], gts


def _leaves(m):
    return [p for g in m.optimizer.param_groups for p in g["params"]]


def _gaussian_groups(m):
    return {g["name"] for g in m.optimizer.param_groups if g["name"] != "env_map"}


def _clone(m):
    """An independent copy of the model: parameters (env_map included), FusedAdam state and statistics."""
    import densify_ref as R
    from fdgs.optim import FusedAdam
    c = copy.copy(m)
    groups, state = [], {}
    for g in m.optimizer.param_groups:
        p = g["params"][0]
        q = nn.Parameter(p.detach().clone().requires_grad_(True))
        setattr(c, "env_map" if g["name"] == "env_map" else R.ATTR[g["name"]], q)
        groups.append({"params": [q], "lr": g["lr"], "name": g["name"]})
        st = m.optimizer.state.get(p)
        if st is not None:
            state[q] = {k: v.clone() for k, v in st.items()}
    c.optimizer = FusedAdam(groups, lr=0.0, betas=m.optimizer.betas, eps=m.optimizer.eps)
    c.optimizer.state = state
    for n in ("xyz_gradient_accum", "t_gradient_accum", "denom", "max_radii2D"):
        setattr(c, n, getattr(m, n).clone())
    return c


class _SkyPipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False
    env_map_res = 500
    fused_prologue = True


def _fn(m, loss_fn, bg):
    from gaussian_renderer import render_batch

    def fn(views, gt):
        pkg = render_batch(views, m, _SkyPipe(), bg)
        loss = loss_fn(m, pkg, gt)
        loss.backward()
        return loss, pkg
    return fn


def _l1(m, pkg, gt):
    return sum((pkg["render"][k] - gt[k]).abs().mean() for k in range(gt.shape[0]))


def _eager_grads(m, cams, gt, loss_fn, bg):
    from gaussian_renderer import render_batch
    for p in _leaves(m):
        p.grad = None
    pkg = render_batch(cams, m, _SkyPipe(), bg)
    loss = loss_fn(m, pkg, gt)
    loss.backward()
    return loss, pkg


def _eager_step(m, hold):
    """FusedAdam.step() as the reference's loop sees it: a held leaf has no gradient."""
    held = m.optimizer.held(hold)
    for p in _leaves(m):
        if id(p) in held:
            p.grad = None
    m.optimizer.step()


# ---- 4. Adam bit for bit --------------------------------------------------------------------------------------------
def test_graphed_iteration_with_a_map_equals_eager_fused_adam_bit_for_bit():
    from fdgs.graph import GraphedStep
    m, cams, _ = _sky_lego()
    bg = torch.zeros(3, device=DEV)
    e = _clone(m)
    step = GraphedStep(_fn(m, _exact_loss, bg), m, optimizer=m.optimizer)
    env0 = m.env_map.detach().clone()
    gauss = _gaussian_groups(m)
    holds = [(), (), gauss, (), {"env_map"}, (), gauss, {"env_map"}, (), ()]
    for it, hold in enumerate(holds):
        views = [cams[(it + k) % len(cams)] for k in range(2)]
        gt = _gt(views, it)
        if it == 7:                                 # the next call captures at capacity 1 and overflows
            step.views.capacity, step._key = 1, None
        step(views, gt, hold=hold)
        _eager_grads(e, views, gt, _exact_loss, bg)
        _eager_step(e, hold)
        _assert_equal(m, e, it)
    assert step.info["overflows"] >= 1 and step.info["captures"] == 2 + step.info["overflows"], step.info
    counts = {g["name"]: float(m.optimizer.state[g["params"][0]]["step"]) for g in m.optimizer.param_groups}
    assert counts["env_map"] == len(holds) - 2 and counts["xyz"] == len(holds) - 2, counts
    assert not torch.equal(m.env_map.detach(), env0)


# ---- 5. miss ----------------------------------------------------------------------------------------------------------
def test_a_ray_that_misses_the_sphere_raises_and_moves_nothing():
    from fdgs.graph import GraphedStep
    m, cams, gts = _sky_lego()
    bg = torch.zeros(3, device=DEV)
    step = GraphedStep(_fn(m, _l1, bg), m, optimizer=m.optimizer)
    out = _outside(int(cams[0].image_width), int(cams[0].image_height))
    bad, good = [cams[0], out], cams[:2]
    gt = torch.stack(gts[:2])

    def unchanged(call):
        before = _clone(m)
        with pytest.raises(AssertionError, match=MISS):
            call()
        _assert_equal(m, before, "miss")

    m.optimizer.init_state()          # every call allocates the state first: compare moments, not their allocation
    unchanged(lambda: step(bad, gt, densify_stats=True))           # in the warm-up
    assert step.info["captures"] == 0
    step(good, gt, densify_stats=True)
    step(good, gt, densify_stats=True)
    captures = step.info["captures"]
    unchanged(lambda: step(bad, gt, densify_stats=True, hold={"opacity"}))   # in a replay
    before = _clone(m)
    step(good, gt, densify_stats=True)
    assert step.info["captures"] == captures, step.info
    assert float(m.optimizer.state[m.env_map]["step"]) == float(before.optimizer.state[before.env_map]["step"]) + 1
    assert not torch.equal(m.env_map.detach(), before.env_map.detach())


# ---- 6. synchronisation ---------------------------------------------------------------------------------------------
def test_the_status_read_is_the_only_synchronisation_with_a_map():
    from fdgs.graph import GraphedStep
    m, cams, gts = _sky_lego()
    bg = torch.zeros(3, device=DEV)
    step = GraphedStep(_fn(m, _l1, bg), m, optimizer=m.optimizer)
    views, gt = cams[:2], torch.stack(gts[:2])
    for _ in range(2):
        step(views, gt, densify_stats=True)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            step(views, gt, densify_stats=True, hold={"env_map"})
        finally:
            torch.cuda.set_sync_debug_mode(0)
    syncs = [w for w in caught if "called a synchronizing CUDA operation" in str(w.message)]
    assert len(syncs) == 1, [str(w.message) for w in syncs]
    assert step.info["captures"] == 1 and step.views.sky


# ---- 7. training ----------------------------------------------------------------------------------------------------
# rel-L2 floors of parameter, exp_avg and exp_avg_sq (each also passes within 4x the eager loop's own run-to-run
# distance).  The eager loop repeats itself almost bit for bit, so the floors carry the comparison: the graph renders
# through the capacity-sized entry, whose blend backward accumulates in another order, and the covariance chain
# (rotations, scales) amplifies that order's rounding -- on an H100 the graphed lego loop of test_gpu_graph_iteration.py
# already sits at 1.05e-5 on the rotations after one iteration.  1e-4 is the chain's bar in the raw-entry tests.
FLOORS = (1e-4, 1e-2, 2e-2)

def test_coffee_martini_shaped_loop_tracks_the_eager_loop():
    import fdgs.densify as D
    from fdgs.dist import ViewBatchStats
    from fdgs.graph import GraphedStep
    from test_gpu_densify_train import _max_grad
    m, cams, gts = _sky_lego(P=20000, W=200, H=200, env_hw=(100, 200))
    bg = torch.zeros(3, device=DEV)
    batch, iters = 4, 40
    densify_at, reset_at, env_until = 15, 25, 20
    step = GraphedStep(_fn(m, _l1, bg), m, optimizer=m.optimizer)
    gauss = _gaussian_groups(m)
    xyz_lr = lambda it: 1.6e-4 * (1.6e-6 / 1.6e-4) ** (it / iters)     # noqa: E731  (expon_lr_func's log-linear decay)

    def hold_of(densify, reset, env_on, last):
        """The graphed iteration's hold: the Gaussian groups on a densification iteration (the map still steps), the
        opacity on an opacity reset (the reset replaces its leaf), the map from env_optimize_until on, everything on
        the last iteration."""
        if last:
            return True
        hold = set(gauss) if densify else ({"opacity"} if reset else set())
        if not env_on:
            hold.add("env_map")
        return hold

    def run_eager(c, views, gt, reset, hold):
        """The reference's order: statistics -> densify / reset -> Gaussian Adam -> env Adam (a held leaf: no step)."""
        _, pkg = _eager_grads(c, views, gt, _l1, bg)
        st = ViewBatchStats(c._xyz.shape[0], DEV)
        for j in range(len(views)):
            st.add_view(pkg["viewspace_points"].grad[j], pkg["radii"][j])
        D.add_densification_stats(c, t_grad=c._t.grad, batch_stats=st, batch_size=len(views))
        if reset:
            D.reset_opacity(c)
        held = c.optimizer.held(hold)
        env_grad = None if id(c.env_map) in held else c.env_map.grad
        c.env_map.grad = None
        _eager_step(c, hold)                                           # the Gaussian Adam
        for p in _leaves(c):
            p.grad = None
        c.env_map.grad = env_grad
        c.optimizer.step()                                             # the env Adam
        return c

    worst = {}
    for it in range(iters):
        for g in m.optimizer.param_groups:
            if g["name"] == "xyz":
                g["lr"] = xyz_lr(it)
        views = [(it * batch + k) % len(cams) for k in range(batch)]
        vc, gt = [cams[k] for k in views], torch.stack([gts[k] for k in views])
        reset, densify, last = it == reset_at, it == densify_at, it == iters - 1
        hold = hold_of(densify, reset, it < env_until, last)
        e1 = run_eager(_clone(m), vc, gt, reset, hold)
        e2 = run_eager(_clone(m), vc, gt, reset, hold)
        step(vc, gt, densify_stats=True, hold=hold)
        if reset:
            D.reset_opacity(m)
        (sg, tg), (s1, t1), (s2, t2) = _state(m), _state(e1), _state(e2)
        for name in sg:
            assert sg[name][3] == s1[name][3], (it, name)
            for i, floor in enumerate(FLOORS):
                err, noise = _rel(sg[name][i], s1[name][i]), _rel(s2[name][i], s1[name][i])
                worst[(name, i)] = max(worst.get((name, i), 0.0), err / max(floor, 4 * noise))
                assert err <= max(floor, 4 * noise), (it, name, i, err, noise)
        for n in tg:
            err, noise = _rel(tg[n], t1[n]), _rel(t2[n], t1[n])
            assert err <= max(1e-3, 4 * noise), (it, n, err, noise)
        if densify:
            P0 = m._xyz.shape[0]
            D.densify_and_prune(m, _max_grad(m), 0.005, 1.2, None)
            assert m._xyz.shape[0] != P0
            assert m.optimizer.param_groups[-1]["params"][0] is m.env_map and m.env_map in m.optimizer.state
    print("worst err / bar:", {"%s.%d" % k: round(v, 3) for k, v in sorted(worst.items())})
    counts = {g["name"]: float(m.optimizer.state[g["params"][0]]["step"]) for g in m.optimizer.param_groups}
    assert counts["env_map"] == env_until, counts
    assert step.info["captures"] >= 2 and step.info["overflows"] == 0, step.info
