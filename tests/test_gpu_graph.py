"""GPU (-m gpu): the batched forward sized by an instance capacity and the training step as one CUDA graph.

  1. exactness: called eagerly at capacity R, R + 1 and 2 R the capacity entry equals rasterize_gaussians_batch bit for
     bit (images, radii, out_means3D, n_contrib, tile ranges and lists), and status = {R, largest tile, 0, 0};
  2. overflow (capacity 0, R - 1, R / 2): status reports it and the true R, the views render as if no Gaussian were
     listed, radii are still the exact call's, the backward returns zero gradients, and no write leaves the binning
     buffer;
  3. a capacity forward + backward makes no host synchronisation on the PyTorch side, and the entry refuses debug while
     the stream is capturing;
  4. graph replay: one capture of render + l1_ssim_loss + backward replayed with several camera sets equals eager
     render_batch (images and radii bit for bit, gradients and densification statistics within _cmp's bars);
  5. GraphedStep re-captures on overflow, densification and an SH degree change, and rejects what it cannot capture;
  6. training: a lego-shaped loop on GraphedStep + FusedAdam with densification tracks the eager render_batch loop.
"""
import ctypes
import math

import pytest
import torch

import helpers
import regimes
from test_gpu_batch import GOLDEN, _batch, _inputs, _settings
from test_gpu_view_parallel import DEV, _Model, _cmp, _views

pytestmark = pytest.mark.gpu


def _C():
    import fdgs
    return fdgs.ext()


def _cap(sts, sc, cfg, g, raw, bg_image, capacity):
    e = torch.Tensor([])
    st = sts[0]
    f32 = lambda k: torch.tensor([s[k] for s in sts], dtype=torch.float32, device=DEV)
    return _C().rasterize_gaussians_batch_capacity(
        st["bg"], sc.means3D, sc.flow_2d, g["opacity"], g["ts"], g["scales"], g["scales_t"], g["rotations"],
        g["rotations_r"], st["scale_modifier"], cfg.get("prefilter_var", -1.0),
        torch.stack([s["viewmatrix"] for s in sts]), torch.stack([s["projmatrix"] for s in sts]),
        torch.stack([s["campos"] for s in sts]), f32("timestamp"), f32("tanfovx"), f32("tanfovy"), st["image_height"],
        st["image_width"], g["sh"], g["sh_rest"], st["sh_degree"], st["sh_degree_t"], st["time_duration"], st["rot_4d"],
        st["gaussian_dim"], st["force_sh_3d"], st["prefiltered"], False, raw, e if bg_image is None else bg_image,
        capacity)


def _largest_tile(img_b, W, H, B):
    return max(int((rg[:, 1] - rg[:, 0]).max()) for rg in (_C().debug_export_binning_view(img_b, W, H, B, v)[0]
                                                             for v in range(B)))


def _check_exact(cfg, sc, cams, raw=False, split=False, sky=False):
    """The capacity entry at R, R + 1, 2 R against the exact entry; returns the largest tile."""
    sts = _settings(cams, sc, cfg)
    B, H, W = len(cams), cfg["H"], cfg["W"]
    g = _inputs(sc, raw, split)
    bgs = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(3)).to(DEV) if sky else None
    ex = _batch(sts, sc, cfg, g, raw, bgs)
    R = ex[0]
    pl_ex = _C().debug_export_binning(ex[7], ex[8], R, W, H)[0]
    big = _largest_tile(ex[8], W, H, B)
    for capacity in sorted({R, R + 1, 2 * R}):
        got = _cap(sts, sc, cfg, g, raw, bgs, capacity)
        assert got[0].tolist() == [R, big, 0, 0], (capacity, got[0].tolist(), R, big)
        for i in range(1, 6):
            assert torch.equal(got[i], ex[i]), (capacity, i)
        assert torch.equal(got[9], ex[9]), capacity
        for v in range(B):
            rg, nc = _C().debug_export_binning_view(got[8], W, H, B, v)
            rg_e, nc_e = _C().debug_export_binning_view(ex[8], W, H, B, v)
            assert torch.equal(rg, rg_e) and torch.equal(nc, nc_e), (capacity, v)
        if capacity > 0:
            pl = _C().debug_export_binning(got[7], got[8], capacity, W, H)[0]
            assert torch.equal(pl[:R], pl_ex), capacity
    return big


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("name", GOLDEN)
def test_capacity_entry_is_the_exact_entry_bit_for_bit(name, B):
    cfg, _, sc, _ = helpers.build(name, device=DEV)
    _check_exact(cfg, sc, _views(cfg, B, DEV))


@pytest.mark.parametrize("tile_cull", [0, 1])
@pytest.mark.parametrize("raw,split,sky", [(False, False, False), (True, True, False), (False, True, True),
                                           (True, False, True)])
def test_capacity_entry_entries_and_tile_modes(tile_cull, raw, split, sky):
    import fdgs
    old = fdgs.lib().fdgs_set_tile_cull(tile_cull)
    try:
        cfg, _, sc, _ = helpers.build("n3v", device=DEV)
        _check_exact(cfg, sc, _views(cfg, 3, DEV), raw=raw, split=split, sky=sky)
    finally:
        fdgs.lib().fdgs_set_tile_cull(old)


def test_capacity_entry_runs_the_large_tile_sort():
    """The host does not know the largest tile, so both size classes of the tile sort run: the regimes, and crowded
    scenes whose tiles take the large class (> 2048 instances) and its in-place fallback (> 16384)."""
    biggest = []
    for regime in ("deep", "huge"):
        cfg, cam, sc, _ = getattr(regimes, regime)()
        sc = sc.to(DEV)
        biggest.append(_check_exact(cfg, sc, [cam.to(DEV)] + _views(cfg, 2, DEV)))
    for crowd in (dict(P=60000, W=96, H=96, seed=21), dict(P=300000, W=64, H=64, seed=22)):
        cfg, _, sc, _ = helpers.build(crowd, device=DEV)
        biggest.append(_check_exact(cfg, sc, _views(cfg, 2, DEV)))
    assert any(2048 < b <= 16384 for b in biggest) and max(biggest) > 16384, biggest


# ---- 2. overflow ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,B", [("small", 1), ("n3v", 3), ("mid", 2)])
def test_overflow_renders_no_gaussian_and_returns_zero_gradients(name, B):
    from fdgs.graph import StaticViews
    from gaussian_renderer import render_batch
    from test_gpu_view_parallel import _Pipe
    cfg, _, sc, _ = helpers.build(name, device=DEV)
    cams = _views(cfg, B, DEV)
    sts = _settings(cams, sc, cfg)
    H, W = cfg["H"], cfg["W"]
    g = _inputs(sc, False, False)
    ex = _batch(sts, sc, cfg, g, False, None)
    R = ex[0]
    assert R > 2
    big = _largest_tile(ex[8], W, H, B)
    bg = sts[0]["bg"].to(DEV)
    for capacity in (0, R - 1, R // 2):
        got = _cap(sts, sc, cfg, g, False, None, capacity)
        assert got[0].tolist() == [R, big, 1, 0], capacity
        assert torch.equal(got[1], bg.view(1, 3, 1, 1).expand(B, 3, H, W).contiguous()), capacity
        assert int(got[2].abs().sum()) == 0 and int(got[3].abs().sum()) == 0, capacity
        assert bool((got[4] == 1.0).all()), capacity     # T = 1: alpha 0
        assert torch.equal(got[5], ex[5]) and torch.equal(got[9], ex[9]), capacity
        for v in range(B):
            rg, nc = _C().debug_export_binning_view(got[8], W, H, B, v)
            assert int(rg.abs().sum()) == 0 and int(nc.abs().sum()) == 0, (capacity, v)
    # the backward over an overflowed forward: zero per-Gaussian gradients
    pc = _Model(sc)
    views = StaticViews(B, H, W, DEV)
    views.load(cams)
    views.capacity = R - 1
    pkg = render_batch(views, pc, _Pipe(), torch.zeros(3, device=DEV))
    assert pkg["status"].tolist()[2] == 1
    G = torch.randn(pkg["render"].shape, generator=torch.Generator().manual_seed(5)).to(DEV)
    ((pkg["render"] * G).sum() + pkg["depth"].sum() + pkg["alpha"].sum()).backward()
    for p in pc.geometry() + pc.sh_leaves:
        assert p.grad is not None and float(p.grad.abs().sum()) == 0.0
    assert float(pkg["viewspace_points"].grad.abs().sum()) == 0.0


def test_overflow_writes_nothing_past_the_binning_buffer():
    """Through the C-ABI with a binning buffer 1 MB longer than requested and filled with a pattern: at capacity R - 1 the
    tail is untouched (R - 1, not a capacity far below R: even a scatter without its overflow guard would write at most
    one key past the buffer's keys, inside the allocation)."""
    import fdgs
    from test_abi_batch import ForwardResult
    from test_abi_graph import ForwardCapacityArgs
    lib = fdgs.lib()
    lib.fdgs_forward_batch_capacity.restype = ctypes.c_int
    lib.fdgs_binning_bytes.restype = ctypes.c_size_t
    cfg, _, sc, _ = helpers.build("mid", device=DEV)
    B, H, W = 2, cfg["H"], cfg["W"]
    cams = _views(cfg, B, DEV)
    sts = _settings(cams, sc, cfg)
    R = _batch(sts, sc, cfg, _inputs(sc, False, False), False, None)[0]
    TAIL = 1 << 20
    keep = []
    requested = {}

    def alloc_fn(tag):
        @ctypes.CFUNCTYPE(ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t)
        def alloc(ctx, n):
            extra = TAIL if tag == "binning" else 0
            t = torch.full((n + extra,), 0xA5, dtype=torch.uint8, device=DEV)
            keep.append(t)
            requested[tag] = (t, n)
            return t.data_ptr()
        return alloc

    allocs = {k: alloc_fn(k) for k in ("geom", "binning", "image")}
    fp = lambda t: ctypes.cast(t.data_ptr(), ctypes.POINTER(ctypes.c_float)) if t is not None and t.numel() else None
    outs = dict(out_means3D=torch.empty(B, sc.P, 3, device=DEV), out_color=torch.empty(B, 3, H, W, device=DEV),
                out_flow=torch.empty(B, 2, H, W, device=DEV), out_depth=torch.empty(B, 1, H, W, device=DEV),
                out_T=torch.empty(B, 1, H, W, device=DEV))
    radii = torch.empty(B, sc.P, dtype=torch.int32, device=DEV)
    status = torch.empty(4, dtype=torch.int32, device=DEV)
    cams_t = dict(viewmatrix=torch.stack([s["viewmatrix"] for s in sts]).contiguous(),
                  projmatrix=torch.stack([s["projmatrix"] for s in sts]).contiguous(),
                  cam_pos=torch.stack([s["campos"] for s in sts]).contiguous())
    scal = {k: torch.tensor([s[k] for s in sts], dtype=torch.float32, device=DEV) for k in ("timestamp", "tanfovx", "tanfovy")}
    bg = sts[0]["bg"].to(DEV).contiguous()
    c = ForwardCapacityArgs()
    a = c.batch.view
    a.P, a.D, a.D_t, a.M, a.width, a.height = sc.P, sc.sh_degree, sc.sh_degree_t, sc.shs.shape[1], W, H
    a.background, a.means3D, a.shs, a.opacities = fp(bg), fp(sc.means3D), fp(sc.shs), fp(sc.opacities)
    a.ts, a.scales, a.scales_t, a.rotations, a.rotations_r = fp(sc.ts), fp(sc.scales), fp(sc.scales_t), fp(sc.rotations), fp(sc.rotations_r)
    a.flows_precomp = fp(sc.flow_2d)
    a.scale_modifier, a.prefilter_var, a.time_duration = sts[0]["scale_modifier"], -1.0, sts[0]["time_duration"]
    a.rot_4d, a.gaussian_dim, a.force_sh_3d = int(sc.rot_4d), sc.gaussian_dim, int(sc.force_sh_3d)
    for k, t in cams_t.items():
        setattr(a, k, fp(t))
    for k, t in outs.items():
        setattr(a, k, fp(t))
    a.radii = ctypes.cast(radii.data_ptr(), ctypes.POINTER(ctypes.c_int))
    c.batch.B = B
    c.timestamps, c.tan_fovx, c.tan_fovy = fp(scal["timestamp"]), fp(scal["tanfovx"]), fp(scal["tanfovy"])
    c.capacity = R - 1
    c.status = ctypes.cast(status.data_ptr(), ctypes.POINTER(ctypes.c_int))
    res = ForwardResult()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = lib.fdgs_forward_batch_capacity(ctypes.byref(c), allocs["geom"], None, allocs["binning"], None, allocs["image"], None,
                                         stream, ctypes.byref(res))
    assert rc == 0, lib.fdgs_last_error()
    torch.cuda.synchronize()
    t, n = requested["binning"]
    assert n == lib.fdgs_binning_bytes(R - 1, W, H)
    assert status.tolist()[:3] == [R, status.tolist()[1], 1]
    assert bool((t[n:] == 0xA5).all())


# ---- 3. synchronisation -----------------------------------------------------------------------------------------
def test_capacity_forward_and_backward_do_not_synchronise():
    from fdgs.graph import StaticViews
    from gaussian_renderer import render_batch
    from test_gpu_view_parallel import _Pipe
    cfg, _, sc, _ = helpers.build("mid", device=DEV)
    cams = _views(cfg, 3, DEV)
    pc = _Model(sc)
    views = StaticViews(3, cfg["H"], cfg["W"], DEV)
    views.load(cams)
    views.capacity = 10 ** 6
    bg = torch.zeros(3, device=DEV)
    render_batch(views, pc, _Pipe(), bg)["render"].sum().backward()     # loads modules, builds the host placeholders
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        render_batch(views, pc, _Pipe(), bg)["render"].sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_debug_is_refused_while_capturing():
    cfg, _, sc, _ = helpers.build("small", device=DEV)
    cams = _views(cfg, 1, DEV)
    sts = _settings(cams, sc, cfg)
    g = _inputs(sc, False, False)
    e = torch.Tensor([])
    st = sts[0]
    dev_scalar = lambda k: torch.tensor([st[k]], dtype=torch.float32, device=DEV)
    call = lambda: _C().rasterize_gaussians_batch_capacity(
        st["bg"], sc.means3D, sc.flow_2d, g["opacity"], g["ts"], g["scales"], g["scales_t"], g["rotations"],
        g["rotations_r"], st["scale_modifier"], -1.0, st["viewmatrix"].view(1, 4, 4), st["projmatrix"].view(1, 4, 4),
        st["campos"].view(1, 3), ts_, fx_, fy_, st["image_height"], st["image_width"], g["sh"], g["sh_rest"],
        st["sh_degree"], st["sh_degree_t"], st["time_duration"], st["rot_4d"], st["gaussian_dim"], st["force_sh_3d"],
        st["prefiltered"], True, False, e, 1000)
    ts_, fx_, fy_ = dev_scalar("timestamp"), dev_scalar("tanfovx"), dev_scalar("tanfovy")
    call()                 # debug is accepted outside a capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        with pytest.raises(RuntimeError, match="capturing"):
            call()


# ---- 4. graph replay --------------------------------------------------------------------------------------------
def _step(pc, pipe):
    from gaussian_renderer import render_batch
    from fdgs.loss import l1_ssim_loss

    def fn(views, gt):
        pkg = render_batch(views, pc, pipe, torch.zeros(3, device=DEV))
        loss = sum(l1_ssim_loss(pkg["render"][k], gt[k]) for k in range(gt.shape[0]))
        loss.backward()
        return loss, pkg
    return fn


def _eager(pc, pipe, cams, gt):
    from fdgs.dist import ViewBatchStats
    from gaussian_renderer import render_batch
    from fdgs.loss import l1_ssim_loss
    for p in pc.geometry() + pc.sh_leaves:
        p.grad = None
    pkg = render_batch(cams, pc, pipe, torch.zeros(3, device=DEV))
    sum(l1_ssim_loss(pkg["render"][k], gt[k]) for k in range(gt.shape[0])).backward()
    stats = ViewBatchStats(pc.get_xyz.shape[0], DEV)
    for k in range(len(cams)):
        stats.add_view(pkg["viewspace_points"].grad[k], pkg["radii"][k])
    return pkg, stats


def _camera_sets(cfg, B, n):
    from fdgs import synth
    out = []
    for s in range(n):
        cams = []
        for v in range(B):
            R, T = synth.pose_from_euler(3.0 * s + 2.0 * v, -1.5 * s - v, 0.5 * s, 0.04 * v - 0.02 * s, 0.01 * s, -0.03 * v)
            cams.append(synth.make_camera(cfg["W"], cfg["H"], timestamp=0.3 + 0.1 * s + 0.05 * v,
                                          negative_fov=cfg.get("negative_fov", False), R=R, T=T).to(DEV))
        out.append(cams)
    return out


@pytest.mark.parametrize("name,B", [("mid", 3), ("n3v", 2), ("small", 1)])
def test_graph_replay_equals_eager_render_batch(name, B):
    from fdgs.dist import ViewBatchStats
    from fdgs.graph import GraphedStep
    from test_gpu_view_parallel import _Pipe
    cfg, _, sc, _ = helpers.build(name, device=DEV)
    got, ref = _Model(sc), _Model(sc)
    step = GraphedStep(_step(got, _Pipe()), lambda: got.geometry() + got.sh_leaves, margin=2.0)
    sets = _camera_sets(cfg, B, 3)
    for s, cams in enumerate(sets):
        gt = torch.rand(B, 3, cfg["H"], cfg["W"], generator=torch.Generator().manual_seed(40 + s)).to(DEV)
        loss, pkg = step(cams, gt)
        gs = ViewBatchStats(sc.P, DEV)
        for k in range(B):
            gs.add_view(pkg["viewspace_points"].grad[k], pkg["radii"][k])
        epkg, rs = _eager(ref, _Pipe(), cams, gt)
        for key in ("render", "radii", "depth", "alpha", "flow"):
            assert torch.equal(pkg[key], epkg[key]), (s, key)
        _cmp(got, ref, gs, rs, tol_sh=2e-6, tol_geo=1e-4, tol_chain=1e-3 if cfg["P"] < 50000 else 5e-3)
    assert step.info["captures"] == 1 and step.info["overflows"] == 0, step.info


# ---- 5. GraphedStep recovery ------------------------------------------------------------------------------------
def test_graphed_step_recaptures_once_on_overflow():
    from fdgs import synth
    from fdgs.graph import GraphedStep
    from test_gpu_view_parallel import _Pipe
    cfg, _, sc, _ = helpers.build("mid", device=DEV)
    got, ref = _Model(sc), _Model(sc)
    step = GraphedStep(_step(got, _Pipe()), lambda: got.geometry() + got.sh_leaves)
    R, T = synth.pose_from_euler(0.0, 180.0, 0.0, 0.0, 0.0, 0.0)    # looking away: R = 0 sizes the first capacity
    away = [synth.make_camera(cfg["W"], cfg["H"], timestamp=0.5, R=R, T=T).to(DEV) for _ in range(2)]
    gt = torch.rand(2, 3, cfg["H"], cfg["W"], generator=torch.Generator().manual_seed(7)).to(DEV)
    step(away, gt)
    assert step.info == {"captures": 1, "overflows": 0, "capacity": 0}
    cams = _views(cfg, 2, DEV)
    loss, pkg = step(cams, gt)
    assert step.info["captures"] == 2 and step.info["overflows"] == 1, step.info
    status = pkg["status"].tolist()
    assert status[2] == 0 and step.info["capacity"] == math.ceil(1.25 * status[0])
    epkg, rs = _eager(ref, _Pipe(), cams, gt)
    for key in ("render", "radii", "depth", "alpha", "flow"):
        assert torch.equal(pkg[key], epkg[key]), key
    from fdgs.dist import ViewBatchStats
    gs = ViewBatchStats(sc.P, DEV)
    for k in range(2):
        gs.add_view(pkg["viewspace_points"].grad[k], pkg["radii"][k])
    _cmp(got, ref, gs, rs, tol_sh=2e-6, tol_geo=1e-4, tol_chain=1e-3 if cfg["P"] < 50000 else 5e-3)


def _train_step(m, bg):
    from gaussian_renderer import render_batch
    from test_gpu_densify_train import _Pipe as TrainPipe

    def fn(views, gt):
        pkg = render_batch(views, m, TrainPipe(), bg)
        loss = sum((pkg["render"][k] - gt[k]).abs().mean() for k in range(gt.shape[0]))
        loss.backward()
        return loss, pkg
    return fn


def test_graphed_step_recaptures_on_densification_and_sh_degree():
    import fdgs.densify as D
    from fdgs.dist import ViewBatchStats
    from fdgs.graph import GraphedStep
    from test_gpu_densify_train import _lego_model, _max_grad
    m, cams, gts = _lego_model(20000, 256, 256, DEV)
    m.active_sh_degree = 2
    bg = torch.zeros(3, device=DEV)
    step = GraphedStep(_train_step(m, bg), m, margin=1.5)
    views, gt = cams[:2], torch.stack(gts[:2])
    for _ in range(2):
        step(views, gt)
    assert step.info["captures"] == 1
    _, pkg = step(views, gt)
    st = ViewBatchStats(m._xyz.shape[0], DEV)
    for k in range(2):
        st.add_view(pkg["viewspace_points"].grad[k], pkg["radii"][k])
    D.add_densification_stats(m, t_grad=m._t.grad, batch_stats=st, batch_size=2)
    P0 = m._xyz.shape[0]
    D.densify_and_prune(m, _max_grad(m), 0.005, 1.2, None)
    assert m._xyz.shape[0] != P0
    step(views, gt)
    assert step.info["captures"] == 2, step.info
    step(views, gt)
    assert step.info["captures"] == 2, step.info
    m.active_sh_degree = 3
    step(views, gt)
    assert step.info["captures"] == 3, step.info


def test_graphed_step_rejects_what_it_cannot_capture():
    from fdgs.dist import ViewParallelStep
    from fdgs.graph import GraphedStep
    from gaussian_renderer import render_batch
    from test_gpu_view_parallel import _Pipe, _SkyPipe
    cfg, _, sc, _ = helpers.build("small", device=DEV)
    pc = _Model(sc)
    cams = _views(cfg, 1, DEV)
    gt = torch.zeros(1, 3, cfg["H"], cfg["W"], device=DEV)
    leaves = lambda: pc.geometry() + pc.sh_leaves
    bg = torch.zeros(3, device=DEV)

    def with_pipe(pipe, **kw):
        return GraphedStep(lambda v, g: _with_loss(render_batch(v, pc, pipe, bg, **kw)), leaves)

    def _with_loss(pkg):
        loss = pkg["render"].sum()
        loss.backward()
        return loss, pkg

    debug = _Pipe(); debug.debug = True
    cov = _Pipe(); cov.compute_cov3D_python = True
    shs = _Pipe(); shs.convert_SHs_python = True
    for step, msg in ((with_pipe(_SkyPipe()), "environment map"), (with_pipe(debug), "debug"),
                      (with_pipe(_Pipe(), override_color=torch.zeros(sc.P, 3, device=DEV)), "override_color"),
                      (with_pipe(cov), "compute_cov3D_python"), (with_pipe(shs), "convert_SHs_python")):
        with pytest.raises(ValueError, match=msg):
            step(cams, gt)
    vstep = ViewParallelStep.__new__(ViewParallelStep)
    old = ViewParallelStep.current
    ViewParallelStep.current = classmethod(lambda cls: vstep)
    try:
        with pytest.raises(ValueError, match="ViewParallelStep"):
            with_pipe(_Pipe())(cams, gt)
    finally:
        ViewParallelStep.current = old


# ---- 6. training --------------------------------------------------------------------------------------------------
def test_training_loop_on_the_graphed_step():
    import fdgs.densify as D
    from fdgs.dist import ViewBatchStats
    from fdgs.graph import GraphedStep
    from gaussian_renderer import render_batch
    from test_gpu_densify_train import _lego_model, _max_grad, _Pipe as TrainPipe
    m, cams, gts = _lego_model(20000, 400, 400, DEV)
    bg = torch.zeros(3, device=DEV)
    batch = 4
    chain = ("xyz", "t", "scaling", "scaling_t", "rotation", "rotation_r")
    step = GraphedStep(_train_step(m, bg), m)

    def params():
        return [p for g in m.optimizer.param_groups for p in g["params"]]

    def eager(views):
        for p in params():
            p.grad = None
        pkg = render_batch([cams[k] for k in views], m, TrainPipe(), bg)
        loss = sum((pkg["render"][j] - gts[k]).abs().mean() for j, k in enumerate(views))
        loss.backward()
        stats = ViewBatchStats(m._xyz.shape[0], DEV)
        for j in range(len(views)):
            stats.add_view(pkg["viewspace_points"].grad[j], pkg["radii"][j])
        return [p.grad.clone() for p in params()], stats, float(loss)

    for it in range(30):
        views = [(it * batch + k) % len(cams) for k in range(batch)]
        ref, rs, loss_e = eager(views)
        again = eager(views)[0]
        for p in params():
            p.grad = None
        loss, pkg = step([cams[k] for k in views], torch.stack([gts[k] for k in views]))
        gs = ViewBatchStats(m._xyz.shape[0], DEV)
        for j in range(batch):
            gs.add_view(pkg["viewspace_points"].grad[j], pkg["radii"][j])
        assert abs(float(loss) - loss_e) <= 1e-5 * abs(loss_e), (it, float(loss), loss_e)
        for g, p, r, r2 in zip(m.optimizer.param_groups, params(), ref, again):
            err = helpers.l2_rel(helpers.to_np(p.grad), helpers.to_np(r))
            if g["name"] in chain:
                tol = max(1e-3, 4 * helpers.l2_rel(helpers.to_np(r2), helpers.to_np(r)))
            else:
                tol = 2e-6 if g["name"] in ("f_dc", "f_rest") else 1e-4
            assert err <= tol, (it, g["name"], err, tol)
        assert helpers.l2_rel(helpers.to_np(gs.grad_norm_sum), helpers.to_np(rs.grad_norm_sum)) <= 1e-4
        assert torch.equal(gs.visibility_count, rs.visibility_count) and torch.equal(gs.max_radii, rs.max_radii)
        D.add_densification_stats(m, t_grad=m._t.grad, batch_stats=gs, batch_size=batch)
        m.optimizer.step()
        m.optimizer.zero_grad(set_to_none=True)
        if it == 15:
            P0 = m._xyz.shape[0]
            D.densify_and_prune(m, _max_grad(m), 0.005, 1.2, None)
            assert m._xyz.shape[0] != P0
    assert step.info["captures"] >= 2, step.info
