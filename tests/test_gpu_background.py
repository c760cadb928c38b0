"""GPU (-m gpu): the per-pixel background image of the rasterizer (include/fdgs.h: fdgs_forward_bg / fdgs_backward_bg) --
the image is `rendered + (1 - alpha) * bg_image` bit for bit, every other output is unchanged, dL/dbg_image is
`(1 - alpha) * g` bit for bit on every pixel, and the Gaussian gradients match autograd through that composition, with
the colour-only blend backward doing the work."""
import ctypes

import pytest
import torch

import helpers
from raw_model import RawModel, Pipe

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = ["small", "flowbg", "ragged", "rotcam", "n3v", "mid", "cfg5"]
CHAIN = {"scales", "scales_t", "rotations", "rotations_r", "ts"}
RAW_CHAIN = {"scaling", "scaling_t", "rotation", "rotation_r", "t"}     # the same leaves under RawModel's names


def _fwd_bg(C, args, bgi):
    """rasterize_gaussians' 30 arguments with a per-pixel background: the extended entry without raw parameters"""
    return C.rasterize_gaussians_ext(*args, torch.empty(0), False, bgi)


def _bwd_bg(C, args, bgi):
    """rasterize_gaussians_backward's 37 arguments with a per-pixel background, dL/dbg_image wanted (index 14)"""
    return C.rasterize_gaussians_backward_ext(*args, torch.empty(0), False, bgi, False, True)


def _bg_image(cfg):
    return torch.rand(3, cfg["H"], cfg["W"], generator=torch.Generator().manual_seed(cfg["seed"] + 7)).to(DEV)


@pytest.fixture(scope="module")
def C():
    import fdgs
    return fdgs.ext()


@pytest.mark.parametrize("name", CASES)
def test_extended_forward_is_the_torch_composition_bit_for_bit(C, name):
    cfg, cam, sc, st = helpers.build(name, device=DEV)
    bgi = _bg_image(cfg)
    fw0 = C.rasterize_gaussians(*helpers.fwd_args(st, sc, cfg))
    fw1 = _fwd_bg(C, helpers.fwd_args(st, sc, cfg), bgi)
    alpha = 1 - fw0[4]
    assert torch.equal(fw1[1], fw0[1] + (1 - alpha) * bgi)
    assert fw1[0] == fw0[0]
    for i in (2, 3, 4, 5, 10):   # flow, depth, T, radii, out_means3D
        assert torch.equal(fw1[i], fw0[i]), i
    vis = fw0[5] > 0             # covs_com: the rows of culled Gaussians are never written
    assert torch.equal(fw1[9][vis], fw0[9][vis])
    # an empty bg_image is "none"
    fw2 = _fwd_bg(C, helpers.fwd_args(st, sc, cfg), torch.empty(0, device=DEV))
    assert torch.equal(fw2[1], fw0[1])

    # dL/dbg_image on every pixel, including the tiles with empty lists
    gc, gd, ga, gf = helpers.pixel_grads(cfg, device=DEV)
    none = torch.empty(0, device=DEV)
    bw = _bwd_bg(C, helpers.bwd_args(st, sc, cfg, fw1, (gc, none, none, none)), bgi)
    assert torch.equal(bw[14], (1 - alpha) * gc)


def _leaves(sc):
    keys = ("means3D", "shs", "opacities", "scales", "scales_t", "rotations", "rotations_r", "ts")
    return {k: getattr(sc, k).detach().clone().requires_grad_(True) for k in keys}


def blend_kernel_floor(grads_fn):
    """How far the two backward formulations of a background lie apart where the rasterizer can express both: a
    CONSTANT background c either through the settings' `bg` (the colour-only kernel folds it into T_final (bg . g), as
    it folds bg_image) or composed in torch as `rendered + (1 - alpha) * c` (autograd hands the alpha image a gradient:
    the AUX kernel's alpha recurrence, whose 1 - acc_alpha cancels where little light is left).  grads_fn(native) ->
    {name: grad}.  That distance is what separates the native path from the torch composition in the test below."""
    a, b = grads_fn(True), grads_fn(False)
    return {k: helpers.l2_rel(helpers.to_np(a[k]), helpers.to_np(b[k])) for k in a}


def _render(st, sc, L, bgi):
    from gaussian_renderer import GaussianRasterizationSettings, GaussianRasterizer
    rast = GaussianRasterizer(GaussianRasterizationSettings(**st))
    m2 = torch.zeros_like(L["means3D"], requires_grad=True)
    out = rast(means3D=L["means3D"], means2D=m2, opacities=L["opacities"], shs=L["shs"], flow_2d=sc.flow_2d, ts=L["ts"],
               scales=L["scales"], scales_t=L["scales_t"], rotations=L["rotations"], rotations_r=L["rotations_r"],
               bg_image=bgi)
    return out, m2


@pytest.mark.parametrize("name", CASES)
def test_gradients_match_autograd_through_the_composition(name):
    cfg, cam, sc, st = helpers.build(name, device=DEV)
    gc = helpers.pixel_grads(cfg, device=DEV)[0]
    bg_a = _bg_image(cfg).requires_grad_(True)
    bg_b = bg_a.detach().clone().requires_grad_(True)
    A, B = _leaves(sc), _leaves(sc)
    (ca, _, da, aa, fa, _), m2a = _render(st, sc, A, bg_a)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        (ca * gc).sum().backward()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert any("blend_bwd2_kernel<3, true, false>" in n for n in names), "colour-only blend backward did not run"
    (cb, _, db, ab, fb, _), m2b = _render(st, sc, B, None)
    assert torch.equal(da, db) and torch.equal(aa, ab) and torch.equal(fa, fb)
    assert torch.equal(ca, cb + (1 - ab) * bg_b)
    ((cb + (1 - ab) * bg_b) * gc).sum().backward()
    assert torch.equal(bg_a.grad, (1 - aa.detach()) * gc)
    assert torch.equal(bg_a.grad, bg_b.grad)
    cbg = float(bg_b.detach().mean())

    def grads(native):
        L = _leaves(sc)
        s = dict(st, bg=(st["bg"] + cbg) if native else st["bg"])
        (c, _, _, a, _, _), m2 = _render(s, sc, L, None)
        ((c if native else c + (1 - a) * cbg) * gc).sum().backward()
        return dict({k: t.grad for k, t in L.items()}, means2D=m2.grad)
    floor = blend_kernel_floor(grads)
    for k in list(A) + ["means2D"]:
        a, b = (m2a.grad, m2b.grad) if k == "means2D" else (A[k].grad, B[k].grad)
        err = helpers.l2_rel(helpers.to_np(a), helpers.to_np(b))
        bar = max(2e-3 if (k in CHAIN and cfg["P"] >= 50000) else 1e-4, 4 * floor[k])
        print("%s %-11s rel-L2 %.2e (constant-background formulations: %.2e, bar %.2e)" % (name, k, err, floor[k], bar))
        assert err <= bar, (k, err, floor[k])


@pytest.mark.parametrize("name", ["small", "n3v", "mid"])
def test_raw_entry_with_background_image(name):
    from gaussian_renderer import GaussianRasterizationSettings, GaussianRasterizer
    cfg, cam, sc, st = helpers.build(name, device=DEV)
    gc = helpers.pixel_grads(cfg, device=DEV)[0]
    rast = GaussianRasterizer(GaussianRasterizationSettings(**st))
    out = {}
    for tag in ("native", "torch"):
        M = RawModel(sc, seed=3, requires_grad=True)
        bgi = _bg_image(cfg).requires_grad_(True)
        m2 = torch.zeros_like(M._xyz, requires_grad=True)
        kw = dict(means3D=M._xyz, means2D=m2, opacity_logits=M._opacity, features_dc=M._features_dc,
                  features_rest=M._features_rest, log_scales=M._scaling, rotations_raw=M._rotation, flow_2d=sc.flow_2d,
                  ts=M._t, log_scales_t=M._scaling_t, rotations_r_raw=M._rotation_r)
        if tag == "native":
            img = rast.forward_raw(bg_image=bgi, **kw)[0]
        else:
            c, _, _, a, _, _ = rast.forward_raw(**kw)
            img = c + (1 - a) * bgi
        (img * gc).sum().backward()
        out[tag] = (img.detach(), M.leaves(), bgi.grad, m2.grad)
    assert torch.equal(out["native"][0], out["torch"][0])
    assert torch.equal(out["native"][2], out["torch"][2])
    for k, a in out["native"][1].items():
        b = out["torch"][1][k]
        # the chain leaves at P >= 50000: the bar of test_gradients_match_autograd_through_the_composition (the same
        # native path run twice differs there by up to 1.2e-4 rel-L2: the blend backward's atomics, amplified)
        bar = 2e-3 if (k in RAW_CHAIN and cfg["P"] >= 50000) else 1e-4
        assert helpers.l2_rel(helpers.to_np(a.grad), helpers.to_np(b.grad)) <= bar, k
    assert helpers.l2_rel(helpers.to_np(out["native"][3]), helpers.to_np(out["torch"][3])) <= 1e-4


def test_extended_entry_with_no_gaussians_is_the_background(C):
    """P = 0: the image is the background and dL/dbg_image is the whole image gradient times T = 1."""
    cfg, cam, sc, st = helpers.build("ragged", device=DEV)
    bgi = _bg_image(cfg)
    a = list(helpers.fwd_args(st, sc, cfg))
    for i, t in enumerate(a):
        if isinstance(t, torch.Tensor) and t.dim() >= 1 and t.shape[0] == cfg["P"] and t.device.type == "cuda":
            a[i] = t[:0].contiguous()
    fw = _fwd_bg(C, a, bgi)
    assert fw[0] == 0 and bool((fw[4] == 1).all())
    assert torch.equal(fw[1], (fw[1] - fw[1]) + st["bg"].view(3, 1, 1) + (1 - (1 - fw[4])) * bgi)
    gc = helpers.pixel_grads(cfg, device=DEV)[0]
    e = torch.empty(0, device=DEV)
    b = list(helpers.bwd_args(st, sc, cfg, fw, (gc, e, e, e)))
    b[1] = a[1]
    bw = _bwd_bg(C, b, bgi)
    assert torch.equal(bw[14], (1 - (1 - fw[4])) * gc)


@pytest.mark.parametrize("name", ["small", "rotcam"])
def test_ctypes_forward_bg_matches_the_extended_entry(C, name):
    """fdgs_forward_bg through ctypes: NULL is fdgs_forward bit for bit, an image is the extension's result."""
    import fdgs
    from test_gpu_ctypes_abi import FwdArgs, FwdResult, ALLOC_FN, _p
    lib = fdgs.lib()
    cfg, cam, sc, st = helpers.build(name, device=DEV)
    P, W, H = cfg["P"], cfg["W"], cfg["H"]
    bgi = _bg_image(cfg)
    keep = []

    @ALLOC_FN
    def alloc(ctx, nbytes):
        t = torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=DEV)
        keep.append(t)
        return t.data_ptr()

    def run(fn, *extra):
        f32 = dict(dtype=torch.float32, device=DEV)
        out = dict(means=torch.empty(P, 3, **f32), color=torch.empty(3, H, W, **f32), flow=torch.empty(2, H, W, **f32),
                   depth=torch.empty(1, H, W, **f32), T=torch.empty(1, H, W, **f32),
                   radii=torch.empty(P, dtype=torch.int32, device=DEV))
        a = FwdArgs()
        a.P, a.D, a.D_t, a.M = P, st["sh_degree"], st["sh_degree_t"], sc.shs.shape[1]
        a.background, a.width, a.height = _p(st["bg"]), W, H
        a.means3D, a.shs, a.flows_precomp, a.opacities = _p(sc.means3D), _p(sc.shs), _p(sc.flow_2d), _p(sc.opacities)
        a.ts, a.scales, a.scales_t, a.scale_modifier = _p(sc.ts), _p(sc.scales), _p(sc.scales_t), st["scale_modifier"]
        a.rotations, a.rotations_r, a.prefilter_var = _p(sc.rotations), _p(sc.rotations_r), -1.0
        a.viewmatrix, a.projmatrix, a.cam_pos = _p(st["viewmatrix"]), _p(st["projmatrix"]), _p(st["campos"])
        a.timestamp, a.time_duration, a.rot_4d, a.gaussian_dim = st["timestamp"], st["time_duration"], 1, 4
        a.tan_fovx, a.tan_fovy = st["tanfovx"], st["tanfovy"]
        a.out_means3D, a.out_color, a.out_flow, a.out_depth, a.out_T = (_p(out["means"]), _p(out["color"]),
                                                                        _p(out["flow"]), _p(out["depth"]), _p(out["T"]))
        a.radii = _p(out["radii"], ctypes.POINTER(ctypes.c_int))
        res = FwdResult()
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        fn.restype = ctypes.c_int
        rc = fn(ctypes.byref(a), *extra, alloc, None, alloc, None, alloc, None, stream, ctypes.byref(res))
        assert rc == 0, lib.fdgs_last_error()
        torch.cuda.synchronize()
        return out

    plain = run(lib.fdgs_forward)
    null = run(lib.fdgs_forward_bg, _p(None))
    img = run(lib.fdgs_forward_bg, _p(bgi))
    fw = _fwd_bg(C, helpers.fwd_args(st, sc, cfg), bgi)
    for k in plain:
        assert torch.equal(plain[k], null[k]), k
    assert torch.equal(img["color"], fw[1])
    for k in ("flow", "depth", "T", "radii", "means"):
        assert torch.equal(img[k], plain[k]), k
