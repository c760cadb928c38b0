"""GPU (-m gpu): the camera gradients of the single-view backward (rasterize_gaussians_backward_camera) entry by entry
against the float64 sum of their per-row terms (camera_chain_f64.py), fed what the backward itself consumed: the
blend gradients geom_bwd_body converted and left in the slab (test_gpu_gauss_f64._outputs), the forward's cov3D, shifted
means and clamp bits.  Every one of the 27 returned entries lies within K bound + tiny of the float64 sum, the bound
being the rows' first-order fp32 bounds plus the kernels' reduction model (calibrated on the CPU oracle by
test_camera_chain_f64.py); the 8 unused entries are exactly 0.  Through the reference-layout entry (colour-only and all
four upstream images, both tile-list modes), the raw-parameter entry with split SH rows, a per-pixel background,
precomputed colours (campos exactly 0) and scenes of one Gaussian."""
import dataclasses

import pytest
import torch

import camera_chain_f64 as CC
import gauss_f64 as G
import helpers
from test_gpu_gauss_f64 import RAW_CASES, _geom, _outputs, _upstream

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = G.CASES + ["regime:deep", "mid"]


@pytest.fixture(scope="module")
def C():
    import fdgs
    return fdgs.ext()


@pytest.fixture(params=[1, 0], ids=["tilecull", "reflists"])
def tile_mode(request):
    import fdgs
    prev = fdgs.set_tile_cull(request.param)
    yield request.param
    fdgs.set_tile_cull(prev)


def _build(case):
    if case.startswith("one:"):
        cfg, cam, sc, st = CC.one_scene(case[4:])
        from fdgs import synth
        sc = sc.to(DEV)
        return cfg, cam, sc, synth.raster_settings(cam, sc, device=DEV), -1.0
    return G.build_case(case, device=DEV)


def _camera_backward(C, args, sh_rest=None, raw=False, bg_image=None, zero_rows=()):
    e = torch.empty(0, device=DEV)
    extra = tuple(zero_rows) if zero_rows else (e, e)
    return C.rasterize_gaussians_backward_camera(*args, e if sh_rest is None else sh_rest, raw,
                                                 e if bg_image is None else bg_image, False, False, *extra)


def _check(label, C, fw, bw, sc, st, has_sh=True):
    torch.cuda.synchronize()
    clamped, vis = _geom(C, fw, sc.P)
    out = _outputs(bw, fw)
    r = CC.restate(sc, st, out, clamped, fw[10], vis, has_sh=has_sh)
    got = torch.cat([bw[15].reshape(-1), bw[16].reshape(-1), bw[17].reshape(-1)])
    worst = CC.check_sums(label, got, r, rows=int(vis.sum()))
    if not has_sh:
        assert bw[17].tolist() == [0.0, 0.0, 0.0], (label, "campos with precomputed colours")
    return worst, vis


@pytest.mark.parametrize("aux", [False, True], ids=["colour", "aux"])
@pytest.mark.parametrize("case", CASES)
def test_camera_grads_vs_float64(C, case, tile_mode, aux):
    if case == "mid" and (tile_mode == 0 or aux):
        pytest.skip("100k Gaussians: one tile mode and upstream are enough")
    cfg, cam, sc, st, pv = G.build_case(case, device=DEV)
    fw = C.rasterize_gaussians(*helpers.fwd_args(st, sc, cfg))
    bw = _camera_backward(C, helpers.bwd_args(st, sc, cfg, fw, _upstream(cfg, aux)))
    _check("%s %s %s" % (case, ["reflists", "tilecull"][tile_mode], "aux" if aux else "colour"), C, fw, bw, sc, st)


@pytest.mark.parametrize("name", CC.ONE_SCENES + ["edge:p1"])
def test_one_gaussian_vs_float64(C, name, tile_mode):
    case = name if name.startswith("edge:") else "one:" + name
    cfg, cam, sc, st, pv = _build(case)
    fw = C.rasterize_gaussians(*helpers.fwd_args(st, sc, cfg))
    bw = _camera_backward(C, helpers.bwd_args(st, sc, cfg, fw, _upstream(cfg, True)))
    _, vis = _check("%s %s" % (case, ["reflists", "tilecull"][tile_mode]), C, fw, bw, sc, st)
    if case.startswith("one:"):
        CC.one_scene_regime(name, st, sc.means3D, fw[10], fw[5].cpu(), vis.cpu())
    else:
        assert int(vis.sum()) == 1


@pytest.mark.parametrize("zero_rows", [False, True], ids=["bwd_zero_rows", "fwd_zero_rows"])
@pytest.mark.parametrize("case", RAW_CASES)
def test_raw_entry_vs_float64(C, case, zero_rows):
    """The raw-parameter entry with SH as features_dc | features_rest (test_gpu_gauss_f64.test_raw_entry_split_rows_
    vs_float64's inputs); the camera terms read the activated values, so the restatement takes the activated scene."""
    cfg, cam, sc, st, pv = G.build_case(case, device=DEV)
    g = torch.Generator().manual_seed(cfg["seed"] + 5)
    P = sc.P
    logits = torch.logit(sc.opacities.double()).float()
    logits[torch.arange(P, device=DEV) % 16 == 3] = 20.0
    norm = lambda q: q * (0.5 + 1.5 * torch.rand(q.shape[0], 1, generator=g)).to(DEV)
    rs = dataclasses.replace(sc, scales=torch.log(sc.scales), scales_t=torch.log(sc.scales_t), opacities=logits,
                             rotations=norm(sc.rotations).contiguous(), rotations_r=norm(sc.rotations_r).contiguous(),
                             shs=sc.shs[:, :1].contiguous())
    rest = sc.shs[:, 1:].contiguous()
    e = torch.empty(0, device=DEV)
    M = sc.shs.shape[1]
    extra = ()
    if zero_rows:
        extra = (torch.full((P, 1, 3), float("nan"), device=DEV), torch.full((P, M - 1, 3), float("nan"), device=DEV))
    fw = C.rasterize_gaussians_ext(*helpers.fwd_args(st, rs, cfg), rest, True, e, *extra)
    bw = _camera_backward(C, helpers.bwd_args(st, rs, cfg, fw, _upstream(cfg, True)), sh_rest=rest, raw=True,
                          zero_rows=extra)
    _check("raw %s %s" % (case, "fwd zero rows" if zero_rows else "bwd zero rows"), C, fw, bw, sc, st)


@pytest.mark.parametrize("case", ["flowbg", "regime:opaque"])
def test_background_image_vs_float64(C, case):
    cfg, cam, sc, st, pv = G.build_case(case, device=DEV)
    bgi = torch.rand(3, cfg["H"], cfg["W"], generator=torch.Generator().manual_seed(cfg["seed"] + 7)).to(DEV)
    fw = C.rasterize_gaussians_ext(*helpers.fwd_args(st, sc, cfg), torch.empty(0), False, bgi)
    bw = _camera_backward(C, helpers.bwd_args(st, sc, cfg, fw, _upstream(cfg, True)), bg_image=bgi)
    _check("%s bg_image" % case, C, fw, bw, sc, st)


@pytest.mark.parametrize("case", ["tiny", "rotcam", "dur10"])
def test_precomputed_colours_vs_float64(C, case):
    """colours given instead of SH: no view direction, so campos is exactly 0; the view and projection entries are
    checked as everywhere else"""
    cfg, cam, sc, st, pv = G.build_case(case, device=DEV)
    colors = torch.rand(sc.P, 3, generator=torch.Generator().manual_seed(cfg["seed"] + 9)).to(DEV)
    e = torch.empty(0, device=DEV)
    fa = list(helpers.fwd_args(st, sc, cfg))
    fa[2], fa[19] = colors, e
    fw = C.rasterize_gaussians(*fa)
    ba = list(helpers.bwd_args(st, sc, cfg, fw, _upstream(cfg, True)))
    ba[4], ba[23] = colors, e
    bw = _camera_backward(C, ba)
    _check("%s colours" % case, C, fw, bw, sc, st, has_sh=False)
