"""GPU (-m gpu): the per-Gaussian backward (preprocess_bwd.cu) row by row against its float64 restatement
(gauss_f64.py), fed what the backward itself consumed and returned.  Every element of dL_dsh, dL_dmeans3D,
dL_dscales(_t), dL_drot(_r) and dL_dts of every rendered row lies within K err + tiny of the float64 value, err being
the first-order bound of an fp32 evaluation of the same expressions (calibrated on the CPU oracle by test_gauss_f64.py);
every row the backward did not render is exactly zero.  Through the reference-layout entry (colour-only and all four upstream images,
both tile-list modes) and the raw-parameter entry with split SH rows (with and without the forward writing the SH
gradient's zero rows)."""
import dataclasses

import pytest
import torch

import gauss_f64 as G
import helpers

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = G.CASES + ["regime:deep", "mid"]
OUT_IDX = dict(dL_dopacity=2, dL_dmeans3D=3, dL_dcov3D=4, dL_dsh=5, dL_dts=7, dL_dscales=8, dL_dscales_t=9, dL_drot=10,
               dL_drot_r=11, dL_dcolors=1)


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


def _upstream(cfg, aux):
    gc, gd, ga, gf = helpers.pixel_grads(cfg, device=DEV)
    e = torch.empty(0, device=DEV)
    return (gc, gd, ga, gf) if aux else (gc, e, e, e)


def _outputs(bw, fw):
    """what check_backward reads: the returned gradients, the forward's cov3D, and dL_dconic, which the entries do not
    return but which shares one allocation with dL_dmeans2D, dL_dcolors, dL_dflows and dL_dopacity (torch_ext.cpp: the
    blend's zero-filled slab, [P,3 | P,4 | P,3 | P,2 | P,1]); geom_bwd_body leaves in it, as in dL_dmeans2D, the blend
    gradients it converted and consumed"""
    out = {k: bw[i] for k, i in OUT_IDX.items()}
    P = bw[0].shape[0]
    slab = bw[0].untyped_storage()
    assert bw[0].storage_offset() == 0 and bw[1].untyped_storage().data_ptr() == slab.data_ptr() and \
        bw[1].storage_offset() == 7 * P and slab.nbytes() == 13 * P * 4, "the blend gradients' slab layout changed"
    out["dL_dconic"] = torch.empty(0, device=bw[0].device).set_(slab, 3 * P, (P, 4), (4, 1))
    out["dL_dmeans2D"] = bw[0]
    out["cov3D"] = fw[9]
    return out


def _geom(C, fw, P):
    """the forward's clamp bits [P,3] and the rows the backward renders (radius > 0 and at least one tile)"""
    geom = C.debug_export_geom(fw[6], P)
    bits = geom[4].to(torch.int32)
    clamped = torch.stack([(bits >> c) & 1 for c in range(3)], 1).bool()
    return clamped, (fw[5] > 0) & (geom[5] != 0)


@pytest.mark.parametrize("aux", [False, True], ids=["colour", "aux"])
@pytest.mark.parametrize("case", CASES)
def test_per_gaussian_backward_vs_float64(C, case, tile_mode, aux):
    if case == "mid" and (tile_mode == 0 or aux):
        pytest.skip("100k Gaussians: one tile mode and upstream are enough")
    cfg, cam, sc, st, pv = G.build_case(case, device=DEV)
    fw = C.rasterize_gaussians(*helpers.fwd_args(st, sc, cfg))
    bw = C.rasterize_gaussians_backward(*helpers.bwd_args(st, sc, cfg, fw, _upstream(cfg, aux)))
    torch.cuda.synchronize()
    clamped, vis = _geom(C, fw, sc.P)
    out = _outputs(bw, fw)
    worst = G.check_backward("%s %s %s" % (case, ["reflists", "tilecull"][tile_mode], "aux" if aux else "colour"),
                             sc, st, pv, out, clamped, fw[10], vis)
    assert all(v <= 1.0 for v in worst.values()), worst


RAW_CASES = ["tiny", "rotcam", "dur10", "norot4d", "dim3", "deg1m4", "edge:clamp", "edge:scale_t", "edge:p129a",
             "regime:opaque"]


@pytest.mark.parametrize("zero_rows", [False, True], ids=["bwd_zero_rows", "fwd_zero_rows"])
@pytest.mark.parametrize("case", RAW_CASES)
def test_raw_entry_split_rows_vs_float64(C, case, zero_rows):
    """The raw-parameter entry: log-scales, logits (one row in 16 at 20: the sigmoid is exactly 1.0f there, so the
    blend's opacity gradient cannot be recovered from the returned one -- such a row must return dL_dopacity == 0 and its
    chain is not checked), un-normalised quaternions, SH as features_dc | features_rest.  With zero_rows the forward
    writes the SH gradient's non-rendered rows into NaN-filled tensors and the backward only the rendered ones."""
    cfg, cam, sc, st, pv = G.build_case(case, device=DEV)
    g = torch.Generator().manual_seed(cfg["seed"] + 5)
    P = sc.P
    logits = torch.logit(sc.opacities.double()).float()
    logits[torch.arange(P, device=DEV) % 16 == 3] = 20.0
    norm = lambda q: q * (0.5 + 1.5 * torch.rand(q.shape[0], 1, generator=g)).to(DEV)
    raw = dict(rotations=norm(sc.rotations).contiguous(), rotations_r=norm(sc.rotations_r).contiguous())
    rs = dataclasses.replace(sc, scales=torch.log(sc.scales), scales_t=torch.log(sc.scales_t), opacities=logits,
                             rotations=raw["rotations"], rotations_r=raw["rotations_r"], shs=sc.shs[:, :1].contiguous())
    rest = sc.shs[:, 1:].contiguous()
    e = torch.empty(0, device=DEV)
    M = sc.shs.shape[1]
    extra = ()
    if zero_rows:
        extra = (torch.full((P, 1, 3), float("nan"), device=DEV), torch.full((P, M - 1, 3), float("nan"), device=DEV))
    fw = C.rasterize_gaussians_ext(*helpers.fwd_args(st, rs, cfg), rest, True, e, *extra)
    bw = C.rasterize_gaussians_backward_ext(*helpers.bwd_args(st, rs, cfg, fw, _upstream(cfg, True)), rest, True, e,
                                            False, False, *extra)
    torch.cuda.synchronize()
    clamped, vis = _geom(C, fw, P)
    # the activations exactly as the kernels apply them (test_gpu_raw_entry.test_activations_bit_identical_to_torch)
    act = dataclasses.replace(sc, scales=torch.exp(rs.scales), scales_t=torch.exp(rs.scales_t),
                              opacities=torch.sigmoid(logits),
                              rotations=torch.nn.functional.normalize(raw["rotations"]),
                              rotations_r=torch.nn.functional.normalize(raw["rotations_r"]))
    out = _outputs(bw, fw)
    out["dL_dsh"] = torch.cat([bw[5], bw[13]], 1)
    worst = G.check_backward("raw %s %s" % (case, "fwd zero rows" if zero_rows else "bwd zero rows"), act, st, pv, out,
                             clamped, fw[10], vis, raw=raw)
    assert all(v <= 1.0 for v in worst.values()), worst
