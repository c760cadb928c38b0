"""GPU (-m gpu): the blend backward (blend_bwd.cu, with geom_bwd_body's map) row by row against its float64 restatement
(blend_bwd_f64.py), started from the forward's own fp32 screen-space state read back through the debug exports.  Every
element of every rendered row of dL_dmeans2D, dL_dconic, dL_dopacity, dL_dcolors and dL_dflows lies within K err + tiny
of the float64 value (the bound calibrated on the CPU oracle by test_blend_bwd_f64.py); every other row of the blend's
slab is exactly 0.  The reference-layout entry (colour-only and all four upstream images, both tile-list modes, with and
without a per-pixel background image) and the batched entry's per-view dL_dmeans2D.  The scenes at the kernel's own
edges (blend_bwd_f64.edge_scene, and regime:huge / regime:needle) assert their edge on the GPU forward's state."""
import numpy as np
import pytest
import torch

import blend_bwd_f64 as BB
import gauss_f64 as G
import helpers
from test_gpu_batch import _batch, _inputs, _settings
from test_gpu_gauss_f64 import _outputs
from test_gpu_view_parallel import _views

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = G.CASES + ["regime:deep"] + BB.EDGE_SCENES


@pytest.fixture(scope="module")
def C():
    import fdgs
    return fdgs.ext()


def forward_state(C, fw, P, W, H, flows, bg):
    """the forward's screen-space state as blend_bwd_f64 reads it, and the rows it rendered"""
    np_ = helpers.to_np
    depths, means2D, conic, rgb, _, tiles = C.debug_export_geom(fw[6], P)
    pl, ranges, nc = C.debug_export_binning(fw[7], fw[8], fw[0], W, H)
    st = dict(W=W, H=H, means2D=np_(means2D), conic_opacity=np_(conic), rgb=np_(rgb), depths=np_(depths),
              flows=np_(flows), point_list=np_(pl), ranges=np_(ranges), n_contrib=np_(nc), final_T=np_(fw[4]),
              bg=np_(bg))
    return st, np_((fw[5] > 0) & (tiles != 0))


def _upstream(cfg, aux):
    g = [helpers.to_np(x) for x in helpers.pixel_grads(cfg)]
    return g if aux else [g[0], None, None, None]


def _dev(gm):
    e = torch.empty(0, device=DEV)
    return tuple(e if g is None else torch.from_numpy(g).to(DEV) for g in gm)


def _got(out, bw):
    return dict(dL_dmeans2D=helpers.to_np(out["dL_dmeans2D"]), dL_dconic=helpers.to_np(out["dL_dconic"])[:, [0, 1, 3]],
                dL_dopacity=helpers.to_np(bw[2]), dL_dcolors=helpers.to_np(bw[1]), dL_dflows=helpers.to_np(bw[6]))


def _report(label, dec, worst):
    s = dec["stats"]
    frac = s["masked"] / s["pixels"]
    print("%-40s masked %.2e (%d pairs exactly on 1/255 decided); worst err/bar: %s" % (
        label, frac, s["cut_exact_pairs"], "  ".join("%s %.3f" % (k[4:], v) for k, v in worst.items())))
    assert frac < BB.MAX_MASKED, (label, "masked fraction", frac)
    assert s["nan"] == 0, (label, "pixels walking a non-finite record", s["nan"])
    assert all(v <= 1.0 for v in worst.values()), worst


def _run(C, case, aux, bgi, tile_label):
    cfg, cam, sc, st3, pv = BB.build_case(case, device=DEV)
    e = torch.empty(0)
    bg_image = torch.rand(3, cfg["H"], cfg["W"], generator=torch.Generator().manual_seed(cfg["seed"] + 7)).to(DEV) \
        if bgi else None
    fargs = helpers.fwd_args(st3, sc, cfg)
    fw = C.rasterize_gaussians_ext(*fargs, e, False, bg_image) if bgi else C.rasterize_gaussians(*fargs)
    torch.cuda.synchronize()
    st, rendered = forward_state(C, fw, sc.P, cfg["W"], cfg["H"], sc.flow_2d, st3["bg"])
    dec = BB.decide(st)
    BB.edge_reached(case, st, dec)
    gm = BB.mask_grads(_upstream(cfg, aux), dec["mask"])
    bargs = helpers.bwd_args(st3, sc, cfg, fw, _dev(gm))
    bw = C.rasterize_gaussians_backward_ext(*bargs, e, False, bg_image, False, False) if bgi else \
        C.rasterize_gaussians_backward(*bargs)
    torch.cuda.synchronize()
    res = BB.backward(st, dec, gm, st["bg"], None if bg_image is None else helpers.to_np(bg_image))
    m, near = BB.marginal(sc, st3, pv)
    label = "%s %s %s%s" % (case, tile_label, "aux" if aux else "colour",
                            " bg_image" if bgi else "")
    worst = BB.check(label, res, _got(_outputs(bw, fw), bw), rendered, near, m)
    _report(label, dec, worst)


@pytest.mark.parametrize("case", CASES)
def test_blend_backward_vs_float64(C, case):
    """all four upstream images (the AUX instantiation: colour, depth, flow and alpha recurrences)"""
    _run(C, case, True, False, "tilecull")


@pytest.mark.parametrize("case", ["small", "dim3", "edge:p1"] + ["regime:" + k for k in ("needle", "huge", "opaque",
                                                                                        "threshold")] + BB.EDGE_SCENES)
def test_colour_only_vs_float64(C, case):
    """the colour-only instantiation (the reference's default training loss)"""
    _run(C, case, False, False, "tilecull")


@pytest.mark.parametrize("aux", [False, True], ids=["colour", "aux"])
@pytest.mark.parametrize("case", ["small", "regime:threshold", "regime:needle", "blend:tail"])
def test_reference_lists_vs_float64(C, case, aux):
    """the reference's tile lists (no per-tile cull): every instance the binning emits is walked"""
    import fdgs
    prev = fdgs.set_tile_cull(0)
    try:
        _run(C, case, aux, False, "reflists")
    finally:
        fdgs.set_tile_cull(prev)


@pytest.mark.parametrize("aux", [False, True], ids=["colour", "aux"])
@pytest.mark.parametrize("case", ["flowbg", "regime:opaque", "blend:stack"])
def test_background_image_vs_float64(C, case, aux):
    """the extended entry with a per-pixel background image: its colour enters dL/dalpha through T_final"""
    _run(C, case, aux, True, "tilecull")


@pytest.mark.parametrize("aux", [False, True], ids=["colour", "aux"])
@pytest.mark.parametrize("name", ["n3v", "blend:stack"])
def test_batched_means2D_vs_float64(C, name, aux):
    """B = 3 views through the batched entry: each view's dL_dmeans2D [P,3] (W10 / W01 after the map, depth in z)
    against the restatement from that view's forward state (the single-view forward, bit-identical per view:
    test_gpu_batch)"""
    cfg, cam, sc, _, pv = BB.build_case(name, device=DEV)
    cams = _views(cfg, 3, DEV)
    sts = _settings(cams, sc, cfg)
    B, H, W = 3, cfg["H"], cfg["W"]
    gin = _inputs(sc, False, False)
    fb = _batch(sts, sc, cfg, gin, False, None)
    decs, states, gms, rendered = [], [], [], []
    for v in range(B):
        fw = C.rasterize_gaussians(*helpers.fwd_args(sts[v], sc, cfg))
        st, r = forward_state(C, fw, sc.P, W, H, sc.flow_2d, sts[v]["bg"])
        rg_v, nc_v = C.debug_export_binning_view(fb[8], W, H, B, v)
        assert np.array_equal(helpers.to_np(nc_v), st["n_contrib"]), v
        dec = BB.decide(st)
        g = helpers.pixel_grads(dict(cfg, seed=cfg["seed"] + v))
        g = [helpers.to_np(x) for x in g]
        gm = BB.mask_grads(g if aux else [g[0], None, None, None], dec["mask"])
        decs.append(dec), states.append(st), gms.append(gm), rendered.append(r)
    stackv = lambda k, c: torch.from_numpy(np.stack([gm[k] if gm[k] is not None else np.zeros((c, H, W), np.float32)
                                                     for gm in gms])).to(DEV) if (k == 0 or aux) else torch.empty(0, device=DEV)
    up = [stackv(0, 3), stackv(1, 1), stackv(2, 1), stackv(3, 2)]
    R, color, flow, depth, T, radii, geom_b, bin_b, img_b, means_b = fb
    st0 = sts[0]
    f32 = lambda k: torch.tensor([s[k] for s in sts], dtype=torch.float32)
    bw = C.rasterize_gaussians_backward_batch(
        st0["bg"], sc.means3D, means_b, radii, sc.flow_2d, gin["opacity"], gin["ts"], gin["scales"], gin["scales_t"],
        gin["rotations"], gin["rotations_r"], st0["scale_modifier"], pv, torch.stack([s["viewmatrix"] for s in sts]),
        torch.stack([s["projmatrix"] for s in sts]), torch.stack([s["campos"] for s in sts]), f32("timestamp"),
        f32("tanfovx"), f32("tanfovy"), *up, gin["sh"], gin["sh_rest"], st0["sh_degree"], st0["sh_degree_t"],
        st0["time_duration"], st0["rot_4d"], st0["gaussian_dim"], st0["force_sh_3d"], geom_b, R, bin_b, img_b, False,
        False, torch.empty(0, device=DEV), False)
    torch.cuda.synchronize()
    for v in range(B):
        res = BB.backward(states[v], decs[v], gms[v], states[v]["bg"])
        got = dict(dL_dmeans2D=helpers.to_np(bw[0][v]))
        label = "batch %s view %d %s" % (name, v, "aux" if aux else "colour")
        _report(label, decs[v], BB.check(label, res, got, rendered[v]))
