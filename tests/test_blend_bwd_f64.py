"""CPU: the float64 restatement of the blend backward (blend_bwd_f64.py) against float64 autograd of a screen-space walk
(blend_f64.walk_tile), its replica of the forward's decisions against the oracle's n_contrib, and its error bound
calibrated on the CPU oracle's render backward (the reference's per-pair arithmetic): every element of every rendered
row within K err + tiny, every unrendered row exactly 0.  The scenes at the blend backward's own edges are 3D
(blend_bwd_f64.edge_scene), so the GPU test runs the same ones."""
import numpy as np
import pytest
import torch

import blend_bwd_f64 as BB
import blend_f64
import gauss_f64 as G
import helpers
import oracle_py

CASES = G.CASES + ["regime:deep"]
F64 = torch.float64


# ---- the scenes' forward state from the oracle -------------------------------------------------------------------------
def case_state(case):
    """(state, upstream gradients, oracle inputs + forward, marginal E, rows near the marginal's cut) of a case"""
    cfg, cam, sc, s3, pv = BB.build_case(case)
    inp = helpers.oracle_inputs(s3, sc, cfg)
    f = oracle_py.forward(inp)
    st = dict(W=cfg["W"], H=cfg["H"], means2D=f["means2D"], conic_opacity=f["conic_opacity"], rgb=f["rgb"],
              depths=f["depths"], flows=inp.keep["flows"], point_list=f["point_list"], ranges=f["ranges"],
              n_contrib=f["n_contrib"], final_T=f["final_T"], bg=inp.keep["background"])
    grads = [helpers.to_np(x) for x in helpers.pixel_grads(cfg)]
    m, near = BB.marginal(sc, s3, pv)
    return st, grads, (inp, f), m, near


# ---- values: the restatement against float64 autograd ------------------------------------------------------------------
def autograd_values(st, dec, grads, bg, bg_image):
    """float64 autograd of the images through blend_f64.walk_tile on the forward's lists; returns (name -> [P,k] numpy,
    pixels walk_tile finds ambiguous in float64)"""
    W, H = st["W"], st["H"]
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64)).clone().requires_grad_(True)
    pix, conic = t(st["means2D"]), t(np.asarray(st["conic_opacity"])[:, :3])
    op, col, dep, fl = t(np.asarray(st["conic_opacity"])[:, 3]), t(st["rgb"]), t(st["depths"]), t(st["flows"])
    ranges = np.asarray(st["ranges"]).astype(np.int64).reshape(-1, 2)
    plist = torch.from_numpy(np.asarray(st["point_list"]).astype(np.int64))
    gx = (W + 15) // 16
    bgv = torch.from_numpy(np.asarray(bg, np.float64)).reshape(3, 1)
    if bg_image is not None:
        bgv = bgv + torch.from_numpy(np.asarray(bg_image, np.float64)).reshape(3, -1)
    gs = [None if g is None else torch.from_numpy(np.asarray(g, np.float64)).reshape(-1, W * H) for g in grads]
    loss = 0.0
    amb = np.zeros(W * H, bool)
    for ti in range(ranges.shape[0]):
        lo, hi = ranges[ti]
        if hi <= lo:
            continue
        ids = plist[lo:hi]
        w, Tf, pid, rec = blend_f64.walk_tile(pix, conic, op, ids, (ti % gx) * 16, (ti // gx) * 16, W, H)
        amb[pid.numpy()] = rec["ambiguous"]
        bgp = bgv if bg_image is None else bgv[:, pid]
        img = [(w @ col[ids]).t() + Tf[None] * bgp, (w @ dep[ids])[None], (1.0 - Tf)[None], (w @ fl[ids]).t()]
        for g, im in zip(gs, img):
            if g is not None:
                loss = loss + (g[:, pid] * im).sum()
    loss.backward()
    P = pix.shape[0]
    z = lambda x, k: x.grad.reshape(P, k).numpy() if x.grad is not None else np.zeros((P, k))
    m2 = z(pix, 2) * np.array([0.5 * W, 0.5 * H])
    # the reference's dL/dconic.y is per element of the symmetric matrix: half the gradient w.r.t. B of -B dx dy
    dcon = z(conic, 3) * np.array([1.0, 0.5, 1.0])
    out = dict(dL_dmeans2D=np.concatenate([m2, z(dep, 1)], 1), dL_dconic=dcon, dL_dopacity=z(op, 1),
               dL_dcolors=z(col, 3), dL_dflows=z(fl, 2))
    return out, amb.reshape(H, W)


VALUE_CASES = ["flowbg", "ragged", "regime:opaque", "regime:threshold", "regime:needle", "edge:p1"] + BB.EDGE_SCENES


@pytest.mark.parametrize("aux,bgi", [(False, False), (True, True)], ids=["colour-bg", "aux-bg_image"])
@pytest.mark.parametrize("case", VALUE_CASES)
def test_values_match_autograd(case, aux, bgi):
    """The restatement's values (both its per-pair and its moment form) against autograd, to 1e-10 relative per tensor"""
    st, grads, _, _, _ = case_state(case)
    dec = BB.decide(st)
    if not aux:
        grads = [grads[0], None, None, None]
    bg_image = np.random.default_rng(3).uniform(0, 1, (3, st["H"], st["W"])).astype(np.float32) if bgi else None
    # both decide in their own precision: mask the union of their uncertain pixels
    _, amb = autograd_values(st, dec, BB.mask_grads(grads, dec["mask"]), st["bg"], bg_image)
    gm = BB.mask_grads(grads, dec["mask"] | amb)
    want, _ = autograd_values(st, dec, gm, st["bg"], bg_image)
    res = BB.backward(st, dec, gm, st["bg"], bg_image)
    for name in BB.OUTPUTS:
        b = want[name]
        scale = max(np.abs(b).max(), 1e-300)
        for form in (res[name].v.numpy(), res[name + "@kernel"].numpy()):
            err = np.abs(form - b).max() / scale
            assert err < 1e-10, (case, name, err)
    print("%s %s %s: values match autograd (masked %d of %d pixels)" % (case, "aux" if aux else "colour",
                                                                        "bg_image" if bgi else "bg",
                                                                        int((dec["mask"] | amb).sum()), amb.size))


# ---- the bound's calibration on the CPU oracle -------------------------------------------------------------------------
def oracle_check(case):
    st, grads, of, m, near = case_state(case)
    dec = BB.decide(st)
    BB.edge_reached(case, st, dec)
    s = dec["stats"]
    frac = s["masked"] / s["pixels"]
    gm = BB.mask_grads(grads, dec["mask"])
    inp, f = of
    g = oracle_py.backward(inp, f, *gm)
    got = {k: g[k] for k in BB.OUTPUTS}
    rendered = (f["radii"] > 0) & (f["tiles_touched"] != 0)
    got["dL_dconic"] = np.asarray(got["dL_dconic"])[:, [0, 1, 3]]
    res = BB.backward(st, dec, gm, st["bg"])
    worst = BB.check("oracle " + case, res, got, rendered, near, m)
    # the forward's T against its float64 product
    T = res["T_final"]
    live = ~torch.isnan(T.v)
    Tg = torch.from_numpy(np.asarray(st["final_T"], np.float64).reshape(-1))
    tw = float(((Tg - T.v).abs()[live] / (G.K * T.e + G.TINY)[live]).max()) if bool(live.any()) else 0.0
    assert tw <= 1.0, (case, "final_T", tw)
    print("oracle %-20s masked %.2e (%d ambiguous, %d n_contrib mismatches, %d pairs exactly on 1/255 decided); "
          "worst err/bar: %s  final_T %.3f" % (case, frac, s["ambiguous"], s["mismatched"], s["cut_exact_pairs"],
                                               "  ".join("%s %.3f" % (k[4:], v) for k, v in worst.items()), tw))
    return worst, frac, dec, st


@pytest.mark.parametrize("case", CASES + BB.EDGE_SCENES)
def test_oracle_within_bound(case):
    """Every element of the oracle's blend gradients within K err + tiny; the masked fraction small"""
    worst, frac, dec, st = oracle_check(case)
    assert all(v <= 1.0 for v in worst.values()), worst
    assert frac < BB.MAX_MASKED, ("masked fraction", frac)
    assert dec["stats"]["nan"] == 0


@pytest.mark.parametrize("case", ["small", "regime:threshold", "regime:opaque", "regime:deep"] + BB.EDGE_SCENES)
def test_replica_reproduces_n_contrib(case):
    """The replicated fp32 decisions give the oracle's n_contrib at every pixel that is not masked as ambiguous; the
    threshold scene's pairs at exactly fp32(1/255) are decided, not masked"""
    st, _, _, _, _ = case_state(case)
    dec = BB.decide(st)
    assert dec["stats"]["mismatched"] == 0, dec["stats"]
    if case == "regime:threshold":
        assert dec["stats"]["cut_exact_pairs"] > 0
