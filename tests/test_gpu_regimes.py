"""GPU (-m gpu): the rasterizer in the regimes of regimes.py (saturated opacity and early termination, the 1/255 cut,
huge / off-screen / near-plane Gaussians, needles, the 0.05 temporal cut, deep stacks), in both tile-list modes and
with both blend-backward instantiations (colour only; all four upstream images), against three checkers:
  A. the compiled, unmodified reference (oracle/_ref): bit-identical forward up to threshold pairs, gradients within
     its own run-to-run spread;
  B. the CPU oracle, with the assertions of test_gpu_parity.test_vs_cpu_oracle;
  C. a float64 restatement of the blend (blend_f64.py) on each scene's 3D twin: ours must be no further from float64
     than twice the reference (or, without it, the oracle)."""
import numpy as np
import pytest
import torch

import blend_f64
import helpers
import oracle_py
import regimes
from fdgs import synth
from test_gpu_parity import check_grad_vs_reference

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SCENES = list(regimes.SCENES)
N_REF = 8
# rows of the 12 gradients that exist for the 3D twin (precomputed colours and covariances) and their float64 names
TWIN_GRADS = {0: "dL_dmeans2D", 1: "dL_dcolors", 2: "dL_dopacity", 3: "dL_dmeans3D", 4: "dL_dcov3D", 6: "dL_dflows"}


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


@pytest.fixture(params=[False, True], ids=["colour", "aux"])
def aux(request):
    return request.param


_oracle_cache = {}


def subset(sc, keep):
    return synth.Scene(**{k: v[keep].contiguous() for k, v in sc.tensors().items()}, sh_degree=sc.sh_degree,
                       sh_degree_t=sc.sh_degree_t, time_duration=sc.time_duration, rot_4d=sc.rot_4d,
                       gaussian_dim=sc.gaussian_dim, force_sh_3d=sc.force_sh_3d)


def scene_and_oracle(name, keep=None):
    """CPU scene (the rows `keep` of it), its oracle forward and the float64 walk records of that forward"""
    key = (name, None if keep is None else keep.numpy().tobytes())
    if key not in _oracle_cache:
        cfg, cam, sc, st = regimes.build(name)
        if keep is not None:
            sc = subset(sc, keep)
            cfg = dict(cfg, P=sc.P)
        f = oracle_py.forward(helpers.oracle_inputs(st, sc, cfg))
        _oracle_cache[key] = (cfg, sc, st, f, regimes.walk_records(cfg, st, f))
    return _oracle_cache[key]


def time_cut_rows(sc, st):
    """rows whose float64 temporal marginal lies within 1e-5 of the 0.05 cut (fp32 roundings may put them either side)"""
    if sc.gaussian_dim != 4 or not sc.rot_4d:
        return np.zeros(sc.P, bool)
    from gaussian_renderer import pyprep
    sxyzt = torch.cat([sc.scales, sc.scales_t], 1).double()
    m = pyprep.marginal_t(sxyzt, 1.0, sc.rotations.double(), sc.rotations_r.double(), sc.ts.double(),
                          float(np.float32(st["timestamp"])))[:, 0].numpy()
    return np.abs(m / 0.05 - 1.0) <= 1e-5


def ill_rows(sc, f):
    """Rendered rows whose fp32 state loses more than 1e-5 relative to cancellation, and the loss factor of each:
    the inversion of the dilated 2D covariance (det = a c - b^2, needles), and, with the 4D rotation, the conditional
    covariance Sigma_xx - Sigma_xt Sigma_tx / Sigma_tt (tiny temporal variances).  Every gradient of the covariance
    chain and dL_dmeans3D (through the EWA Jacobian) of such a row inherits that loss."""
    ill, loss = blend_f64.ill_conditioned(f["conic_opacity"])
    if sc.gaussian_dim == 4 and sc.rot_4d:
        from gaussian_renderer import pyprep
        S = pyprep.covariance_4d(torch.cat([sc.scales, sc.scales_t], 1).double(), 1.0, sc.rotations.double(),
                                 sc.rotations_r.double()).numpy()
        d = np.stack([S[:, j, j] for j in range(3)], 1)
        c = d - np.stack([S[:, j, 3] ** 2 for j in range(3)], 1) / S[:, 3, 3:4]
        with np.errstate(divide="ignore", invalid="ignore"):
            kt = np.where(c > 0, d / c, np.inf).max(1)
        loss = np.maximum(loss, 4 * 2.0 ** -24 * kt / 1e-5)
    vis = f["radii"] > 0
    return vis & (loss > 1.0), np.where(vis, loss, 1.0)


CHAIN = ("dL_dts", "dL_dscales", "dL_dscales_t", "dL_drot", "dL_drot_r", "dL_dcov3D")
FED = CHAIN + ("dL_dmeans3D",)


def ambiguous_pixels(cfg, recs):
    amb = np.zeros(cfg["W"] * cfg["H"], bool)
    for pid, ids, rec in recs.values():
        amb[pid] = rec["ambiguous"]
    return amb


def upstream(cfg, aux, zeros_for_missing):
    gc, gd, ga, gf = helpers.pixel_grads(cfg, device=DEV)
    if aux:
        return gc, gd, ga, gf
    if zeros_for_missing:
        return gc, 0 * gd, 0 * ga, 0 * gf
    e = torch.empty(0, device=DEV)
    return gc, e, e, e


def run(mod, name, aux, zeros_for_missing=False, rows=None):
    cfg, cam, sc, st = regimes.build(name, device=DEV)
    if rows is not None:
        sc = subset(sc, rows.to(DEV))
        cfg = dict(cfg, P=sc.P)
    fw = mod.rasterize_gaussians(*helpers.fwd_args(st, sc, cfg))
    bw = mod.rasterize_gaussians_backward(*helpers.bwd_args(st, sc, cfg, fw, upstream(cfg, aux, zeros_for_missing)))
    torch.cuda.synchronize()
    return cfg, sc, st, fw, bw


def require_ref():
    if not oracle_py.ref_available():
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    return oracle_py.ref_module()


def drop_cut_rows(name, rdiff, sc0, st0, who):
    """Rows on the temporal cut that two fp32 builds decide differently (the marginal's last bits depend on the build;
    libm's exp2f is not ex2.approx): a different radius, or a mean shifted by one and not the other.  Any other
    differing row fails.  Returns the rows to keep (None: all)."""
    cut = time_cut_rows(sc0, st0)
    assert not (rdiff & ~cut).any(), np.nonzero(rdiff & ~cut)[0][:8]
    print("%s: %d rows on the temporal cut decided differently from the %s%s" % (
        name, int(rdiff.sum()), who, "; everything below is compared on the scene without them" if rdiff.any() else ""))
    return torch.from_numpy(~rdiff) if rdiff.any() else None


# ---- A. the compiled reference --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SCENES)
def test_regime_vs_compiled_reference(C, name, tile_mode, aux):
    ref = require_ref()
    np_ = helpers.to_np
    cfg, sc0, st0, f, recs = scene_and_oracle(name)
    cfg, sc, st, fw, bw = run(C, name, aux)
    rfw = run(ref, name, aux, zeros_for_missing=True)[3]
    shift = np.abs(np_(fw[10]) - np_(rfw[10])).max(1) > 1e-6 * np.abs(np_(rfw[10])).max(1)
    keep = drop_cut_rows(name, (np_(fw[5]) != np_(rfw[5])) | shift, sc0, st0, "reference")
    if keep is not None:
        cfg, sc0, st0, f, recs = scene_and_oracle(name, keep)
        cfg, sc, st, fw, bw = run(C, name, aux, rows=keep)
    runs = [run(ref, name, aux, zeros_for_missing=True, rows=keep) for _ in range(N_REF)]
    rfw = runs[0][3]
    assert helpers.bitdiff(np_(fw[5]), np_(rfw[5])) == 0, "radii"
    # per Gaussian: bit-identical.  With the 4D rotation the conditional mean and covariance are fp32 chains the
    # reference's sm_90a build contracts differently from the build the oracle and the golden vectors restate: there
    # they agree to rounding
    both = np_(rfw[5]) > 0
    om, rm, oc, rc = np_(fw[10]), np_(rfw[10]), np_(fw[9]), np_(rfw[9])
    mdiff = (om != rm).any(1) | ((oc != rc).any(1) & both)
    if sc0.rot_4d:
        e_m, e_c = helpers.max_rel(om, rm), helpers.max_rel(oc[both], rc[both])
        print("%s: rows whose out_means3D / cov3D differ from the reference by rounding: %d (max rel %.1e / %.1e)"
              % (name, int(mdiff.sum()), e_m, e_c))
        assert e_m < 1e-6 and e_c < 1e-5
    else:
        assert not mdiff.any()
    # images: where no row differs, an element may differ only at a pixel whose walk has a decision within 1e-5 of its
    # threshold; otherwise the rows' rounding reaches the image (amplified by the rows of ill_rows: on time_edge the
    # depth image moves by ~3e-5 relative)
    images = ((1, "color"), (2, "flow"), (3, "depth"), (4, "T"))
    if mdiff.any():
        for i, key in images:
            e = helpers.l2_rel(np_(fw[i]), np_(rfw[i]))
            print("  image %s vs reference: l2 %.2e (bar 1e-4)" % (key, e))
            assert e < 1e-4, key
    else:
        amb = ambiguous_pixels(cfg, recs)
        n_diff = 0
        for i, key in images:
            a, b = np_(fw[i]), np_(rfw[i])
            d = (a.view(np.int32) != b.view(np.int32)).reshape(a.shape[0], -1).any(0) if a.ndim == 3 else \
                (a.view(np.int32) != b.view(np.int32)).reshape(-1)
            assert not (d & ~amb).any(), (key, "differs from the reference at an unambiguous pixel",
                                          np.nonzero(d & ~amb)[0][:8])
            n_diff += int(d.sum())
        print("%s: image elements differing from the reference, all at threshold pixels: %d" % (name, n_diff))
        assert n_diff <= max(2, cfg["W"] * cfg["H"] // 2000)
    # gradients against the mean and spread of the reference's own 8 runs; the rows of ill_rows separately for the
    # tensors their loss reaches
    ill, _ = ill_rows(sc0, f)
    ill_t = torch.from_numpy(ill).to(DEV)
    go = None
    if ill.any():
        # On those rows the reference's sm_90a state differs from ours by rounding (above) that their loss of precision
        # amplifies, so they also get the CPU oracle -- the other build's arithmetic, bit-identical to ours in state --
        # as one more sample of the reference (helpers.add_other_build); its measured distance is printed with the bar.
        inp = helpers.oracle_inputs(st0, sc0, cfg)
        go = oracle_py.backward(inp, f, *[np_(t) if t.numel() else np.zeros((c, cfg["H"], cfg["W"]), np.float32)
                                          for t, c in zip(upstream(cfg, aux, False), (3, 1, 1, 2))])
    for k, gname in enumerate(helpers.GRAD_NAMES):
        rr = [r[4][k].reshape(r[4][k].shape[0], -1) for r in runs]
        if rr[0].numel() == 0:
            continue
        ours = bw[k].reshape(bw[k].shape[0], -1)
        assert torch.isfinite(ours).all(), gname
        groups = [("", None)]
        if gname in FED and ill.any():
            groups = [("", ~ill_t), (" (ill rows)", ill_t)]
        for label, m in groups:
            z = (lambda x: x) if m is None else (lambda x: x * m[:, None].to(x.dtype))
            s = helpers.ref_summary([z(x) for x in rr])
            if label:
                helpers.add_other_build(s, z(torch.from_numpy(go[helpers.ORACLE_GRAD_KEYS[k]].reshape(ours.shape)).to(DEV)))
                print("%s%s: oracle l2 %.2e from the reference's mean, its runs' spread %.2e;"
                      % (name, label, s["stats"][4], s["stats"][0]), end=" ")
            else:
                print("%s:" % name, end=" ")
            check_grad_vs_reference(gname, z(ours), s)


# ---- B. the CPU oracle ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SCENES)
def test_regime_vs_cpu_oracle(C, name, tile_mode, aux):
    np_ = helpers.to_np
    cfg, sc0, st0, f, recs = scene_and_oracle(name)
    cfg, sc, st, fw, bw = run(C, name, aux)
    keep = drop_cut_rows(name, (np_(fw[5]) != f["radii"]) | (np_(fw[10]) != f["out_means3D"]).any(1), sc0, st0, "oracle")
    if keep is not None:
        cfg, sc0, st0, f, recs = scene_and_oracle(name, keep)
        cfg, sc, st, fw, bw = run(C, name, aux, rows=keep)
    assert helpers.bitdiff(np_(fw[5]), f["radii"]) == 0
    geom = C.debug_export_geom(fw[6], cfg["P"])
    binning = C.debug_export_binning(fw[7], fw[8], fw[0], cfg["W"], cfg["H"])
    if tile_mode == 0:
        assert fw[0] == f["num_rendered"]
        assert helpers.bitdiff(np_(binning[0]), f["point_list"]) == 0
        assert helpers.bitdiff(np_(binning[1]), f["ranges"]) == 0
        nd = helpers.bitdiff(np_(binning[2]), f["n_contrib"])
        print("%s: n_contrib differs from the oracle at %d pixels (bar %d)" % (name, nd, max(2, cfg["W"] * cfg["H"] // 20000)))
        assert nd <= max(2, cfg["W"] * cfg["H"] // 20000)
    else:
        assert fw[0] <= f["num_rendered"]
    vis = f["radii"] > 0
    assert helpers.bitdiff(np_(fw[10]), f["out_means3D"]) == 0
    for ours, key in ((geom[0], "depths"), (geom[1], "means2D"), (geom[3], "rgb"), (fw[9], "cov3D")):
        assert helpers.bitdiff(np_(ours)[vis], f[key][vis]) == 0, key
    co = np_(geom[2])
    assert helpers.bitdiff(co[vis][:, :3], f["conic_opacity"][vis][:, :3]) == 0
    assert helpers.max_rel(co[vis][:, 3], f["conic_opacity"][vis][:, 3]) < 1e-6
    for idx, key in ((1, "color"), (2, "flow"), (3, "depth")):
        e = helpers.max_rel(np_(fw[idx]), f[key])
        print("%s vs oracle image %-5s max %.2e (bar 1e-5)" % (name, key, e))
        assert e < 1e-5, key
    assert helpers.psnr(np_(fw[1]), f["color"]) > 100
    gin = [np_(t) if t.numel() else np.zeros((k, cfg["H"], cfg["W"]), np.float32)
           for t, k in zip(upstream(cfg, aux, False), (3, 1, 1, 2))]
    inp = helpers.oracle_inputs(st0, sc0, cfg)
    g = oracle_py.backward(inp, f, *gin)
    ill, loss = ill_rows(sc0, f)
    # on those rows the oracle is held to the compiled reference's own run-to-run spread (measured here), which their
    # loss of precision amplifies just as it amplifies the differences between builds
    refruns = [run(oracle_py.ref_module(), name, aux, True, rows=keep)[4] for _ in range(N_REF)] \
        if ill.any() and oracle_py.ref_available() else None
    for k, (gname, okey, ours) in enumerate(zip(helpers.GRAD_NAMES, helpers.ORACLE_GRAD_KEYS, bw)):
        r = g[okey]
        if r.size == 0:
            continue
        a = np_(ours).reshape(r.shape)
        # the bars of test_vs_cpu_oracle, except on the rows of ill_rows for the tensors their loss reaches
        bl2, bmx = (3e-4 if gname in CHAIN else 1e-4), 1e-3
        well = ~ill if gname in FED else np.ones(len(a), bool)
        l2, mx = helpers.l2_rel(a[well], r[well]), helpers.max_rel(a[well], r[well])
        print("%s vs oracle %-13s l2 %.2e (bar %.0e) max %.2e (bar %.0e)" % (name, gname, l2, bl2, mx, bmx), end="")
        if gname in FED and ill.any():
            l2i = helpers.l2_rel(a[ill], r[ill])
            if refruns is None:
                print("; %d ill rows l2 %.2e (not checked: no compiled reference to measure their spread)"
                      % (int(ill.sum()), l2i), end="")
            else:
                rs = [np_(x[k]).reshape(r.shape)[ill].astype(np.float64) for x in refruns]
                m = sum(rs) / len(rs)
                spread = max(helpers.l2_rel(x, m) for x in rs)
                print("; %d ill rows l2 %.2e (bar %.1e = max(%.0e, 8 x the reference's spread %.1e))"
                      % (int(ill.sum()), l2i, max(bl2, 8 * spread), bl2, spread), end="")
                assert l2i < max(bl2, 8 * spread), (gname, "ill rows", l2i, spread)
        print()
        assert l2 < bl2, gname
        assert mx < bmx, gname


# ---- C. float64 -----------------------------------------------------------------------------------------------------
def _dist(a, b, keep=None):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if keep is not None:
        a, b = a[..., keep], b[..., keep]
    n = np.sqrt((b * b).sum())
    m = np.abs(b).max() if b.size else 0.0
    l2 = np.sqrt(((a - b) ** 2).sum()) / n if n > 0 else 0.0
    mx = np.abs(a - b).max() / m if m > 0 else 0.0
    return l2, mx


@pytest.mark.parametrize("name", SCENES)
def test_regime_vs_float64(C, name, tile_mode, aux):
    cfg, sc0, st0, f, recs = scene_and_oracle(name)
    rows, st3, t = regimes.twin(cfg, sc0, st0, f)
    inp = regimes.twin_oracle_inputs(st3, t)
    ft = oracle_py.forward(inp)
    gc, gd, ga, gf = (helpers.to_np(x) for x in helpers.pixel_grads(cfg))
    ill, _ = blend_f64.ill_conditioned(ft["conic_opacity"])
    r64 = blend_f64.forward_backward(st3, regimes.f64_lists(ft), t, (gc, gd, ga, gf) if aux else (gc, None, None, None),
                                     ill=ill)
    masked = (r64["ambiguous"] | r64["ill"]).reshape(-1)
    gi = r64["grads_in"]
    H, W = cfg["H"], cfg["W"]
    dev = lambda x: torch.from_numpy(x).to(DEV)
    e = torch.empty(0, device=DEV)
    ours_up = (dev(gi[0]), e, e, e) if not aux else tuple(dev(x) for x in gi)
    full_up = tuple(dev(x) if x is not None else torch.zeros(k, H, W, device=DEV) for x, k in zip(gi, (3, 1, 1, 2)))

    fw = C.rasterize_gaussians(*regimes.twin_args(st3, t, DEV))
    np_ = helpers.to_np
    geom = C.debug_export_geom(fw[6], len(rows))
    assert helpers.bitdiff(np_(geom[1]), f["means2D"][rows]) == 0
    assert helpers.bitdiff(np_(geom[2])[:, :3], f["conic_opacity"][rows, :3]) == 0
    assert helpers.max_rel(np_(geom[2])[:, 3], f["conic_opacity"][rows, 3]) < 1e-6
    bw = C.rasterize_gaussians_backward(*regimes.twin_bwd_args(st3, t, DEV, fw, ours_up))
    torch.cuda.synchronize()
    pix = lambda x: np_(x).reshape(x.shape[0], -1)
    imgs = {"color": pix(fw[1]), "flow": pix(fw[2]), "depth": pix(fw[3]), "alpha": 1.0 - pix(fw[4])}
    want = {k: r64["images"][k].reshape(r64["images"][k].shape[0], -1) for k in ("color", "flow", "depth", "alpha")}
    ok_rows = ~r64["frustum_clamp"]

    if oracle_py.ref_available():
        ref = oracle_py.ref_module()
        others = []
        for _ in range(N_REF):
            rf = ref.rasterize_gaussians(*regimes.twin_args(st3, t, DEV))
            rb = ref.rasterize_gaussians_backward(*regimes.twin_bwd_args(st3, t, DEV, rf, full_up))
            torch.cuda.synchronize()
            others.append(({"color": pix(rf[1]), "flow": pix(rf[2]), "depth": pix(rf[3]), "alpha": 1.0 - pix(rf[4])},
                           {k: np_(rb[i]) for i, k in TWIN_GRADS.items()}))
        who = "reference"
    else:
        go = oracle_py.backward(inp, ft, *[np_(x) for x in full_up])
        others = [({"color": ft["color"].reshape(3, -1), "flow": ft["flow"].reshape(2, -1),
                    "depth": ft["depth"].reshape(1, -1), "alpha": ft["alpha"].reshape(1, -1)},
                   {k: go[k] for k in TWIN_GRADS.values()})]
        who = "oracle"
    print("%s (%s, %s): %d of %d pixels ambiguous, %d where an ill-conditioned conic blends, %d rows under the frustum "
          "clamp" % (name, ["reflists", "tilecull"][tile_mode], "aux" if aux else "colour", int(r64["ambiguous"].sum()),
                     masked.size, int(r64["ill"].sum()), int((~ok_rows).sum())))
    illp = (r64["ill"] & ~r64["ambiguous"]).reshape(-1)
    for k in want:
        for label, sel in (("", ~masked), (" ill px", illp)):
            if not sel.any():
                continue
            l2, mx = _dist(imgs[k], want[k], sel)
            dl = [_dist(o[0][k], want[k], sel) for o in others]
            bl2, bmx = max(1e-6, 2 * max(d[0] for d in dl)), max(1e-5, 2 * max(d[1] for d in dl))
            print("  image %-12s l2 %.2e (bar %.2e)  max %.2e (bar %.2e)   [%s l2 %.2e]" % (
                k + label, l2, bl2, mx, bmx, who, max(d[0] for d in dl)))
            assert l2 <= bl2 and mx <= bmx, (k + label, l2, bl2, mx, bmx)
    for i, k in TWIN_GRADS.items():
        a = np_(bw[i]).reshape(r64["grads"][k].shape)[ok_rows]
        w = r64["grads"][k][ok_rows]
        if not np.abs(w).max() > 0:
            assert np.abs(a).max() == 0, k
            continue
        l2, mx = _dist(a.T, w.T)
        dl = [_dist(o[1][k].reshape(-1, w.shape[1])[ok_rows].T, w.T) for o in others]
        bl2, bmx = max(1e-5, 2 * max(d[0] for d in dl)), max(1e-4, 2 * max(d[1] for d in dl))
        print("  grad  %-12s l2 %.2e (bar %.2e)  max %.2e (bar %.2e)   [%s l2 %.2e]" % (k, l2, bl2, mx, bmx, who,
                                                                                    max(d[0] for d in dl)))
        assert l2 <= bl2 and mx <= bmx, (k, l2, bl2, mx, bmx)


# ---- the raw-parameter entry with saturated logits ------------------------------------------------------------------
def test_opaque_raw_entry_with_saturated_logits():
    """Logits in [3, 20]: the sigmoid saturates to exactly 1.0f from about 17 on.  The fused raw entry against the getter
    path (torch sigmoid + autograd through it), at the bars of test_gpu_raw_entry."""
    from gaussian_renderer import render
    from raw_model import RawModel, Pipe, PipeUnfused
    cfg, cam, sc, st = regimes.build("opaque", device=DEV)
    cam = cam.to(DEV)
    g = torch.Generator().manual_seed(31)
    logits = (3.0 + 17.0 * torch.rand(sc.P, 1, generator=g)).to(DEV)
    assert int((torch.sigmoid(logits) == 1.0).sum()) >= 100
    gc = helpers.pixel_grads(cfg, device=DEV)[0]
    models = []
    for pipe in (PipeUnfused(), Pipe()):
        m = RawModel(sc, seed=1, requires_grad=True)
        with torch.no_grad():
            m._opacity.copy_(logits)
        pkg = render(cam, m, pipe, torch.tensor(cfg["bg"], device=DEV))
        (pkg["render"] * gc).sum().backward()
        models.append((m, pkg))
    (A, pa), (B, pb) = models
    assert torch.equal(pa["radii"], pb["radii"])
    assert helpers.psnr(helpers.to_np(pb["render"]), helpers.to_np(pa["render"])) > 90.0
    for k, a in A.leaves().items():
        b = B.leaves()[k]
        err = helpers.l2_rel(helpers.to_np(b.grad), helpers.to_np(a.grad))
        print("opaque raw entry %-13s l2 %.2e" % (k, err))
        assert err < 1e-4, (k, err)
