"""CPU: the float64 restatement of the camera gradient's per-row terms (camera_chain_f64.py) against float64 autograd,
and its error bound calibrated on the CPU oracle (oracle_camera_terms).

  - values: on the 3D twins of tiny, small and rotcam without frustum-clamped rows, the restated terms summed over the
    rows equal camera_f64's autograd dL/dviewmatrix and dL/dprojmatrix, fed the same float64 blend gradients; the
    campos terms equal autograd of the SH colour w.r.t. the camera position, in 3D and in 4D with D_t = 2;
  - per row: on every gauss_f64.CASES scene and the one-Gaussian scenes (beyond the frustum clamp, at the near plane,
    negative FoV, 4D SH with campos != 0) every term the oracle computes in fp32 lies within K (e + alt) + tiny of the
    restatement (alt: the other frustum-clamp branch on the rows near it), and it writes nothing to the unused entries;
  - reduction: the oracle's terms summed in float32 in the kernels' order lie within the entry bound;
  - teeth: seven deliberately wrong variants of the terms, rounded to fp32, are each rejected on some scene."""
import functools
import math
import types

import numpy as np
import pytest
import torch

import blend_f64 as BF
import camera_chain_f64 as CC
import camera_f64 as CF
import gauss_f64 as G
import helpers
import oracle_py
from gaussian_renderer import pyprep
from test_camera_grad_f64 import _twin


# ---- values against float64 autograd ----------------------------------------------------------------------------------
def _blend_grads(st3, lists, t, grads):
    """the float64 blend's gradients in the form computeCov2DCUDA consumes: dL_dmeans2D (per NDC unit, and the depth
    gradient) and dL_dconic [P,4] with the reference's halved off-diagonal entry"""
    f = lambda k: torch.as_tensor(np.asarray(t[k], np.float32)).to(torch.float64).requires_grad_(True)
    r = BF.render(st3, lists, f("means3D"), f("cov3D"), f("colors"), f("opacity").reshape(-1), f("flows"))
    for k in ("ndc", "depth", "conic"):
        r[k].retain_grad()
    L = sum((r["images"][k] * torch.as_tensor(np.asarray(g, np.float32)).double()).sum()
            for g, k in zip(grads, ("color", "depth", "alpha", "flow")) if g is not None)
    L.backward()
    c = r["conic"].grad
    dconic = torch.stack([c[:, 0], 0.5 * c[:, 1], torch.zeros_like(c[:, 0]), c[:, 2]], 1)
    return torch.cat([r["ndc"].grad, r["depth"].grad[:, None]], 1), dconic


@pytest.mark.parametrize("name", ["tiny", "small", "rotcam"])
def test_sums_match_autograd_of_the_3d_twin(name):
    st3, lists, t, grads = _twin(name)
    ref = CF.camera_grads(st3, lists, t, grads)
    assert not ref["frustum_clamp"].any()
    dmean2D, dconic = _blend_grads(st3, lists, t, grads)
    P = dmean2D.shape[0]
    out = dict(dL_dmeans2D=dmean2D, dL_dconic=dconic, cov3D=torch.from_numpy(t["cov3D"]))
    r = CC.restate(None, st3, out, None, torch.from_numpy(t["means3D"]), torch.ones(P, dtype=torch.bool), has_sh=False,
                   exact=True)
    assert not bool(r["near"].any())
    v = r["terms"].v
    want = np.concatenate([ref["view"].reshape(-1), ref["proj"].reshape(-1), np.zeros(3)])
    # relative to the magnitude of what each entry is computed from: sum |term| + its fp32 bound / U (an entry whose
    # rows all cancel to ~0, e.g. one the camera's symmetry makes exactly 0, is then judged by its operands' size)
    scale = (v.abs() + r["terms"].e / G.U).sum(0).numpy()
    err = np.abs(v.sum(0).numpy() - want)
    print("%s: %d rows, worst |sum - autograd| / scale %.2e" % (name, P, (err / np.maximum(scale, 1e-300)).max()))
    assert np.all(err <= 1e-9 * scale), (err, scale)
    assert np.all(v[:, CC.UNUSED].numpy() == 0)


@pytest.mark.parametrize("dim", [3, 4])
def test_campos_terms_match_autograd(dim, monkeypatch):
    """Each row's campos terms against autograd of pyprep.eval_shfs_4d w.r.t. its own copy of the camera position (3D:
    no temporal blocks; 4D: D_t = 2), with the kernel's constants; the SH direction is taken at the given means"""
    for name in ("C0", "C1", "C2", "C3"):
        monkeypatch.setattr(pyprep, name, getattr(G, name))
    g = torch.Generator().manual_seed(17)
    n, dur, timestamp, deg_t = 128, G.f32(2.0), G.f32(0.7), 2 if dim == 4 else 0
    sh = torch.randn(n, 48, 3, generator=g, dtype=torch.float64)
    means = torch.randn(n, 3, generator=g, dtype=torch.float64) + torch.tensor([0.0, 0.0, 4.0], dtype=torch.float64)
    campos = torch.tensor([0.1, -0.2, 0.3]).double()          # fp32 values: the settings hold a float tensor
    cp = campos.expand(n, 3).clone().requires_grad_(True)
    ts = torch.rand(n, 1, generator=g, dtype=torch.float64) * dur
    drgb = torch.randn(n, 3, generator=g, dtype=torch.float64)
    clamped = torch.rand(n, 3, generator=g) < 0.2
    dirs = means - cp
    dirs = dirs / dirs.norm(dim=1, keepdim=True)
    rgb = pyprep.eval_shfs_4d(3, deg_t, sh.transpose(1, 2), dirs, ts - timestamp, dur * math.pi / G.MY_PI)
    (torch.where(clamped, 0.0, drgb) * rgb).sum().backward()
    sc = types.SimpleNamespace(shs=sh, ts=ts, means3D=means, gaussian_dim=dim, force_sh_3d=False, sh_degree=3,
                               sh_degree_t=deg_t, time_duration=dur)
    st = dict(viewmatrix=torch.eye(4), projmatrix=torch.eye(4), campos=campos.float(), timestamp=timestamp,
              image_height=64, image_width=64, tanfovx=0.5, tanfovy=0.5)
    z = lambda k: torch.zeros(n, k, dtype=torch.float64)
    out = dict(dL_dmeans2D=z(3), dL_dconic=z(4), cov3D=z(6) + 0.01, dL_dcolors=drgb)
    r = CC.restate(sc, st, out, clamped, means, torch.ones(n, dtype=torch.bool))
    a = r["terms"].v[:, CC.GROUPS["campos"]]
    err = ((a - cp.grad).abs().max() / cp.grad.abs().max()).item()
    print("campos terms vs autograd (%dD): max rel %.2e" % (dim, err))
    assert err < 1e-12


def test_near_clamp_rows_carry_the_other_branch():
    """A row on the frustum clamp in x (view x/z = 1.3 tan fovx (1 + 1e-6)): the clamp drops the view-space x gradient,
    the other branch keeps it, so the row's alt of dL/dV[12] (= vx) is |vx| of a row just inside the clamp"""
    cfg, cam, sc, st = CC.one_scene("clamp_x")
    lim = float(np.float32(1.3) * np.float32(st["tanfovx"]))
    z = 4.0
    means = torch.tensor([[lim * (1 + 1e-6) * z, -0.2, z], [lim * (1 - 1e-6) * z, -0.2, z]], dtype=torch.float64)
    g = torch.Generator().manual_seed(3)
    out = dict(dL_dmeans2D=torch.randn(2, 3, generator=g, dtype=torch.float64).expand(2, 3).clone(),
               dL_dconic=torch.randn(1, 4, generator=g, dtype=torch.float64).expand(2, 4).clone(),
               cov3D=torch.tensor([[2.0, 0.1, 0.2, 1.5, 0.3, 1.0]], dtype=torch.float64).expand(2, 6).clone())
    r = CC.restate(None, st, out, None, means, torch.ones(2, dtype=torch.bool), has_sh=False)
    assert r["near"].tolist() == [True, True]
    v, alt = r["terms"].v, r["alt"]
    assert v[0, 12] == 0 and v[1, 12] != 0
    assert abs(alt[0, 12] - v[1, 12].abs()) <= 1e-4 * v[1, 12].abs()
    assert abs(alt[1, 12] - v[1, 12].abs()) <= 1e-4 * v[1, 12].abs()
    assert (alt[:, 16:] == 0).all()          # the projection does not see the clamp


# ---- the bound's calibration on the CPU oracle -------------------------------------------------------------------------
SCENES = G.CASES + ["one:" + n for n in CC.ONE_SCENES]


def build(case):
    if case.startswith("one:"):
        return CC.one_scene(case[4:])
    return G.build_case(case)[:4]


@functools.lru_cache(maxsize=None)
def oracle_case(case):
    """(restate's arguments, the oracle's terms [P,27]) of one scene"""
    cfg, cam, sc, st = build(case)
    inp = helpers.oracle_inputs(st, sc, cfg)
    f = oracle_py.forward(inp)
    g = oracle_py.backward(inp, f, *(helpers.to_np(x) for x in helpers.pixel_grads(cfg)))
    terms = oracle_py.camera_terms(inp, f, g)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    out = dict(dL_dmeans2D=t(g["dL_dmeans2D"]), dL_dconic=t(g["dL_dconic"]), dL_dcolors=t(g["dL_dcolors"]),
               cov3D=t(f["cov3D"]))
    vis = t((f["radii"] > 0) & (f["tiles_touched"] != 0))
    args = (sc, st, out, t(f["clamped"]).bool(), t(f["out_means3D"]), vis)
    if case.startswith("one:"):
        CC.one_scene_regime(case[4:], st, sc.means3D, args[4], f["radii"], vis)
    return args, terms


@functools.lru_cache(maxsize=None)
def restated(case, mutation=None):
    return CC.restate(*oracle_case(case)[0], mutation=mutation)


@pytest.mark.parametrize("case", SCENES)
def test_oracle_rows_within_bound(case):
    args, terms = oracle_case(case)
    r = restated(case)
    worst = CC.check_rows("oracle rows " + case, CC.layout(terms), r)
    print("oracle rows %-24s rows %5d (%d near the frustum clamp); worst err/bar: %s"
          % (case, int(args[5].sum()), int(r["near"].sum()), "  ".join("%s %.3f" % kv for kv in worst.items())))


@pytest.mark.parametrize("case", SCENES)
def test_kernel_order_sum_within_entry_bound(case):
    args, terms = oracle_case(case)
    CC.check_sums("oracle sum " + case, CC.layout(CC.kernel_order_sum(terms)), restated(case), rows=int(args[5].sum()))


def test_kernel_order_sum_follows_the_kernels():
    """the model's order on a hand-checkable input: 130 rows -> two blocks, the second holding rows 128 and 129"""
    t = np.zeros((130, CC.TERMS), np.float32)
    t[:, 0] = 1.0
    t[0, 1], t[1, 1] = 1.0, 2.0 ** -24              # within one warp's butterfly: 1 + 2^-24 rounds to 1
    t[0, 2], t[128, 2] = 1.0, 2.0 ** -24            # across blocks, in fp64: survives until the final rounding
    t[0, 3], t[128, 3], t[129, 3] = 1.0, 2.0 ** -24, 2.0 ** -24
    s = CC.kernel_order_sum(t)
    assert s[0] == 130.0 and s[1] == 1.0 and s[2] == 1.0 and s[3] == np.float32(1.0 + 2.0 ** -23)


@pytest.mark.parametrize("mutation", CC.MUTATIONS)
def test_mutations_are_rejected(mutation):
    """each wrong variant, rounded to fp32, fails the per-row check on some scene, and its entry sums (rounded to fp32)
    fail the entry check the GPU test applies on some scene"""
    rejected = {}
    for case in SCENES:
        args, _ = oracle_case(case)
        if mutation == "unshifted_sh" and args[0].gaussian_dim != 4:
            continue
        cand = restated(case, mutation)["terms"].v.float().double()
        for kind, check in (("rows", lambda: CC.check_rows("rows", cand, restated(case))),
                            ("sums", lambda: CC.check_sums("sums", cand.sum(0).float(), restated(case)))):
            if kind in rejected:
                continue
            try:
                check()
            except AssertionError as e:
                rejected[kind] = case
                print("%s: %s rejected on %s: %s" % (mutation, kind, case, str(e)[:120]))
        if len(rejected) == 2:
            return
    pytest.fail("mutation %s passed on every scene: %s" % (mutation, rejected))
