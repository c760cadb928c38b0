"""CPU: the float64 restatement of the per-Gaussian backward (gauss_f64.py) against float64 autograd of the Python
preprocess (gaussian_renderer/pyprep.py) and finite differences, and its error bound calibrated on the CPU oracle: every
element the oracle's backward returns lies within the bound's one slack factor K of the restatement fed the oracle's own
inputs."""
import math

import pytest
import torch

import gauss_f64 as G
import helpers
import oracle_py
from gaussian_renderer import pyprep


def _rows(n, seed):
    g = torch.Generator().manual_seed(seed)
    s = torch.exp(math.log(0.05) + 0.8 * torch.randn(n, 4, generator=g, dtype=torch.float64))
    ql = torch.nn.functional.normalize(torch.randn(n, 4, generator=g, dtype=torch.float64), dim=1)
    qr = torch.nn.functional.normalize(torch.randn(n, 4, generator=g, dtype=torch.float64), dim=1)
    timestamp = G.f32(0.4)
    cov_t = pyprep.covariance_4d(s, 1.0, ql, qr)[:, 3, 3]
    t = timestamp + cov_t.sqrt() * torch.randn(n, generator=g, dtype=torch.float64)   # marginal mostly above the cut
    gcov = torch.randn(n, 6, generator=g, dtype=torch.float64)
    gmean = torch.randn(n, 3, generator=g, dtype=torch.float64)
    dop = torch.randn(n, generator=g, dtype=torch.float64)
    opac = 0.1 + 0.8 * torch.rand(n, generator=g, dtype=torch.float64)
    return s, ql, qr, t, timestamp, gcov, gmean, dop, opac


def _loss(s, ql, qr, t, timestamp, gcov, gmean, dop, opac, prefilter_var):
    """the scalar whose gradient the chain computes: the upstream gradients dotted with the conditional covariance, the
    mean offset and the effective opacity (pyprep normalises the quaternions itself)"""
    cov3, off = pyprep.conditional_covariance_and_offset(s, 1.0, ql, qr, (timestamp - t)[:, None])
    marg = pyprep.marginal_t(s, 1.0, ql, qr, t[:, None], timestamp, prefilter_var)[:, 0]
    return (gcov * cov3).sum() + (gmean * off).sum() + (dop * opac * marg).sum()


def _restated(s, ql, qr, t, timestamp, gcov, gmean, dop, opac, prefilter_var):
    """gradients of _loss from the restatement: w.r.t. the 4 scales, the raw quaternions (through F.normalize) and t"""
    n = s.shape[0]
    E = G.E
    qln = torch.nn.functional.normalize(ql, dim=1)
    qrn = torch.nn.functional.normalize(qr, dim=1)
    marg = pyprep.marginal_t(s, 1.0, qln, qrn, t[:, None], timestamp, prefilter_var)[:, 0]
    r = G.chain_rot4d([E(s[:, i]) for i in range(4)], [E(qln[:, i]) for i in range(4)], [E(qrn[:, i]) for i in range(4)],
                      E(t), E(opac), timestamp, prefilter_var, [E(gcov[:, i]) for i in range(6)],
                      [E(gmean[:, i]) for i in range(3)], E(dop * marg))
    gl = G.normalize_bwd([E(ql[:, i]) for i in range(4)], r["rot"])
    gr = G.normalize_bwd([E(qr[:, i]) for i in range(4)], r["rot_r"])
    v = lambda es: torch.stack([e.v for e in es], 1)
    return v(r["scales"] + [r["scale_t"]]), v(gl), v(gr), r["dt"].v


@pytest.mark.parametrize("prefilter_var", [-1.0, G.f32(0.01)])
def test_chain_matches_autograd(prefilter_var):
    """The covariance / marginal / mean-shift chain (no quirks) against autograd of pyprep, to 1e-12"""
    args = _rows(256, 5)
    s, ql, qr, t = (a.clone().requires_grad_(True) for a in args[:4])
    _loss(s, ql, qr, t, *args[4:], prefilter_var).backward()
    ours = _restated(*args, prefilter_var)
    for name, a, b in zip(("scales", "rot", "rot_r", "t"), ours, (s.grad, ql.grad, qr.grad, t.grad)):
        err = ((a - b).abs().max() / b.abs().max()).item()
        print("chain vs autograd %-6s max rel %.2e" % (name, err))
        assert err < 1e-12, (name, err)


def test_chain_finite_differences():
    """The restatement as the backward of pyprep's forward: torch.autograd.gradcheck (central differences)"""
    PV = G.f32(0.01)
    fixed = _rows(6, 7)

    class Chain(torch.autograd.Function):
        @staticmethod
        def forward(ctx, s, ql, qr, t):
            ctx.save_for_backward(s, ql, qr, t)
            return _loss(s, ql, qr, t, *fixed[4:], PV)

        @staticmethod
        def backward(ctx, go):
            return tuple(go * x for x in _restated(*ctx.saved_tensors, *fixed[4:], PV))

    assert torch.autograd.gradcheck(Chain.apply, tuple(a.clone().requires_grad_(True) for a in fixed[:4]),
                                    eps=1e-7, atol=1e-6, rtol=1e-6)


@pytest.mark.parametrize("deg_t", [1, 2])
def test_sh_matches_autograd(deg_t, monkeypatch):
    """Every dL_dsh coefficient but the quirk's [1] (SURVEY 8(a) quirk 3) against autograd of pyprep.eval_shfs_4d, with
    the kernel's constants: the fp32 basis constants and its pi (a duration scaled by pi / MY_PI)"""
    for name in ("C0", "C1", "C2", "C3"):
        monkeypatch.setattr(pyprep, name, getattr(G, name))
    g = torch.Generator().manual_seed(3)
    n, dur, timestamp = 128, G.f32(2.0), G.f32(0.7)
    sh = torch.randn(n, 48, 3, generator=g, dtype=torch.float64, requires_grad=True)
    means = torch.randn(n, 3, generator=g, dtype=torch.float64) + torch.tensor([0.0, 0.0, 4.0], dtype=torch.float64)
    campos = torch.tensor([0.1, -0.2, 0.3], dtype=torch.float64)
    ts = torch.rand(n, generator=g, dtype=torch.float64) * dur
    drgb = torch.randn(n, 3, generator=g, dtype=torch.float64)
    clamped = torch.rand(n, 3, generator=g) < 0.2
    dirs = means - campos
    dirs = dirs / dirs.norm(dim=1, keepdim=True)
    rgb = pyprep.eval_shfs_4d(3, deg_t, sh.transpose(1, 2), dirs, (ts - timestamp)[:, None], dur * math.pi / G.MY_PI)
    (torch.where(clamped, 0.0, drgb) * rgb).sum().backward()
    dsh, _, _ = G.sh_backward(sh.detach(), drgb, clamped, means, campos, ts, timestamp, dur, 3, deg_t, True)
    keep = torch.ones(48, dtype=torch.bool)
    keep[1] = False
    a, b = dsh.v[:, keep], sh.grad[:, keep]
    err = ((a - b).abs().max() / b.abs().max()).item()
    print("dL_dsh vs autograd (deg_t %d): max rel %.2e" % (deg_t, err))
    assert err < 1e-12
    assert torch.equal(dsh.v[:, 1], G.C0 * torch.where(clamped, 0.0, drgb))     # quirk: l0m0 in place of l1m1


def test_chain_3d_matches_autograd():
    """The 3D / non-rot-4D branch against autograd of a float64 forward of computeCov3D (forward.cu:242-276): Sigma from
    M[c][r] = s_r R(q)[c][r] with the quaternion NOT normalised (SURVEY 8(a) quirk 4)"""
    g = torch.Generator().manual_seed(11)
    n = 256
    s = torch.exp(math.log(0.05) + 0.8 * torch.randn(n, 3, generator=g, dtype=torch.float64)).requires_grad_(True)
    q = (torch.randn(n, 4, generator=g, dtype=torch.float64) * (0.5 + torch.rand(n, 1, generator=g,
                                                                                  dtype=torch.float64))).requires_grad_(True)
    gcov = torch.randn(n, 6, generator=g, dtype=torch.float64)
    r, x, y, z = q.unbind(1)
    R = [[1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)],
         [2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)],
         [2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]]
    M = [[s[:, k] * R[c][k] for k in range(3)] for c in range(3)]
    dot = lambda i, j: sum(M[i][k] * M[j][k] for k in range(3))
    cov = torch.stack([dot(0, 0), dot(1, 0), dot(2, 0), dot(1, 1), dot(2, 1), dot(2, 2)], 1)
    (gcov * cov).sum().backward()
    E = G.E
    ours = G.chain_3d([E(s.detach()[:, i]) for i in range(3)], [E(q.detach()[:, i]) for i in range(4)],
                      [E(gcov[:, i]) for i in range(6)])
    for name, a, b in (("scales", ours["scales"], s.grad), ("rot", ours["rot"], q.grad)):
        a = torch.stack([e.v for e in a], 1)
        err = ((a - b).abs().max() / b.abs().max()).item()
        print("3D chain vs autograd %-6s max rel %.2e" % (name, err))
        assert err < 1e-12, (name, err)


@pytest.mark.parametrize("deg_t", [0, 1, 2])
def test_sh_direction_matches_autograd(deg_t, monkeypatch):
    """The SH part of dL_dmeans3D (the basis derivatives weighted by the temporal weights, through dnormvdv) against
    autograd of pyprep.eval_shfs_4d w.r.t. the means, with the kernel's constants"""
    for name in ("C0", "C1", "C2", "C3"):
        monkeypatch.setattr(pyprep, name, getattr(G, name))
    g = torch.Generator().manual_seed(13)
    n, dur, timestamp = 128, G.f32(2.0), G.f32(0.7)
    sh = torch.randn(n, 48, 3, generator=g, dtype=torch.float64)
    means = (torch.randn(n, 3, generator=g, dtype=torch.float64) +
             torch.tensor([0.0, 0.0, 4.0], dtype=torch.float64)).requires_grad_(True)
    campos = torch.tensor([0.1, -0.2, 0.3], dtype=torch.float64)
    ts = torch.rand(n, generator=g, dtype=torch.float64) * dur
    drgb = torch.randn(n, 3, generator=g, dtype=torch.float64)
    clamped = torch.rand(n, 3, generator=g) < 0.2
    dirs = means - campos
    dirs = dirs / dirs.norm(dim=1, keepdim=True)
    rgb = pyprep.eval_shfs_4d(3, deg_t, sh.transpose(1, 2), dirs, (ts - timestamp)[:, None], dur * math.pi / G.MY_PI)
    (torch.where(clamped, 0.0, drgb) * rgb).sum().backward()
    _, _, dm = G.sh_backward(sh, drgb, clamped, means.detach(), campos, ts, timestamp, dur, 3, deg_t, True)
    a = torch.stack([e.v for e in dm], 1)
    err = ((a - means.grad).abs().max() / means.grad.abs().max()).item()
    print("SH direction gradient vs autograd (deg_t %d): max rel %.2e" % (deg_t, err))
    assert err < 1e-12


# ---- the bound's calibration on the CPU oracle -------------------------------------------------------------------------
def oracle_worst(case):
    cfg, cam, sc, st, pv = G.build_case(case)
    inp = helpers.oracle_inputs(st, sc, cfg)
    f = oracle_py.forward(inp)
    gc, gd, ga, gf = (helpers.to_np(x) for x in helpers.pixel_grads(cfg))
    g = oracle_py.backward(inp, f, gc, gd, ga, gf)
    t = lambda k: torch.from_numpy(g[k])
    out = dict(dL_dsh=t("dL_dsh"), dL_dts=t("dL_dts"), dL_dscales=t("dL_dscales"), dL_dscales_t=t("dL_dscales_t"),
               dL_drot=t("dL_drotations"), dL_drot_r=t("dL_drotations_r"), dL_dopacity=t("dL_dopacity"),
               dL_dcolors=t("dL_dcolors"), dL_dcov3D=t("dL_dcov3D"), dL_dmeans3D=t("dL_dmeans3D"),
               dL_dmeans2D=t("dL_dmeans2D"), dL_dconic=t("dL_dconic"), cov3D=torch.from_numpy(f["cov3D"]))
    return G.check_backward("oracle " + case, sc, st, pv, out, torch.from_numpy(f["clamped"]).bool(),
                            torch.from_numpy(f["out_means3D"]), torch.from_numpy(f["radii"] > 0))


@pytest.mark.parametrize("case", G.CASES)
def test_oracle_within_bound(case):
    """Every element of the oracle's dL_dsh, dL_dmeans3D, dL_dscales(_t), dL_drot(_r) and dL_dts within K err + tiny"""
    worst = oracle_worst(case)
    assert all(v <= 1.0 for v in worst.values()), worst
