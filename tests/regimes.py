"""Scenes in the regimes trained scenes reach and the semi-transparent synthetic scenes of helpers.CONFIGS never do:
saturated opacities with the 0.99 clamp and whole tiles terminating early, many pairs on the 1/255 cut, huge and
off-screen Gaussians, needles, temporal marginals on the 0.05 cut, and deep semi-transparent stacks.  Every builder is
deterministic and CPU-generated from a seed and returns what helpers.build returns: (cfg, cam, sc, st).

preconditions(name, ...) asserts that a scene actually reaches its regime, from the CPU oracle's forward and the
float64 walk of blend_f64.  TEST INFRASTRUCTURE."""
import math

import numpy as np
import torch

import blend_f64
import helpers
import oracle_py
from fdgs import synth

W0, H0 = 192, 144
F32_CUT = np.float32(0.00392156886)                        # 1/255 in fp32
F32_BELOW = np.nextafter(F32_CUT, np.float32(0.0))


def _cat(a, b):
    kw = {k: torch.cat([getattr(a, k), getattr(b, k)]).contiguous() for k in a.tensors()}
    return synth.Scene(**kw, sh_degree=a.sh_degree, sh_degree_t=a.sh_degree_t, time_duration=a.time_duration,
                       rot_4d=a.rot_4d, gaussian_dim=a.gaussian_dim, force_sh_3d=a.force_sh_3d)


def _finish(name, cfg, cam, sc, bg=(0.0, 0.0, 0.0)):
    cfg = dict(cfg, name=name, P=sc.P, bg=bg)
    st = synth.raster_settings(cam, sc, bg=torch.tensor(bg, dtype=torch.float32))
    return cfg, cam, sc, st


def _px_world(cam, z):
    return (2 * abs(math.tan(cam.FoVx * 0.5)) / cam.image_width) * z


def _zrot(theta):
    """unit quaternion (r, x, y, z) of a rotation by theta about the view axis"""
    return torch.stack([torch.cos(theta / 2), torch.zeros_like(theta), torch.zeros_like(theta), torch.sin(theta / 2)], 1)


def opaque():
    """4D.  A deep tail of nearly opaque Gaussians (10 % exactly 1.0) behind a wall of large opaque ones at z 3-4 that
    covers the left part of the image; the right band shows the tail only."""
    seed = 9101
    cam = synth.make_camera(W0, H0)
    g = torch.Generator().manual_seed(seed)
    tail = synth.make_scene(5700, cam, seed, zmin=6.0, zmax=10.0, opacity_lo=0.95, opacity_hi=1.0)
    one = torch.rand(tail.P, generator=g) < 0.1
    tail.opacities[one] = 1.0
    half = torch.rand(tail.P, generator=g) < 0.5          # half of the tail at its temporal peak
    tail.ts[half] = cam.timestamp
    wall = synth.make_scene(300, cam, seed + 1, zmin=3.0, zmax=4.0, opacity_lo=0.995, opacity_hi=1.0, frustum=1.0)
    tanx = abs(math.tan(cam.FoVx * 0.5))
    z = wall.means3D[:, 2]
    wall.means3D[:, 0] = (-1.1 + 1.0 * torch.rand(wall.P, generator=g)) * tanx * z     # centres on the left 55 %
    sig = _px_world(cam, z)[:, None] * (6.0 + 10.0 * torch.rand(wall.P, 3, generator=g))
    wall.scales = sig.contiguous()
    wall.ts[:] = cam.timestamp                            # dt = 0: the marginal is exactly 1
    wall.scales_t[:] = 1.0
    # in front of both, over the left third: one near-point Gaussian per pixel centre (the 0.3 px^2 low-pass alone: G at
    # the next pixel is exp(-1/0.6) ~ 0.19), opacities U(0.99, 1.0), so nearly every pixel there blends its own one clamped
    W1 = W0 // 3
    ys, xs = torch.meshgrid(torch.arange(H0, dtype=torch.float64), torch.arange(W1, dtype=torch.float64), indexing="ij")
    n = W1 * H0
    pts = synth.make_scene(n, cam, seed + 2, zmin=2.0, zmax=2.5, opacity_lo=0.99, opacity_hi=1.0)
    pz = pts.means3D[:, 2].double()
    P00 = float(cam.full_proj_transform[0, 0])
    P11 = float(cam.full_proj_transform[1, 1])
    pts.means3D[:, 0] = (((2 * xs.reshape(-1) + 1) / W0 - 1.0) * (pz + 1e-7) / P00).float()
    pts.means3D[:, 1] = (((2 * ys.reshape(-1) + 1) / H0 - 1.0) * (pz + 1e-7) / P11).float()
    pts.opacities[torch.rand(n, generator=g) < 0.1] = 1.0
    pts.scales = (_px_world(cam, pts.means3D[:, 2])[:, None] * 1e-3).expand(n, 3).contiguous()
    pts.scales_t[:] = 1.0
    pts.ts[:] = cam.timestamp
    ident = torch.tensor([1.0, 0.0, 0.0, 0.0]).expand(n, 4).contiguous()
    pts.rotations, pts.rotations_r = ident.clone(), ident.clone()     # no mixing of time into space
    return _finish("opaque", dict(W=W0, H=H0, seed=seed), cam, _cat(_cat(tail, wall), pts), bg=(0.25, 0.5, 0.75))


def threshold():
    """3D.  Opacities on the 1/255 cut: exactly fp32(1/255), its fp32 predecessor, and 1/255 (1 + U(0, 0.05)); the
    first two classes centred exactly on pixel centres (power = 0, G = 1)."""
    seed = 9102
    cam = synth.make_camera(W0, H0)
    n_centred, n_rest = 2400, 1500
    sc = synth.make_scene(n_centred + n_rest, cam, seed, gaussian_dim=3, rot_4d=False, zmin=3.0, zmax=9.0)
    g = torch.Generator().manual_seed(seed + 7)
    P = sc.P
    cls = torch.where(torch.arange(P) < n_centred, torch.arange(P) % 2, torch.full((P,), 2))
    op = torch.where(cls == 0, torch.tensor(float(F32_CUT)), torch.tensor(float(F32_BELOW)))
    op = torch.where(cls == 2, (1.0 / 255.0) * (1.0 + 0.05 * torch.rand(P, generator=g)), op)
    sc.opacities = op[:, None].float().contiguous()
    # centred ones: classes 0 and 1 of the first n_centred; solve the pixel centre in float64, then nudge by ulps
    idx = torch.nonzero(cls < 2).squeeze(1)
    z = sc.means3D[idx, 2].double()
    kx = torch.randint(2, W0 - 2, (idx.numel(),), generator=g).double()
    ky = torch.randint(2, H0 - 2, (idx.numel(),), generator=g).double()
    P00 = float(cam.full_proj_transform[0, 0])
    P11 = float(cam.full_proj_transform[1, 1])
    x = ((2 * kx + 1) / W0 - 1.0) * (z + 1e-7) / P00
    y = ((2 * ky + 1) / H0 - 1.0) * (z + 1e-7) / P11
    sc.means3D[idx, 0] = x.float()
    sc.means3D[idx, 1] = y.float()
    cfg, cam, sc, st = _finish("threshold", dict(W=W0, H=H0, seed=seed), cam, sc)
    # keep, among the centred ones, only those whose fp32 means2D are integers (ulp nudges give each a few chances)
    for step in range(12):
        f = oracle_py.forward(helpers.oracle_inputs(st, sc, cfg), stages=("preprocess",))
        m = f["means2D"][idx.numpy()]
        bad_x = m[:, 0] != np.round(m[:, 0])
        bad_y = m[:, 1] != np.round(m[:, 1])
        if not (bad_x.any() or bad_y.any()) or step == 11:
            break
        for col, bad, want in ((0, bad_x, kx), (1, bad_y, ky)):
            cur = sc.means3D[idx, col].numpy().copy()
            direction = np.sign(want.numpy() - m[:, col]).astype(np.float32)
            cur[bad] = np.nextafter(cur[bad], cur[bad] + direction[bad] * np.float32(1.0))
            sc.means3D[idx, col] = torch.from_numpy(cur)
    miss = torch.from_numpy(bad_x | bad_y)
    keep = torch.ones(P, dtype=torch.bool)
    keep[idx[miss]] = False
    sc = synth.Scene(**{k: v[keep].contiguous() for k, v in sc.tensors().items()}, sh_degree=sc.sh_degree,
                     sh_degree_t=sc.sh_degree_t, rot_4d=False, gaussian_dim=3)
    return _finish("threshold", dict(W=W0, H=H0, seed=seed), cam, sc)


def huge():
    """4D.  Screen sigma 30-400 px, some centres up to two image widths off-screen, ~100 at view z in (0.2, 0.3], over
    a normal background population."""
    seed = 9103
    cam = synth.make_camera(W0, H0)
    g = torch.Generator().manual_seed(seed)
    base = synth.make_scene(1500, cam, seed)
    big = synth.make_scene(450, cam, seed + 1, zmin=2.0, zmax=8.0, opacity_lo=0.2, opacity_hi=0.7)
    tanx, tany = abs(math.tan(cam.FoVx * 0.5)), abs(math.tan(cam.FoVy * 0.5))
    near = torch.arange(big.P) < 100
    z = big.means3D[:, 2].clone()
    z[near] = 0.2 + 0.1 * (1.0 - torch.rand(int(near.sum()), generator=g))          # (0.2, 0.3]
    reach = 1.0 + 4.0 * torch.rand(big.P, generator=g) ** 2  # |x| up to 5 tan: up to two image widths off-screen
    big.means3D[:, 0] = (2 * torch.rand(big.P, generator=g) - 1) * reach * tanx * z
    big.means3D[:, 1] = (2 * torch.rand(big.P, generator=g) - 1) * 1.2 * tany * z
    big.means3D[:, 2] = z
    sig_px = torch.exp(math.log(30.0) + math.log(400.0 / 30.0) * torch.rand(big.P, 3, generator=g))
    big.scales = (_px_world(cam, z)[:, None] * sig_px).contiguous()
    big.ts[:] = cam.timestamp           # dt = 0 and a short time axis: the 4D rotation barely mixes time into space
    big.scales_t[:] = 0.01
    return _finish("huge", dict(W=W0, H=H0, seed=seed), cam, _cat(base, big), bg=(0.1, 0.1, 0.1))


def needle():
    """4D (3D rotation, temporal marginal).  Projected major sigma 30-300 px, the minor axes at the 0.3 px^2 low-pass,
    rotated 20-70 degrees off the image axes."""
    seed = 9104
    cam = synth.make_camera(W0, H0)
    g = torch.Generator().manual_seed(seed)
    base = synth.make_scene(1000, cam, seed, rot_4d=False)
    nd = synth.make_scene(200, cam, seed + 1, rot_4d=False, zmin=3.0, zmax=8.0, opacity_lo=0.5, opacity_hi=1.0,
                          frustum=0.9)
    z = nd.means3D[:, 2]
    maj = torch.exp(math.log(30.0) + math.log(10.0) * torch.rand(nd.P, generator=g))
    s = torch.empty(nd.P, 3)
    s[:, 0] = _px_world(cam, z) * maj
    s[:, 1] = _px_world(cam, z) * 1e-3
    s[:, 2] = _px_world(cam, z) * 1e-3
    nd.scales = s.contiguous()
    deg = 20.0 + 50.0 * torch.rand(nd.P, generator=g)
    deg = torch.where(torch.rand(nd.P, generator=g) < 0.5, deg, deg + 90.0)
    nd.rotations = _zrot(torch.deg2rad(deg)).contiguous()
    nd.ts[:] = cam.timestamp
    nd.scales_t[:] = 0.5
    return _finish("needle", dict(W=W0, H=H0, seed=seed), cam, _cat(base, nd), bg=(0.0, 0.2, 0.0))


def time_edge():
    """4D.  Timestamps solved in float64 so that the temporal marginal lies within about 1e-6 of the 0.05 cut, some
    Gaussians with dt = 0 exactly, scales_t from 1e-3 to 10."""
    from gaussian_renderer import pyprep
    seed = 9105
    cam = synth.make_camera(W0, H0)
    g = torch.Generator().manual_seed(seed)
    sc = synth.make_scene(3000, cam, seed, time_duration=1.0)
    P = sc.P
    sc.scales_t = torch.exp(math.log(1e-3) + math.log(1e4) * torch.rand(P, 1, generator=g)).contiguous()
    sc.opacities[:] = 1.0                   # the effective opacity the oracle exports is then the fp32 marginal itself
    sxyzt = torch.cat([sc.scales, sc.scales_t], 1).double()
    cov_t = pyprep.covariance_4d(sxyzt, 1.0, sc.rotations.double(), sc.rotations_r.double())[:, 3, 3]
    eps = 2e-6 * (torch.rand(P, generator=g).double() - 0.5)               # target marginal 0.05 (1 + eps)
    dt = torch.sqrt(-2.0 * torch.log(torch.tensor(0.05, dtype=torch.float64) * (1 + eps)) * cov_t)
    sign = torch.where(torch.rand(P, generator=g) < 0.5, -1.0, 1.0).double()
    ts = cam.timestamp - sign * dt
    zero = torch.arange(P) % 10 == 0
    ts[zero] = cam.timestamp
    sc.ts = ts.float()[:, None].contiguous()
    return _finish("time_edge", dict(W=W0, H=H0, seed=seed), cam, sc)


def deep():
    """3D.  ~20k faint Gaussians (opacity 0.005-0.03, sigma 3-6 px): long lists, no pixel terminates."""
    seed = 9106
    cam = synth.make_camera(128, 96)
    g = torch.Generator().manual_seed(seed)
    sc = synth.make_scene(20000, cam, seed, gaussian_dim=3, rot_4d=False, opacity_lo=0.005, opacity_hi=0.03,
                          frustum=1.0)
    z = sc.means3D[:, 2]
    sc.scales = (_px_world(cam, z)[:, None] * (3.0 + 3.0 * torch.rand(sc.P, 3, generator=g))).contiguous()
    return _finish("deep", dict(W=128, H=96, seed=seed), cam, sc, bg=(0.5, 0.5, 0.5))


SCENES = {"opaque": opaque, "threshold": threshold, "huge": huge, "needle": needle, "time_edge": time_edge, "deep": deep}
_cache = {}


def build(name, device="cpu"):
    if name not in _cache:
        _cache[name] = SCENES[name]()
    cfg, cam, sc, st = _cache[name]
    if device == "cpu":
        return cfg, cam, sc, st
    return cfg, cam, sc.to(device), synth.raster_settings(cam, sc, bg=torch.tensor(cfg["bg"]), device=device)


# ---- the 3D twin: the same Gaussians through the precomputed colour / covariance path ---------------------------------
def twin(cfg, sc, st, f):
    """The visible Gaussians of a scene as a 3D scene with precomputed colours and covariances: means3D = out_means3D,
    cov3D_precomp = the forward's cov3D, colors_precomp = its rgb, opacity = the effective opacity.  f: the oracle
    forward of the scene.  Returns (rows of the original, settings, dict of float32 arrays)."""
    rows = np.nonzero(f["radii"] > 0)[0]
    flows = helpers.to_np(sc.flow_2d)[rows]
    t = dict(means3D=f["out_means3D"][rows], cov3D=f["cov3D"][rows], colors=f["rgb"][rows],
             opacity=f["conic_opacity"][rows, 3].copy(), flows=flows)
    t = {k: np.ascontiguousarray(v, np.float32) for k, v in t.items()}
    st3 = dict(st)
    st3.update(rot_4d=False, gaussian_dim=3, sh_degree=0, sh_degree_t=0)
    return rows, st3, t


def twin_oracle_inputs(st3, t):
    return oracle_py.OracleInputs(st3, t["means3D"], t["opacity"][:, None], colors_precomp=t["colors"],
                                  flow_2d=t["flows"], cov3D_precomp=t["cov3D"])


def twin_args(st3, t, device):
    """positional arguments of rasterize_gaussians for the twin (the precomputed path of fwd_args)"""
    e = torch.Tensor([]).to(device)
    d = lambda k: torch.from_numpy(t[k]).to(device)
    return (st3["bg"].to(device), d("means3D"), d("colors"), d("flows"), d("opacity")[:, None].contiguous(), e, e, e, e,
            e, 1.0, d("cov3D"), -1.0, st3["viewmatrix"].to(device), st3["projmatrix"].to(device), st3["tanfovx"],
            st3["tanfovy"], st3["image_height"], st3["image_width"], e, 0, 0, st3["campos"].to(device),
            st3["timestamp"], st3["time_duration"], False, 3, False, False, False)


def twin_bwd_args(st3, t, device, fw, grads):
    e = torch.Tensor([]).to(device)
    d = lambda k: torch.from_numpy(t[k]).to(device)
    (num_rendered, color, flow, depth, T, radii, geom, binning, img, covs, out_means3D) = fw
    return (st3["bg"].to(device), d("means3D"), out_means3D, radii, d("colors"), d("flows"),
            d("opacity")[:, None].contiguous(), e, e, e, e, e, 1.0, d("cov3D"), -1.0, st3["viewmatrix"].to(device),
            st3["projmatrix"].to(device), st3["tanfovx"], st3["tanfovy"], *grads, e, 0, 0, st3["campos"].to(device),
            st3["timestamp"], st3["time_duration"], False, 3, False, geom, num_rendered, binning, img, False)


def f64_lists(f):
    return dict(ranges=f["ranges"], point_list=f["point_list"])


# ---- preconditions ----------------------------------------------------------------------------------------------------
def walk_records(cfg, st, f):
    """float64 walk over the oracle's (reference) lists with the oracle's fp32 means2D / conic / opacity"""
    pix = torch.from_numpy(f["means2D"]).double()
    con = torch.from_numpy(f["conic_opacity"][:, :3]).double()
    op = torch.from_numpy(f["conic_opacity"][:, 3]).double()
    W, H = cfg["W"], cfg["H"]
    ranges = f["ranges"].reshape(-1, 2).astype(np.int64)
    pl = torch.from_numpy(f["point_list"].astype(np.int64))
    gx = (W + 15) // 16
    out = {}
    with torch.no_grad():
        for t in range(ranges.shape[0]):
            lo, hi = ranges[t]
            if hi > lo:
                _, _, pid, rec = blend_f64.walk_tile(pix, con, op, pl[lo:hi], (t % gx) * 16, (t // gx) * 16, W, H)
                out[t] = (pid.numpy(), pl[lo:hi].numpy(), rec)
    return out


def preconditions(name, cfg, sc, st, f):
    """Asserts that the scene reaches its regime; returns the measured quantities (printed by the tests)."""
    W, H = cfg["W"], cfg["H"]
    recs = walk_records(cfg, st, f)
    stats = {}
    if name == "opaque":
        clamp = np.zeros(W * H, bool)
        term = np.zeros(W * H, bool)
        full_tiles = 0
        ranges = f["ranges"].reshape(-1, 2).astype(np.int64)
        nc = f["n_contrib"].reshape(-1).astype(np.int64)
        for t, (pid, ids, rec) in recs.items():
            clamp[pid] = rec["clamp_hit"]
            term[pid] = rec["terminated"]
            length = ranges[t, 1] - ranges[t, 0]
            if rec["terminated"].all() and len(pid) == 256 and length - nc[pid].max() >= 256:
                full_tiles += 1
        stats = dict(clamped=clamp.mean(), terminated=term.mean(), full_tiles=full_tiles,
                     eff_opacity_gt_099=int((f["conic_opacity"][f["radii"] > 0, 3] > 0.99).sum()))
        assert stats["clamped"] >= 0.25 and stats["eff_opacity_gt_099"] >= 1000, stats
        assert 0.30 <= stats["terminated"] <= 0.90 and full_tiles >= 8, stats
    elif name == "threshold":
        above = below = 0
        for pid, ids, rec in recs.values():
            a = rec["alpha"][rec["walked"]]
            near = np.abs(a - blend_f64.CUT) <= 1e-5 * blend_f64.CUT
            above += int((near & (a >= blend_f64.CUT)).sum())
            below += int((near & (a < blend_f64.CUT)).sum())
        stats = dict(above=above, below=below)
        assert above >= 500 and below >= 500, stats
    elif name in ("huge", "needle"):
        contrib = np.zeros(sc.P, bool)
        far = np.zeros(sc.P, bool)
        m2 = f["means2D"].astype(np.float64)
        for pid, ids, rec in recs.values():
            hit = rec["incl"]                                      # [pixels, list]
            contrib[ids[hit.any(0)]] = True
            py, px = np.divmod(pid, W)
            d = np.hypot(m2[ids, 0][None, :] - px[:, None], m2[ids, 1][None, :] - py[:, None])
            far[ids[(hit & (d > 20.0)).any(0)]] = True
        con = f["conic_opacity"].astype(np.float64)
        if name == "huge":
            x0 = np.clip(((m2[:, 0] - f["radii"]) / 16).astype(np.int64), 0, (W + 15) // 16)
            x1 = np.clip(((m2[:, 0] + f["radii"] + 15) / 16).astype(np.int64), 0, (W + 15) // 16)
            y0 = np.clip(((m2[:, 1] - f["radii"]) / 16).astype(np.int64), 0, (H + 15) // 16)
            y1 = np.clip(((m2[:, 1] + f["radii"] + 15) / 16).astype(np.int64), 0, (H + 15) // 16)
            rect = (x1 - x0) * (y1 - y0)
            off = (m2[:, 0] < 0) | (m2[:, 0] >= W) | (m2[:, 1] < 0) | (m2[:, 1] >= H)
            pv = helpers.to_np(sc.means3D).astype(np.float64)       # camera at the origin, identity view
            tanx = abs(float(st["tanfovx"]))
            fcl = np.abs(f["out_means3D"][:, 0] / f["out_means3D"][:, 2]) > 1.3 * tanx
            stats = dict(rect_gt_32=int(((rect > 32) & contrib).sum()), offscreen_rendered=int((off & contrib).sum()),
                         frustum_clamp=int((fcl & contrib).sum()),
                         near=int(((pv[:, 2] > 0.2) & (pv[:, 2] <= 0.3) & contrib).sum()))
            assert stats["rect_gt_32"] >= 20 and stats["offscreen_rendered"] >= 20 and stats["frustum_clamp"] >= 10, stats
            assert stats["near"] >= 50, stats
        else:
            thin = (con[:, 0] * con[:, 2] - con[:, 1] ** 2) < 2e-3 * con[:, 0] * con[:, 2]
            stats = dict(thin_far=int((thin & contrib & far).sum()))
            assert stats["thin_far"] >= 50, stats
    elif name == "time_edge":
        from gaussian_renderer import pyprep
        vis = f["radii"] > 0
        m32 = f["conic_opacity"][:, 3].astype(np.float64)          # opacity 1: the fp32 marginal of a rendered one
        sxyzt = torch.cat([sc.scales, sc.scales_t], 1).double()
        m64 = pyprep.marginal_t(sxyzt, 1.0, sc.rotations.double(), sc.rotations_r.double(), sc.ts.double(),
                                float(np.float32(st["timestamp"])))[:, 0].numpy()
        near_above = vis & (np.abs(m32 / 0.05 - 1) <= 1e-6)
        # culled ones: the fp32 value is not exported; float64 of the same fp32 inputs stands in for it.  Only rows the
        # marginal alone culls count: they render once dt shrinks by 1 % (the marginal then lies ~2 % above the cut)
        ts = sc.ts.clone()
        tsf = float(np.float32(st["timestamp"]))
        ts2 = (tsf - 0.99 * (tsf - ts.double())).float()
        sc2 = synth.Scene(**dict(sc.tensors(), ts=ts2), sh_degree=sc.sh_degree, sh_degree_t=sc.sh_degree_t,
                          time_duration=sc.time_duration, rot_4d=sc.rot_4d, gaussian_dim=sc.gaussian_dim,
                          force_sh_3d=sc.force_sh_3d)
        vis2 = oracle_py.forward(helpers.oracle_inputs(st, sc2, cfg), stages=("preprocess",))["radii"] > 0
        near_below = ~vis & vis2 & (np.abs(m64 / 0.05 - 1) <= 1e-6) & (m64 <= 0.05 * (1 + 1e-7))
        stats = dict(above=int(near_above.sum()), below=int(near_below.sum()),
                     dt_zero=int((helpers.to_np(sc.ts)[:, 0] == np.float32(st["timestamp"])).sum()))
        assert stats["above"] >= 50 and stats["below"] >= 50, stats
    elif name == "deep":
        nc = f["n_contrib"].reshape(-1)
        best = 0
        for t, (pid, ids, rec) in recs.items():
            if not rec["terminated"].any():
                best = max(best, int(nc[pid].max()))
        stats = dict(max_n_contrib_unterminated_tile=best)
        assert best >= 3 * 128, stats
    return stats
