"""Float64 restatement of the camera gradient's per-row terms (preprocess_bwd.cu: the `if (CAM)` blocks of
geom_bwd_body) with a first-order bound on the error an fp32 evaluation of the same expressions may carry, and the
bound of their sum as geom_bwd_cam_kernel and camera_grad_finish_kernel reduce it.

Per rendered row (radius > 0 and at least one tile), in the layout of the tensors the rasterizer takes (element [c][r]
is the gradient of element [c][r], so dL/dV[4c + r]):
  view  [c][r], c, r < 3   m_c g_r + sum_i J[i][r] dL/dT[i][c]      (t = W m + V[12..14] and T = J W, W[r][c] = V[4c + r])
        [3][r], r < 3      g_r                                      g = (vx, vy, vz), the view-space point's gradient
        [c][3]             0                                        (view-space w feeds nothing)
  proj  [c][r], r = 0,1,3  m_c gp_r, m_3 = 1, gp = (d2x m_w, d2y m_w, -(mul1 d2x + mul2 d2y))
        [c][2]             0                                        (clip z feeds nothing)
  campos[k]                -(the SH direction part of dL/dmean[k])  (the direction is m - campos)
with the reference's clamp semantics (x_grad_mul / y_grad_mul, and the clamped tx, ty inside j02, j12).  All of it comes
from gauss_f64.ewa_chain and gauss_f64.sh_backward, the chain dL_dmeans3D is checked with.

The reduction model of an entry (geom_bwd_cam_kernel, camera_grad_finish_kernel):
  - rows are grouped into blocks of GB_THREADS = 128; each block sums a term in fp32 by a 5-level xor butterfly within
    each warp and then the 4 warp sums in order: every row's term passes through at most 8 roundings;
  - the blocks' partials are summed in fp64 (a lane-strided sum and a butterfly) and rounded to fp32 once.
So |fp32 entry - sum_i t_i| <= sum_i e_i + (8 U + nblocks 2^-53) sum_i |t_i| + U |sum_i t_i|, to first order, where e_i
is row i's bound.  A change to that structure changes REDUCTION_ROUNDINGS.

Rows near the frustum clamp (gauss_f64: within 1e-5 of 1.3 tan fov) may branch differently in fp32 and float64: both
branches are evaluated in float64 and their difference is added to the row's (and the entry's) bound.  No row is dropped.
TEST INFRASTRUCTURE."""
import numpy as np
import torch

import gauss_f64 as G
from gauss_f64 import E, K, TINY, U, esum

TERMS = 27
ENTRIES = 35             # view [16] | proj [16] | campos [3]
GB_THREADS = 128         # preprocess_bwd.cu: rows per block of geom_bwd_cam_kernel
REDUCTION_ROUNDINGS = 8  # 5 butterfly levels + 3 adds of the 4 warp sums
GROUPS = dict(view=slice(0, 16), proj=slice(16, 32), campos=slice(32, 35))


def term_index(s):
    """camera_grad_finish_kernel's scatter of term s into the [view 16 | proj 16 | campos 3] entries"""
    if s < 12:
        return 4 * (s // 3) + s % 3
    if s < 24:
        j = (s - 12) % 3
        return 16 + 4 * ((s - 12) // 3) + (3 if j == 2 else j)
    return 32 + s - 24


LAYOUT = [term_index(s) for s in range(TERMS)]
UNUSED = [4 * c + 3 for c in range(4)] + [16 + 4 * c + 2 for c in range(4)]   # exactly 0 in every output


def layout(terms):
    """[..., 27] terms (the oracle's rows, in the kernel's term order) -> [..., 35] entries"""
    t = np.asarray(terms)
    out = np.zeros(t.shape[:-1] + (ENTRIES,), t.dtype)
    out[..., LAYOUT] = t
    return out


MUTATIONS = ("textbook_clamp", "no_jt", "no_depth", "unshifted_sh", "campos_sign", "proj_col2", "transposed")


def _terms(ch, dm, mutation=None):
    """35 E (None: a structural zero) from ewa_chain's intermediates ch and the SH direction part dm (3 E)"""
    m, dT0, dT1 = ch["m"], ch["dT0"], ch["dT1"]
    vx, vy, vz = ch["vx"], ch["vy"], ch["vz"]
    if mutation == "no_depth":
        vz = ch["vz0"]
    if mutation == "textbook_clamp":
        # the derivative of the clamp: a clamped tx = lim tz moves with tz (the reference drops this term)
        vz = esum([vz, E(1.0 - ch["xgm"]) * ch["cx"] * (-ch["fx"] * ch["t2"] * ch["dJ02"]),
                   E(1.0 - ch["ygm"]) * ch["cy"] * (-ch["fy"] * ch["t2"] * ch["dJ12"])])
    g = [vx, vy, vz]
    out = [None] * ENTRIES
    for c in range(3):
        w = [ch["j00"] * dT0[c], ch["j11"] * dT1[c], ch["j02"] * dT0[c] + ch["j12"] * dT1[c]]
        for r in range(3):
            out[4 * c + r] = m[c] * g[r] if mutation == "no_jt" else m[c] * g[r] + w[r]
    for r in range(3):
        out[12 + r] = g[r]
    gp = [ch["d2x"] * ch["m_w"], ch["d2y"] * ch["m_w"], -(ch["mul1"] * ch["d2x"] + ch["mul2"] * ch["d2y"])]
    for c in range(4):
        for j, r in enumerate((0, 1, 2 if mutation == "proj_col2" else 3)):
            out[16 + 4 * c + r] = gp[j] if c == 3 else m[c] * gp[j]
    for k in range(3):
        out[32 + k] = dm[k] if mutation == "campos_sign" else -dm[k]
    if mutation == "transposed":
        for base in (0, 16):
            blk = out[base:base + 16]
            out[base:base + 16] = [blk[4 * r + c] for c in range(4) for r in range(4)]
    return out


def _stack(es, P, dev):
    z = torch.zeros(P, dtype=torch.float64, device=dev)
    return G.stack([E(z) if e is None else e for e in es], 1)


def restate(sc, st, out, clamped, means_out, vis, has_sh=True, exact=False, mutation=None):
    """The camera terms of every row as E [P,35] (rows not in vis: exactly 0), the float64 difference of the other
    frustum-clamp branch on the rows near it [P,35], and that near mask [P].

    sc: the scene (shs, ts, the SH and time settings; means3D for the 'unshifted_sh' mutation); st: raster settings;
    out: what the backward consumed -- dL_dmeans2D (after the blend map: x, y per NDC unit and the depth gradient),
    dL_dconic [P,4], dL_dcolors and the forward's cov3D; clamped [P,3] bool: the forward's clamp bits; means_out [P,3]:
    the forward's shifted means; vis [P] bool: the rendered rows.  exact: the float64 camera constants (gauss_f64.
    ewa_consts) instead of the kernels' fp32 ones.  mutation: one of MUTATIONS, a deliberately wrong variant."""
    P = means_out.shape[0]
    dev = means_out.device
    if has_sh:
        sh_means = sc.means3D if mutation == "unshifted_sh" else means_out
        dm = G.sh_backward(sc.shs, out["dL_dcolors"], clamped, sh_means, st["campos"].cpu().double(),
                           sc.ts[:, 0] if sc.gaussian_dim == 4 else None, st["timestamp"], sc.time_duration,
                           sc.sh_degree, sc.sh_degree_t, not (sc.gaussian_dim == 3 or sc.force_sh_3d))[2]
    else:
        dm = [E(torch.zeros(P, dtype=torch.float64, device=dev))] * 3
    args = (means_out, out["cov3D"], out["dL_dmeans2D"], out["dL_dconic"], st)
    ch = G.ewa_chain(*args, exact=exact)
    t = _stack(_terms(ch, dm, mutation), P, dev)
    near = ch["near"].to(dev)
    alt = torch.zeros_like(t.v)
    if bool(near.any()):
        for fx, fy in ((True, False), (False, True), (True, True)):
            flip = (ch["nx"] & fx, ch["ny"] & fy)
            a = _stack(_terms(G.ewa_chain(*args, exact=exact, flip=flip), dm, mutation), P, dev)
            alt = torch.maximum(alt, (a.v - t.v).abs())
    vis = vis.to(dev)
    keep = vis[:, None]
    zero = torch.zeros((), dtype=torch.float64, device=dev)
    t = E(torch.where(keep, t.v, zero), torch.where(keep, t.e, zero))
    return dict(terms=t, alt=torch.where(keep, alt, zero), near=near & vis)


def reduce(r):
    """The float64 sum [35] of the rows' terms and its bound under the kernel's reduction (module docstring)."""
    t, alt = r["terms"], r["alt"]
    nblocks = (t.v.shape[0] + GB_THREADS - 1) // GB_THREADS
    a = t.v.abs().sum(0)
    v = t.v.sum(0)
    bound = t.e.sum(0) + alt.sum(0) + (REDUCTION_ROUNDINGS * U + nblocks * 2.0 ** -53) * a + U * v.abs()
    return v, bound


def kernel_order_sum(terms):
    """numpy: [P,27] fp32 terms summed as the kernels do -- per 128-row block an fp32 xor butterfly over each warp's
    32 lanes and the 4 warp sums in order; the blocks' partials in fp64 (lane l takes blocks l, l + 32, ..., then an
    fp64 butterfly); one rounding to fp32.  Returns [27] float32."""
    t = np.asarray(terms, np.float32)
    P = t.shape[0]
    nb = max((P + GB_THREADS - 1) // GB_THREADS, 1)
    pad = np.zeros((nb * GB_THREADS, TERMS), np.float32)
    pad[:P] = t
    v = pad.reshape(nb, 4, 32, TERMS)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[:, :, lanes ^ o]).astype(np.float32)
    w = v[:, 0, 0]
    for k in range(1, 4):
        w = (w + v[:, k, 0]).astype(np.float32)
    part = w.astype(np.float64)                                   # [nb, 27]
    acc = np.zeros((32, TERMS), np.float64)
    for b in range(nb):
        acc[b % 32] += part[b]
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[lanes ^ o]
    return acc[0].astype(np.float32)


def check_rows(label, got, r):
    """Every row's 35 entries (got [P,35]) within K (e + alt) + TINY of the restatement; the unused entries exactly 0.
    Returns the worst err / bar per group."""
    t = r["terms"]
    g = torch.as_tensor(np.asarray(got)).double().to(t.v.device)
    assert int(torch.count_nonzero(g[:, UNUSED])) == 0, (label, "a row writes an unused entry")
    err = (g - t.v).abs()
    bar = K * (t.e + r["alt"]) + TINY
    return _verdict(label, err, bar, g, t.v)


def check_sums(label, got, r, rows=None):
    """The 35 returned entries (got [35]) within K bound + TINY of the float64 sum, the unused ones exactly 0.  Prints
    and returns the worst err / bar per group."""
    v, bound = reduce(r)
    g = torch.as_tensor(np.asarray(got, np.float64) if not torch.is_tensor(got) else got.detach().cpu().double())
    g = g.reshape(-1).to(v.device)
    assert g.numel() == ENTRIES
    assert int(torch.count_nonzero(g[UNUSED])) == 0, (label, "an unused entry is not 0", g[UNUSED].tolist())
    worst = _verdict(label, (g - v).abs()[None], (K * bound + TINY)[None], g[None], v[None])
    if rows is not None:
        print("%-40s rows %6d (%d near the frustum clamp); worst err/bar: %s"
              % (label, rows, int(r["near"].sum()), "  ".join("%s %.3f" % kv for kv in worst.items())))
    return worst


# ---- scenes of one Gaussian, where a wrong term cannot hide inside a sum ----------------------------------------------
ONE_SCENES = ["clamp_x", "clamp_y", "clamp_xy", "near", "negfov", "sh4d"]


def one_scene(name):
    """(cfg, cam, sc, st) of one Gaussian on a 96x64 image (tan fov 0.93 x 0.62, clamp limits 1.2 x 0.80):
      clamp_x / clamp_y / clamp_xy  its centre at view x/z = 1.5 and / or y/z = 1.0, beyond the 1.3 tan(fov) frustum
                                    clamp, with a footprint (sigma ~ 20 px) that still reaches the image;
      near                          at view z = 0.25 (the near plane is 0.2): a screen sigma of ~100-170 px;
      negfov                        the N3V camera (FoV -1: tan fov < 0, every row under the clamp) at the centre;
      sh4d                          rot_4d, SH degree 3 with D_t = 2, the posed camera of rotcam (campos != 0) and a
                                    timestamp 0.3 temporal sigma off (the shifted mean is not the mean)."""
    from fdgs import synth
    import helpers
    seed = 9400 + ONE_SCENES.index(name)
    R = T = None
    if name == "sh4d":
        R, T = synth.pose_from_euler(*helpers.CONFIGS["rotcam"]["pose"])
    cam = synth.make_camera(96, 64, negative_fov=name == "negfov", R=R, T=T)
    sc = synth.make_scene(1, cam, seed, zmin=4.0, zmax=4.0, frustum=0.2)
    sc.ts[:] = cam.timestamp
    if name != "sh4d":
        x = 6.0 if name in ("clamp_x", "clamp_xy") else 0.3
        y = 4.0 if name in ("clamp_y", "clamp_xy") else -0.2
        z = 4.0
        if name == "near":
            x, y, z = 0.01, -0.02, 0.25
            sc.scales[:] = torch.tensor([0.8, 0.5, 0.6])
        elif name.startswith("clamp"):
            sc.scales[:] = 1.5
        sc.means3D[:] = torch.tensor([x, y, z])
    else:
        sc.ts[:] = cam.timestamp + 0.3 * sc.scales_t
    sc.opacities[:] = 0.7
    st = synth.raster_settings(cam, sc)
    return dict(W=96, H=64, seed=seed, P=1), cam, sc, st


def one_scene_regime(name, st, means, means_out, radii, vis):
    """asserts on the forward's state that a one-Gaussian scene reaches its regime"""
    assert bool(vis.all()), (name, "not rendered")
    V = st["viewmatrix"].double().cpu()
    mh = torch.cat([means_out.double().cpu(), torch.ones(1, 1, dtype=torch.float64)], 1)
    t = (mh @ V)[0]
    tanx, tany = float(st["tanfovx"]), float(st["tanfovy"])
    outx, outy = abs(t[0] / t[2]) > 1.3 * abs(tanx), abs(t[1] / t[2]) > 1.3 * abs(tany)
    if name.startswith("clamp"):
        assert (outx, outy) == ("x" in name[6:], "y" in name[6:]), (name, t)
    elif name == "near":
        assert 0.2 < float(t[2]) < 0.3 and int(radii[0]) > 300, (name, t, radii)
    elif name == "negfov":
        assert tanx < 0 and tany < 0, name
    elif name == "sh4d":
        assert st["sh_degree"] == 3 and st["sh_degree_t"] == 2 and st["rot_4d"]
        assert float(st["campos"].abs().max()) > 0.1
        assert float((means_out.cpu() - means.cpu()).abs().max()) > 1e-3, (name, "the mean is not shifted")


def _verdict(label, err, bar, got, want):
    assert torch.isfinite(got).all(), (label, "non-finite")
    ratio = err / bar
    worst = {k: float(ratio[:, s].max()) if ratio.shape[0] else 0.0 for k, s in GROUPS.items()}
    if max(worst.values()) > 1.0:
        i, j = torch.nonzero(ratio > 1.0)[0].tolist()
        raise AssertionError("%s: %d entries beyond K bound + tiny (worst err/bar %s); first at row %d, entry %d: got %r, "
                             "float64 %r, bar %.3g" % (label, int((ratio > 1).sum()), worst, i, j, got[i, j].item(),
                                                       want[i, j].item(), bar[i, j].item()))
    return worst
