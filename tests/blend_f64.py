"""The 3D rasterizer (precomputed colours and covariances) restated in float64 torch, for the regime tests: projection,
EWA splatting with the 0.3 low-pass, and the per-tile front-to-back blend over given tile lists, with autograd for the
gradients.  Decisions (power > 0, the 1/255 cut, the T < 1e-4 stop) are taken in float64 on the float64 values.  The
reference's semantics, not textbook ones, are restated:
  - the 0.99 clamp of alpha is straight-through in the backward (reference: backward.cu uses dL/dG = o dL/dalpha);
  - the pair whose alpha would take T below 1e-4 does not blend;
  - dL/dmeans2D is per NDC unit (columns x, y) plus dL/ddepth (column 2);
  - the conic's backward divides by det^2 + 1e-7 (backward.cu computeCov2DCUDA).
TEST INFRASTRUCTURE."""
import numpy as np
import torch

F64 = torch.float64
CUT = 1.0 / 255.0
T_STOP = 1e-4
AMBIG = 1e-5           # a decision this close (relative) to its threshold makes the pixel ambiguous ...


class _Conic(torch.autograd.Function):
    """(a, b, c) of the dilated 2D covariance -> (c, -b, a) / det, with the reference's backward (det^2 + 1e-7)."""

    @staticmethod
    def forward(ctx, a, b, c):
        det = a * c - b * b
        ctx.save_for_backward(a, b, c)
        return c / det, -b / det, a / det

    @staticmethod
    def backward(ctx, gx, gy, gz):
        a, b, c = ctx.saved_tensors
        det = a * c - b * b
        inv = 1.0 / (det * det + 1e-7)
        da = inv * (-c * c * gx + b * c * gy + (det - a * c) * gz)
        dc = inv * (-a * a * gz + a * b * gy + (det - a * c) * gx)
        db = inv * (2.0 * b * c * gx - (det + 2.0 * b * b) * gy + 2.0 * a * b * gz)
        return da, db, dc


def project(st, means3D, cov3D):
    """float64 means2D (pixels), NDC xy and depth [P], the conic [P,3] and whether the frustum clamp is active [P]."""
    W, H = int(st["image_width"]), int(st["image_height"])
    view = torch.as_tensor(st["viewmatrix"]).detach().cpu().to(F64).t()      # row-major world -> camera
    proj = torch.as_tensor(st["projmatrix"]).detach().cpu().to(F64).t()
    tanx = float(np.float32(st["tanfovx"]))
    tany = float(np.float32(st["tanfovy"]))
    fx, fy = W / (2.0 * tanx), H / (2.0 * tany)
    ones = torch.ones(means3D.shape[0], 1, dtype=F64)
    mh = torch.cat([means3D, ones], 1)
    t = mh @ view.T
    ph = mh @ proj.T
    pw = 1.0 / (ph[:, 3] + 1e-7)
    ndc = torch.stack([ph[:, 0] * pw, ph[:, 1] * pw], 1)
    depth = t[:, 2]
    pix = torch.stack([((ndc[:, 0] + 1.0) * W - 1.0) * 0.5, ((ndc[:, 1] + 1.0) * H - 1.0) * 0.5], 1)
    limx, limy = 1.3 * tanx, 1.3 * tany
    txtz, tytz = t[:, 0] / t[:, 2], t[:, 1] / t[:, 2]
    clamped = (txtz.detach().abs() > limx) | (tytz.detach().abs() > limy)
    tx = txtz.clamp(-limx, limx) * t[:, 2]
    ty = tytz.clamp(-limy, limy) * t[:, 2]
    tz = t[:, 2]
    z = torch.zeros_like(tz)
    J = torch.stack([torch.stack([fx / tz, z, -fx * tx / (tz * tz)], 1),
                     torch.stack([z, fy / tz, -fy * ty / (tz * tz)], 1)], 1)          # [P,2,3]
    Tm = J @ view[:3, :3]
    c = cov3D
    S = torch.stack([torch.stack([c[:, 0], c[:, 1], c[:, 2]], 1), torch.stack([c[:, 1], c[:, 3], c[:, 4]], 1),
                     torch.stack([c[:, 2], c[:, 4], c[:, 5]], 1)], 1)
    cov2 = Tm @ S @ Tm.transpose(1, 2)
    cx, cy, cz = _Conic.apply(cov2[:, 0, 0] + 0.3, cov2[:, 0, 1], cov2[:, 1, 1] + 0.3)
    return pix, ndc, depth, torch.stack([cx, cy, cz], 1), clamped


def walk_tile(pix, conic, opacity, ids, x0, y0, W, H, ill=None):
    """One tile's float64 walk.  Returns the blend weights w [n,L] (autograd-carrying), T_final [n], the pixel indices,
    and decision records for the pixels: ambiguous [n], terminated [n], clamped contributor [n], and per pair the float64
    alpha and whether it blends / was walked (numpy)."""
    xs = torch.arange(x0, min(x0 + 16, W), dtype=F64)
    ys = torch.arange(y0, min(y0 + 16, H), dtype=F64)
    py, px = torch.meshgrid(ys, xs, indexing="ij")
    px, py = px.reshape(-1, 1), py.reshape(-1, 1)
    pid = (py.long() * W + px.long()).reshape(-1)
    m = pix[ids]
    co = conic[ids]
    o = opacity[ids]
    dx = m[None, :, 0] - px
    dy = m[None, :, 1] - py
    power = -0.5 * (co[None, :, 0] * dx * dx + co[None, :, 2] * dy * dy) - co[None, :, 1] * dx * dy
    G = torch.exp(power)
    og = o[None, :] * G
    alpha = og + (torch.clamp_max(og, 0.99) - og).detach()              # straight-through clamp
    with torch.no_grad():
        p, a = power.detach(), alpha.detach()
        valid = (p <= 0) & (a >= CUT)
        one_m = torch.where(valid, 1.0 - a, torch.ones_like(a))
        Tb = torch.cumprod(torch.cat([torch.ones_like(a[:, :1]), one_m[:, :-1]], 1), 1)
        test_T = Tb * (1.0 - a)
        stop = valid & (test_T < T_STOP)
        before = torch.cumsum(stop.to(torch.int64), 1) - stop.to(torch.int64) == 0     # pairs walked (stop included)
        incl = valid & before & ~stop
        # ... and where fp32 cannot evaluate power to that accuracy: far from a needle's centre the terms of the
        # quadratic form are thousands of times larger than their sum (rounding bound 2^-22 of the terms), which matters
        # for a pair that blends or that the error could lift over the cut
        err = 2.0 ** -22 * (0.5 * (co[None, :, 0].detach() * dx.detach() ** 2 + co[None, :, 2].detach() * dy.detach() ** 2)
                            + (co[None, :, 1].detach() * dx.detach() * dy.detach()).abs())
        amb = before & ((p.abs() <= AMBIG) | ((a - CUT).abs() <= AMBIG * CUT) | ((err > AMBIG) & (a * torch.exp(err) >= CUT)) |
                        (valid & ((test_T - T_STOP).abs() <= AMBIG * T_STOP)))
        ambiguous = amb.any(1)
        # pixels where a Gaussian with an ill-conditioned fp32 conic may blend (see ill_conditioned)
        ill_px = (before & (a >= 0.5 * CUT) & ill[ids][None, :]).any(1) if ill is not None else torch.zeros_like(ambiguous)
        terminated = stop.any(1)
        clamp_hit = (incl & (og >= 0.99)).any(1)
    f = torch.where(incl, 1.0 - alpha, torch.ones_like(alpha))
    Tb = torch.cumprod(torch.cat([torch.ones_like(f[:, :1]), f[:, :-1]], 1), 1)
    w = torch.where(incl, alpha * Tb, torch.zeros_like(alpha))
    T_final = torch.prod(f, 1)
    rec = dict(ambiguous=ambiguous.numpy(), ill=ill_px.numpy(), terminated=terminated.numpy(), clamp_hit=clamp_hit.numpy(),
               alpha=a.numpy(), incl=incl.numpy(), walked=before.numpy())
    return w, T_final, pid, rec


def ill_conditioned(conic_opacity):
    """Rows whose fp32 conic loses more than 1e-5 relative when fp32 inverts the dilated 2D covariance: det = a c - b^2
    cancels log2(a c / det) bits (needles), i.e. rows with 4 * 2^-24 * a c / det > 1e-5.  Returns the mask and the
    per-row loss factor (bound / 1e-5, at least 1)."""
    con = np.asarray(conic_opacity, np.float64)[:, :3]
    ac = con[:, 0] * con[:, 2]
    det = ac - con[:, 1] ** 2
    with np.errstate(divide="ignore", invalid="ignore"):
        kappa = np.where(det > 0, ac / det, np.inf)
    loss = np.maximum(1.0, 4 * 2.0 ** -24 * kappa / 1e-5)
    return loss > 1.0, loss


def render(st, lists, means3D, cov3D, colors, opacity, flows, with_records=False, ill=None):
    """Images (colour [3,H,W], depth [1,H,W], alpha [1,H,W], flow [2,H,W]), the per-pixel ambiguity mask [H,W], and the
    intermediates whose gradients the rasterizer returns.  lists: dict(ranges [tiles,2], point_list) in the reference's
    order.  All tensors float64 on the CPU."""
    W, H = int(st["image_width"]), int(st["image_height"])
    bg = torch.as_tensor(st["bg"]).detach().cpu().to(F64)
    pix, ndc, depth, conic, fclamp = project(st, means3D, cov3D)
    ranges = np.asarray(lists["ranges"]).reshape(-1, 2).astype(np.int64)
    plist = torch.from_numpy(np.asarray(lists["point_list"]).astype(np.int64))
    gx = (W + 15) // 16
    feats = torch.cat([colors, depth[:, None], flows], 1)                # [P, 6]
    out = torch.zeros(H * W, 6, dtype=F64)
    T_img = torch.ones(H * W, dtype=F64)
    pieces, tpieces, pids = [], [], []
    amb = np.zeros(H * W, bool)
    illp = np.zeros(H * W, bool)
    ill_t = torch.from_numpy(np.asarray(ill, bool)) if ill is not None else None
    records = {}
    for t in range(ranges.shape[0]):
        lo, hi = ranges[t]
        x0, y0 = (t % gx) * 16, (t // gx) * 16
        if hi <= lo:
            continue
        ids = plist[lo:hi]
        w, Tf, pid, rec = walk_tile(pix, conic, opacity, ids, x0, y0, W, H, ill_t)
        pieces.append(w @ feats[ids])
        tpieces.append(Tf)
        pids.append(pid)
        amb[pid.numpy()] = rec["ambiguous"]
        illp[pid.numpy()] = rec["ill"]
        if with_records:
            records[t] = (pid.numpy(), ids.numpy(), rec)
    if pids:
        pid = torch.cat(pids)
        out = out.index_put((pid,), torch.cat(pieces))
        T_img = T_img.index_put((pid,), torch.cat(tpieces))
    color = (out[:, :3] + T_img[:, None] * bg[None, :]).t().reshape(3, H, W)
    imgs = dict(color=color, depth=out[:, 3].reshape(1, H, W), alpha=(1.0 - T_img).reshape(1, H, W),
                flow=out[:, 4:6].t().reshape(2, H, W), T=T_img.reshape(H, W))
    return dict(images=imgs, ambiguous=amb.reshape(H, W), ill=illp.reshape(H, W), frustum_clamp=fclamp.numpy(), ndc=ndc, depth=depth,
                pix=pix, conic=conic, records=records)


def forward_backward(st, lists, twin, grads, mask_ambiguous=True, ill=None):
    """twin: dict of float32 arrays/tensors means3D [P,3], cov3D [P,6], colors [P,3], opacity [P], flows [P,2].
    grads: upstream (colour [3,H,W], depth [1,H,W], alpha [1,H,W], flow [2,H,W]); any may be None (no gradient).
    ill: rows with an ill-conditioned fp32 conic (ill_conditioned); the pixels where they may blend are masked like the
    ambiguous ones and returned as "ill".
    Returns images, the masked upstream gradients (float32 numpy, to feed every implementation alike), the gradients
    dL/d(means3D, cov3D, colors, opacity, flows, means2D) as float64 numpy, and the masks."""
    leaf = lambda k: torch.as_tensor(np.asarray(twin[k], np.float32)).to(F64).requires_grad_(True)
    L = {k: leaf(k) for k in ("means3D", "cov3D", "colors", "opacity", "flows")}
    r = render(st, lists, L["means3D"], L["cov3D"], L["colors"], L["opacity"].reshape(-1), L["flows"], ill=ill)
    r["ndc"].retain_grad()
    r["depth"].retain_grad()
    keep = torch.from_numpy(~(r["ambiguous"] | r["ill"])).to(F64) if mask_ambiguous else 1.0
    masked = []
    loss = 0.0
    for g, key in zip(grads, ("color", "depth", "alpha", "flow")):
        if g is None:
            masked.append(None)
            continue
        gm = (torch.as_tensor(np.asarray(g, np.float32)).to(F64) * keep).to(torch.float32)
        masked.append(gm.numpy())
        loss = loss + (r["images"][key] * gm.to(F64)).sum()
    loss.backward()
    W, H = int(st["image_width"]), int(st["image_height"])
    m2 = torch.cat([r["ndc"].grad, r["depth"].grad[:, None]], 1)
    out = dict(dL_dmeans3D=L["means3D"].grad, dL_dcov3D=L["cov3D"].grad, dL_dcolors=L["colors"].grad,
               dL_dopacity=L["opacity"].grad.reshape(-1, 1), dL_dflows=L["flows"].grad, dL_dmeans2D=m2)
    return dict(images={k: v.detach().numpy() for k, v in r["images"].items()}, grads_in=masked,
                grads={k: v.detach().numpy() for k, v in out.items()}, ambiguous=r["ambiguous"], ill=r["ill"],
                frustum_clamp=r["frustum_clamp"], W=W, H=H)
