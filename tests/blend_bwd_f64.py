"""Float64 restatement of the blend backward (blend_bwd.cu, finished by preprocess_bwd.cu geom_bwd_body's linear map)
with a first-order bound on the error of any fp32 evaluation with the kernel's structure or the reference's per-pair
structure.

The inputs are the forward's own fp32 screen-space state -- means2D (pixels), conic_opacity (A, B, C, blended opacity),
rgb, depths, the tile lists (point_list, ranges), n_contrib and final_T -- plus the per-Gaussian flows, the background
(and the optional per-pixel background image) and the upstream image gradients.  The oracle's forward() dict and the
GPU's debug exports provide the same fields, so one function serves both.

Contributors are the fp32 forward's (decide): its power expression (blend_fwd.cu, fma emulated as one rounding of the
exact float64 product-sum), power > 0, alpha < 1/255f and test_T < 1e-4f are replicated in float32.  A pixel is masked
(its upstream gradient zeroed, for the kernel and the restatement alike) only where a decision lies within the fp32
uncertainty of expf of its threshold, or where the replica's last contributor differs from the forward's n_contrib.
(power < pmin never decides: pmin = -(log(255 o) + 0.02) lies 2 % below the alpha cut.)

Values (backward) are float64 of the same contributors; every value is a gauss_f64.E whose error covers:
  - T: the forward's front-to-back product for final_T and the backward's recovery T_final / prod (1 - alpha);
  - power: the exact per-pixel expression with expf, or the kernel's expansion about the 8x4 warp rectangle's centre
    with ex2.approx -- the larger bound, since which path a pair took is not observable; except that the kernel's
    exact flag (|A X^2| + |C Y^2| + 2 |B X Y| >= 128 about the warp rectangle's centre) forces the exact path;
  - the back-to-front acc recurrences of colour, depth, flow and alpha (contracting: 1 - alpha <= 1);
  - the reductions: per (warp, Gaussian) the tf32-split tensor-core sum over 32 pixels, the re-centring of the raw
    moments on the Gaussian's mean, then an order-free esum over all partials of a row (RED order); or, per pair, the
    reference's products summed in any order.

Intrinsic constants (relative):
  EXPF  expf: 2 ulp = 2^-22 (CUDA C++ Programming Guide, mathematical functions, single precision: expf, 2 ulp).
  EX2   ex2.approx.ftz.f32: 2^-22 (PTX ISA, ex2: maximum relative error over the full range).
  RCP   rcp.approx.ftz.f32: 2^-23 (PTX ISA, rcp.approx: 1 ulp).
  Tensor core (mma.sync m16n8k8 tf32, fp32 accumulate):
    split: hi = x & 0xffffe000 keeps 11 significant bits, lo = x - hi is read as tf32 (11 bits), so the pair
           represents x within 2^-20 |x|; a product of two split operands within 2^-19 |a b|;
    accumulation: (k + 1) 2^-23 sum |terms| per k-term group, the accumulator counted as a term.  This is an
           ASSUMPTION -- a conservative model of truncating alignment -- because NVIDIA does not document how the
           tensor core accumulates.  No measurement sets any constant here.
TEST INFRASTRUCTURE."""
import numpy as np
import torch

from gauss_f64 import E, K, TINY, U, esum

F64 = torch.float64
EXPF = 2.0 ** -22
EX2 = 2.0 ** -22
RCP = 2.0 ** -23
SPLIT = 2.0 ** -20
ACC = 9 * 2.0 ** -23          # (k + 1) 2^-23, k = 8
CUT32 = np.float32(1.0 / 255.0)
TSTOP32 = np.float32(1e-4)
CLAMP32 = np.float32(0.99)
LOG2E = 1.4426950408889634
LN2 = 0.6931471805599453
ULP = 2.0 ** -23              # relative spacing of fp32
# largest masked fraction of a scene's pixels: the regime scene `threshold` puts about 900 pairs within ulps of the
# 1/255 cut by construction (its pairs at exactly fp32(1/255) and G = 1 are decided, not masked), about 3 % of its pixels
MAX_MASKED = 0.05


def _tile_pixels(t, gx, W, H):
    """the 256 pixels of tile t, row-major 16x16 (pixel coordinates, and whether each lies inside the image)"""
    x0, y0 = (t % gx) * 16, (t // gx) * 16
    ys, xs = np.mgrid[y0:y0 + 16, x0:x0 + 16]
    xs, ys = xs.reshape(-1), ys.reshape(-1)
    return xs, ys, (xs < W) & (ys < H)


def fp32_power(mx, my, A, B, C, px, py):
    """forward.cu:578-581 as compiled (blend_fwd.cu): fma(fma(dx, dx*A, dy*(dy*C)), -0.5, -(dy*(dx*B))) in float32,
    each fma one rounding of the exact float64 product-sum.  mx..C [n] float32, px, py [m] float32 -> [m, n]"""
    f32, f64 = np.float32, np.float64
    dx = mx[None, :] - px[:, None]
    dy = my[None, :] - py[:, None]
    dxA = dx * A[None, :]
    dyyC = dy * (dy * C[None, :])
    inner = (dx.astype(f64) * dxA.astype(f64) + dyyC.astype(f64)).astype(f32)
    dydxB = dy * (dx * B[None, :])
    return (-0.5 * inner.astype(f64) - dydxB.astype(f64)).astype(f32)


def decide(st):
    """The fp32 forward's contributors and the pixels to mask.  st: dict of numpy arrays means2D [P,2], conic_opacity
    [P,4], point_list [R], ranges [tiles,2], n_contrib [H,W], W, H.  Returns dict(tiles=[(t, pid [256], inside [256],
    ids [n], contrib [256, n] bool)], mask [H,W] bool (True: masked), stats), stats holding the edges the state
    reaches (edge_reached): pixels that terminate / do not, the per-warp column counts mod 8, the largest offset of a
    contributing Gaussian's mean from a warp rectangle's centre and the largest |A X^2| + |C Y^2| + 2 |B X Y| there."""
    W, H = int(st["W"]), int(st["H"])
    gx = (W + 15) // 16
    m2 = np.asarray(st["means2D"], np.float32)
    co = np.asarray(st["conic_opacity"], np.float32)
    pl = np.asarray(st["point_list"]).astype(np.int64).reshape(-1)
    ranges = np.asarray(st["ranges"]).astype(np.int64).reshape(-1, 2)
    nc = np.asarray(st["n_contrib"]).astype(np.int64).reshape(-1)
    mask = np.zeros(H * W, bool)
    tiles = []
    n_amb = n_mis = n_nan = 0
    n_cut_exact = n_term = n_open = 0
    tail_mods, far_max, flag_max = set(), 0.0, 0.0
    for t in range(ranges.shape[0]):
        lo, hi = ranges[t]
        xs, ys, inside = _tile_pixels(t, gx, W, H)
        pid = np.where(inside, ys * W + xs, 0)
        fwd_n = np.where(inside, nc[pid], 0)
        if hi <= lo:
            if (fwd_n != 0).any():
                mask[pid[inside & (fwd_n != 0)]] = True
                n_mis += int((inside & (fwd_n != 0)).sum())
            continue
        ids = pl[lo:hi]
        power = fp32_power(m2[ids, 0], m2[ids, 1], co[ids, 0], co[ids, 1], co[ids, 2], xs.astype(np.float32),
                           ys.astype(np.float32))
        o = co[ids, 3].astype(np.float64)[None, :]
        p64 = power.astype(np.float64)
        with np.errstate(over="ignore", invalid="ignore"):
            G32 = np.exp(p64).astype(np.float32)
            og32 = G32 * co[ids, 3][None, :]
            og64 = o * np.exp(p64)
        a32 = np.minimum(og32, CLAMP32)
        nan = ~np.isfinite(power) | ~np.isfinite(og64)
        valid = (power <= 0) & ~(a32 < CUT32) & ~nan
        # expf is within 2 ulp, o * G one more rounding; power == 0 gives G = 1 exactly (expf(0) = 1): then og = o
        unc = np.where(power == 0, 0.0, 4 * ULP * og64)
        amb_cut = (power <= 0) & (np.abs(og64 - np.float64(CUT32)) <= unc)
        n_cut_exact += int(((power == 0) & (og32 == CUT32)).sum())
        a64 = a32.astype(np.float64)
        ua = np.where(og64 > 0.99 * (1 + 1e-6), 0.0, 4 * ULP * a64)          # clamped robustly: exactly 0.99
        with np.errstate(invalid="ignore"):
            factor = np.where(valid, (np.float32(1.0) - a32), np.float32(1.0)).astype(np.float32)
        cp = np.cumprod(factor, axis=1, dtype=np.float32)                  # test_T of every valid pair, in order
        stop = valid & (cp < TSTOP32)
        first = np.where(stop.any(1), stop.argmax(1), power.shape[1])
        pos = np.arange(power.shape[1])[None, :]
        walked = pos <= first[:, None]
        contrib = valid & (pos < first[:, None])
        rel = np.cumsum(np.where(valid, ua / np.maximum(1.0 - a64, 1e-3) + 2 * U, 0.0), axis=1)
        amb_T = valid & walked & (np.abs(cp.astype(np.float64) - np.float64(TSTOP32)) <= rel * cp.astype(np.float64))
        last = np.where(contrib.any(1), power.shape[1] - np.argmax(contrib[:, ::-1], 1), 0)
        amb = ((amb_cut | amb_T) & walked).any(1) & inside
        bad = (nan & walked).any(1) & inside
        mis = (last != fwd_n) & inside
        m = amb | mis | bad
        n_amb += int(amb.sum())
        n_mis += int((mis & ~amb).sum())
        n_nan += int(bad.sum())
        mask[pid[m & inside]] = True
        stopped = inside & (first < power.shape[1]) & contrib.any(1)
        n_term += int(stopped.sum())
        n_open += int((inside & ~stopped & contrib.any(1)).sum())
        # the kernel's view of the tile: per 8x4 warp, the Gaussians contributing to any of its pixels (its columns),
        # their offset from the warp rectangle's centre and the magnitude of the expansion's terms (the exact flag)
        wc = (contrib & inside[:, None]).reshape(4, 4, 2, 8, -1).any((1, 3))          # [wy, wx, n]
        cols = wc.sum(2)
        tail_mods.update(int(c) % 8 for c in cols.reshape(-1) if c > 0)
        if wc.any():
            wy, wx, j = np.nonzero(wc)
            x0, y0 = (t % gx) * 16, (t // gx) * 16
            X = m2[ids[j], 0].astype(np.float64) - (x0 + 8 * wx + 3.5)
            Y = m2[ids[j], 1].astype(np.float64) - (y0 + 4 * wy + 1.5)
            c = co[ids[j]].astype(np.float64)
            far_max = max(far_max, float(np.maximum(np.abs(X), np.abs(Y)).max()))
            flag_max = max(flag_max, float((np.abs(c[:, 0] * X * X) + np.abs(c[:, 2] * Y * Y)
                                            + 2 * np.abs(c[:, 1] * X * Y)).max()))
        n = int(fwd_n.max())
        contrib = contrib[:, :n] & (inside & ~m)[:, None]
        tiles.append((t, pid, inside & ~m, ids[:n], contrib))
    stats = dict(pixels=W * H, masked=int(mask.sum()), ambiguous=n_amb, mismatched=n_mis, nan=n_nan,
                 cut_exact_pairs=n_cut_exact, terminated=n_term, open=n_open, tail_mods=sorted(tail_mods),
                 far_max=far_max, flag_max=flag_max)
    return dict(tiles=tiles, mask=mask.reshape(H, W), stats=stats)


def mask_grads(grads, mask):
    """upstream gradients (colour [3,H,W], depth [1,H,W], alpha [1,H,W], flow [2,H,W]; None: none) with the masked
    pixels zeroed, float32 numpy"""
    keep = ~np.asarray(mask)
    return [None if g is None else (np.asarray(g, np.float32) * keep[None]).astype(np.float32) for g in grads]


class _Acc:
    """per-row accumulation of partial sums: value, error, |value| and count -> E with the order-free sum bound"""

    def __init__(self, P, width):
        z = lambda: torch.zeros(P, width, dtype=F64)
        self.v, self.e, self.a, self.n = z(), z(), z(), z()

    def add(self, rows, v, e):
        """rows [k] long; v, e [k, width]"""
        self.v.index_add_(0, rows, v)
        self.e.index_add_(0, rows, e)
        self.a.index_add_(0, rows, v.abs())
        self.n.index_add_(0, rows, (v != 0).to(F64))

    def E(self):
        return E(self.v, self.e + (self.n - 1).clamp_min(0) * U * self.a)


def _chain_err(terms):
    """accumulation bound of the per (warp, Gaussian) tensor-core chain.  terms [4 (row s), 8 (pixels), ...] |terms| of
    a hi product; the chain is hi(s = 0), lo(0), hi(1), lo(1), ...; a lo group's terms are at most 2^-10 of its hi"""
    S = terms.abs().sum(1)                        # [4, ...]
    err = torch.zeros_like(S[0])
    before = torch.zeros_like(S[0])
    for s in range(4):
        for g in (S[s], 2.0 ** -10 * S[s]):
            err = err + ACC * (g + before)
            before = before + g
    return err


def backward(st, dec, grads, bg, bg_image=None):
    """The float64 blend backward over decide()'s contributors with the (masked) upstream gradients.
    st: as decide, plus rgb [P,3], depths [P], flows [P,2], final_T [H,W]; bg [3]; bg_image [3,H,W] or None;
    grads: (colour, depth, alpha, flow) float32 numpy, any None.  Returns dict name -> E over all P rows:
    dL_dmeans2D [P,3] (x, y per NDC unit after geom_bwd_body's map, z the depth gradient), dL_dconic [P,3] (x, y, w),
    dL_dopacity [P,1] (the blend sum: times the marginal for 4D rows, see opacity()), dL_dcolors [P,3], dL_dflows [P,2];
    and 'T_final' (float64 E of the forward's T per pixel, NaN where not walked) for checking the forward's."""
    W, H = int(st["W"]), int(st["H"])
    HW = W * H
    P = np.asarray(st["means2D"]).shape[0]
    t64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64))
    m2, co, rgb = t64(st["means2D"]), t64(st["conic_opacity"]), t64(st["rgb"])
    depth, flows = t64(st["depths"]).reshape(-1), t64(st["flows"]).reshape(-1, 2)
    Tfin = t64(st["final_T"]).reshape(-1)
    gc, gd, ga, gf = grads
    zeros = lambda k: torch.zeros(k, HW, dtype=F64)
    gpix = t64(gc).reshape(3, HW)
    aux = [t64(gd).reshape(1, HW) if gd is not None else zeros(1), t64(gf).reshape(2, HW) if gf is not None else zeros(2),
           t64(ga).reshape(1, HW) if ga is not None else zeros(1)]
    has_aux = any(g is not None for g in (gd, ga, gf))
    bgp = t64(np.asarray(bg, np.float32)).reshape(3, 1).expand(3, HW)
    bg_err = torch.zeros(3, HW, dtype=F64)
    if bg_image is not None:
        bgi = t64(bg_image).reshape(3, HW)
        bgp = bgp + bgi
        bg_err = U * bgp.abs()
    # kernel structure: moments W00 W10 W01 W20 W11 W02, then a1-weighted colour r g b, depth, flow x y
    kern = _Acc(P, 12)
    # per-pair structure: means2D x y (mapped), depth, conic x y w, opacity, colour r g b, flow x y
    pair = _Acc(P, 12)
    T_out = torch.full((HW,), float("nan"), dtype=F64)
    T_err = torch.zeros(HW, dtype=F64)
    for (t, pid_np, live_np, ids_np, contrib_np) in dec["tiles"]:
        n = len(ids_np)
        if n == 0 or not contrib_np.any():
            continue
        gx = (W + 15) // 16
        xs, ys, _ = _tile_pixels(t, gx, W, H)
        pid = torch.from_numpy(pid_np)
        ids = torch.from_numpy(ids_np)
        inc = torch.from_numpy(contrib_np)
        incf = inc.to(F64)
        px = torch.from_numpy(xs.astype(np.float64))[:, None]
        py = torch.from_numpy(ys.astype(np.float64))[:, None]
        mx, my = m2[ids, 0][None, :], m2[ids, 1][None, :]
        A, B, C, o = (co[ids, k][None, :] for k in range(4))
        dx, dy = mx - px, my - py
        # ---- power and G: the exact path and the polynomial path ----
        power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
        S = 0.5 * A.abs() * dx * dx + 0.5 * C.abs() * dy * dy + (B * dx * dy).abs()
        G = torch.exp(power) * incf
        eG_exact = G * (torch.expm1(6 * U * S) + EXPF)
        rcx = torch.from_numpy((8 * (xs // 8) + 3.5).astype(np.float64))[:, None]
        rcy = torch.from_numpy((4 * (ys // 4) + 1.5).astype(np.float64))[:, None]
        X, Y = mx - rcx, my - rcy
        u, v = px - rcx, py - rcy
        T0 = 0.5 * A.abs() * X * X + 0.5 * C.abs() * Y * Y + (B * X * Y).abs()
        Q = LOG2E * (T0 + ((A * X).abs() + (B * Y).abs()) * u.abs() + ((C * Y).abs() + (B * X).abs()) * v.abs()
                     + 0.5 * A.abs() * u * u + (B * u * v).abs() + 0.5 * C.abs() * v * v)
        eG_poly = G * (torch.expm1(LN2 * 13 * U * Q) + EX2)
        # the kernel evaluates every pair of an instance whose expansion has large cancelling terms exactly (its flag
        # |A X^2| + |C Y^2| + 2 |B X Y| >= 128, fp32 on the same inputs): there the path is known; elsewhere it is not
        flagged = (A * X * X).abs() + (C * Y * Y).abs() + 2 * (B * X * Y).abs() >= 128.0 * (1 + 1e-5)
        eG = torch.where(flagged, eG_exact, torch.maximum(eG_exact, eG_poly))
        og = o * G
        e_og = o * eG + U * og
        alpha = torch.clamp_max(og, 0.99) * incf
        e_a = torch.where(og - e_og > 0.99, torch.zeros_like(og), e_og) * incf
        one_m = torch.where(inc, 1.0 - alpha, torch.ones_like(alpha))
        # ---- T: float64 front-to-back; error: the forward's product for final_T and the backward's recovery ----
        Tb = torch.cumprod(torch.cat([torch.ones_like(one_m[:, :1]), one_m[:, :-1]], 1), 1)
        Tf = torch.prod(one_m, 1)
        rin = torch.where(inc, e_a / one_m, torch.zeros_like(alpha))
        rel_f = (rin + 2 * U * incf).sum(1, keepdim=True)
        rel_b = torch.flip(torch.cumsum(torch.flip((rin + (2 * U + RCP) * incf), [1]), 1), [1])
        T = E(Tb, Tb * (rel_f + rel_b))
        TfE = E(Tf[:, None], Tf[:, None] * rel_f)
        live = torch.from_numpy(live_np)
        T_out[pid[live]] = Tf[live]
        T_err[pid[live]] = (Tf[:, None] * rel_f)[:, 0][live]
        a1 = E(alpha, e_a) * T
        a1 = E(a1.v * incf, a1.e * incf)
        # ---- the back-to-front acc recurrences: channel values f [npix, n] and their upstream gradients ----
        feats = [rgb[ids, k][None, :].expand_as(alpha) for k in range(3)]
        gs = [gpix[k, pid][:, None] for k in range(3)]
        if has_aux:
            feats += [depth[ids][None, :].expand_as(alpha), flows[ids, 0][None, :].expand_as(alpha),
                      flows[ids, 1][None, :].expand_as(alpha), torch.ones_like(alpha)]
            gs += [aux[0][0, pid][:, None], aux[1][0, pid][:, None], aux[1][1, pid][:, None], aux[2][0, pid][:, None]]
        wT = alpha * Tb                                       # float64 blend weights
        Tn = Tb * one_m                                       # T after each contributor
        terms = []
        for f, g in zip(feats, gs):
            s = f * wT
            behind = torch.flip(torch.cumsum(torch.flip(s, [1]), 1), [1]) - s
            acc = torch.where(inc, behind / Tn, torch.zeros_like(s))
            d = f - acc
            acc_new = acc + alpha * d
            local = torch.where(inc, d.abs() * e_a + 3 * U * ((alpha * f).abs() + acc.abs()) + U * acc_new.abs(),
                                torch.zeros_like(s))
            e_acc = torch.flip(torch.cumsum(torch.flip(local, [1]), 1), [1]) - local
            terms.append(E(d, e_acc + U * d.abs()) * g)
        D = esum(terms)
        D = E(D.v, D.e + U * D.v.abs())
        bgdot = esum([E(bgp[k, pid][:, None], bg_err[k, pid][:, None]) * gs[k] for k in range(3)])
        tb = -(TfE * bgdot)
        rom = E(1.0 / one_m, ((U * one_m + e_a) / one_m ** 2 + RCP / one_m))
        dLda = D * T + tb * rom
        dLda = E(dLda.v * incf, dLda.e * incf)
        GE = E(G, eG)
        w = GE * dLda
        # ---- kernel structure: per (warp, Gaussian) tensor-core sums, re-centred on the mean ----
        # pixel index = 16 * ly + lx; warp (ly // 4, lx // 8), MMA row s = ly % 4, k-lane = lx % 8
        def warp_view(x):
            return x.reshape(4, 4, 2, 8, n).permute(1, 3, 0, 2, 4)          # [s, lane, wy, wx, n]
        uu, vv = warp_view(u.expand(256, n)), warp_view(v.expand(256, n))
        wv, we = warp_view(w.v), warp_view(w.e)
        monos = [torch.ones_like(uu), uu, vv, uu * uu, uu * vv, vv * vv]
        M = []
        for mono in monos:
            tv = wv * mono
            val = tv.sum((0, 1))
            err = (we * mono.abs()).sum((0, 1)) + SPLIT * tv.abs().sum((0, 1)) + _chain_err(tv)
            M.append(E(val, err))
        Xw = warp_view(X.expand(256, n))[0, 0]
        Yw = warp_view(Y.expand(256, n))[0, 0]
        XE, YE = E(Xw, U * Xw.abs()), E(Yw, U * Yw.abs())
        W10 = XE * M[0] - M[1]
        W01 = YE * M[0] - M[2]
        W20 = XE * W10 - (XE * M[1] - M[3])
        W11 = YE * W10 - (XE * M[2] - M[4])
        W02 = YE * W01 - (YE * M[2] - M[5])
        parts = [M[0], W10, W01, W20, W11, W02]
        a1v, a1e = warp_view(a1.v), warp_view(a1.e)
        col_g = gs[:3] + ([gs[3], gs[4], gs[5]] if has_aux else [])
        for g in col_g:
            gw = warp_view(g.expand(256, n))
            tv = a1v * gw
            val = tv.sum((0, 1))
            err = (a1e * gw.abs()).sum((0, 1)) + 2 * SPLIT * tv.abs().sum((0, 1)) + (1 + 2.0 ** -10) * _chain_err(tv) \
                + U * val.abs()
            parts.append(E(val, err))
        while len(parts) < 12:
            parts.append(E(torch.zeros_like(M[0].v)))
        rows = ids[None, None, :].expand(4, 2, n).reshape(-1)
        kern.add(rows, torch.stack([p.v.reshape(-1) for p in parts], 1), torch.stack([p.e.reshape(-1) for p in parts], 1))
        # ---- per-pair structure (the reference's arithmetic) ----
        dxE, dyE = E(dx, U * dx.abs()), E(dy, U * dy.abs())
        dLdG = dLda * o
        gdx, gdy = GE * dxE, GE * dyE
        mxg = dLdG * (-(gdx * A) - gdy * B) * (0.5 * W)
        myg = dLdG * (-(gdy * C) - gdx * B) * (0.5 * H)
        pt = [mxg, myg, None, (gdx * dxE) * dLdG * -0.5, (gdx * dyE) * dLdG * -0.5, (gdy * dyE) * dLdG * -0.5, GE * dLda]
        pt += [a1 * g for g in gs[:3]]
        pt[2] = a1 * gs[3] if has_aux else E(torch.zeros_like(alpha))
        pt += [a1 * gs[4], a1 * gs[5]] if has_aux else [E(torch.zeros_like(alpha))] * 2
        sel = inc.reshape(-1)
        prow = ids[None, :].expand(256, n).reshape(-1)[sel]
        pair.add(prow, torch.stack([p.v.reshape(-1)[sel] for p in pt], 1), torch.stack([p.e.reshape(-1)[sel] for p in pt], 1))
    # ---- geom_bwd_body's map of the moment sums, and the per-row results ----
    k = kern.E()
    kc = lambda i: E(k.v[:, i], k.e[:, i])
    A, B, C, o = (E(co[:, i]) for i in range(4))
    W00, W10, W01, W20, W11, W02 = (kc(i) for i in range(6))
    kx = -0.5 * float(W) * o * (A * W10 + B * W01)
    ky = -0.5 * float(H) * o * (C * W01 + B * W10)
    hs = o * -0.5
    kmap = [kx, ky, kc(9), hs * W20, hs * W11, hs * W02, W00, kc(6), kc(7), kc(8), kc(10), kc(11)]
    pr = pair.E()
    res = {}
    names = [("dL_dmeans2D", [0, 1, 2]), ("dL_dconic", [3, 4, 5]), ("dL_dopacity", [6]), ("dL_dcolors", [7, 8, 9]),
             ("dL_dflows", [10, 11])]
    for name, idx in names:
        v = pr.v[:, idx]
        e = torch.maximum(pr.e[:, idx], torch.stack([kmap[i].e for i in idx], 1))
        res[name] = E(v, e)
        res[name + "@kernel"] = torch.stack([kmap[i].v for i in idx], 1)
    res["T_final"] = E(T_out, T_err)
    return res


def marginal(sc, st, prefilter_var):
    """the temporal marginal of every row as gauss_f64 states it (an E on the CPU) and the rows within 1e-5 of its
    0.05 cut; None for scenes whose blended opacity carries no marginal gradient (3D, non-rot 4D)"""
    import gauss_f64 as G
    if sc.gaussian_dim != 4 or not sc.rot_4d:
        return None, None
    P = sc.P
    mod = G.f32(st["scale_modifier"])
    s = [E(mod) * G.col(sc.scales.cpu(), i) for i in range(3)] + [E(mod) * G.col(sc.scales_t.cpu(), 0)]
    zero = E(torch.zeros(P, dtype=F64))
    r = G.chain_rot4d(s, [G.col(sc.rotations.cpu(), i) for i in range(4)], [G.col(sc.rotations_r.cpu(), i) for i in range(4)],
                      G.col(sc.ts.cpu(), 0), E(sc.opacities.reshape(-1).cpu().double()), st["timestamp"], prefilter_var,
                      [zero] * 6, [zero] * 3, zero)
    m = r["marginal"]
    return m, (m.v / G.CUT - 1.0).abs() <= 1e-5


def opacity(res, marginal=None, near_cut=None):
    """dL_dopacity as the backward returns it: the blend sum, times the temporal marginal (an E) for rot-4D rows.
    Returns (E [P,1], rows to skip: within 1e-5 of the marginal's 0.05 cut)"""
    d = res["dL_dopacity"]
    if marginal is None:
        return d, torch.zeros(d.v.shape[0], dtype=torch.bool)
    m = E(marginal.v[:, None], marginal.e[:, None])
    return d * m, near_cut


def compare(name, got, want, rows):
    """Every element of got [P, k] on rows within K err + TINY of want (E [P, k]); returns worst err / bar"""
    g = torch.as_tensor(np.asarray(got, np.float64)).reshape(want.v.shape).to(F64)
    err = (g - want.v).abs()[rows]
    bar = (K * want.e + TINY)[rows]
    if err.numel() == 0:
        return 0.0
    assert torch.isfinite(g[rows]).all(), (name, "non-finite")
    ratio = err / bar
    worst = float(ratio.max())
    if worst > 1.0:
        r, j = torch.nonzero(ratio > 1.0)[0].tolist()
        idx = int(torch.nonzero(rows).reshape(-1)[r])
        raise AssertionError("%s: %d elements beyond K err + tiny (worst err/bar %.3g); first at row %d, element %d: got %r, "
                             "float64 %r, error bound %.3g" % (name, int((ratio > 1).sum()), worst, idx, j,
                                                               float(g[idx, j]), float(want.v[idx, j]),
                                                               float(want.e[idx, j])))
    return worst


OUTPUTS = ("dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors", "dL_dflows")


def check(label, res, got, rendered, skip_opacity=None, marginal=None):
    """got: name -> [P, k] array of what the backward returned (dL_dconic as x, y, w).  rendered [P] bool.  Every element
    of every rendered row within K err + TINY; every other row exactly 0.  Returns name -> worst err/bar."""
    rendered = torch.as_tensor(np.asarray(rendered, bool))
    worst = {}
    for name in OUTPUTS:
        if name not in got or got[name] is None:
            continue
        want = res[name]
        rows = rendered.clone()
        if name == "dL_dopacity":
            want, near = opacity(res, marginal, skip_opacity)
            rows &= ~near
        worst[name] = compare("%s %s" % (label, name), got[name], want, rows)
        g = np.asarray(got[name]).reshape(rendered.shape[0], -1)[~rendered.numpy()]
        assert int(np.count_nonzero(g)) == 0, (label, name, "non-zero on a row the forward did not render")
    return worst


# ---- scenes at the blend backward's own edges (3D Gaussians, so that they run through every entry) --------------------
def edge_scene(name):
    """(cfg, cam, sc, st) of one scene; edge_reached asserts its edge on the forward's state:
      stack   3D, 200 Gaussians of opacity 0.95-0.989 and screen sigma 4-9 px stacked on the image centre: pixels that
              terminate by T < 1e-4 and pixels that do not (the backward recovers T from final_T by 1 / (1 - alpha));
      tail    3D, 40 Gaussians of sigma 3-8 px over a 128x64 image: per-warp column counts covering 1..7 mod 8 (the
              flush of a partial tile at the end of each warp's walk);
      far     3D, one Gaussian of screen sigma 250 px centred 300 px left of and above the image, over 60 small ones:
              contributing means hundreds of pixels from the warp rectangle (the raw moments' re-centring), under
              random-sign upstream gradients whose sum cancels;
      ragged  3D, a 17x5 image, a multiple of neither the 16x16 tile nor the 8x4 warp footprint."""
    import regimes
    from fdgs import synth
    seed = {"stack": 9401, "tail": 9402, "far": 9403, "ragged": 9404}[name]
    g = torch.Generator().manual_seed(seed)
    W, H = {"stack": (64, 48), "tail": (128, 64), "far": (96, 64), "ragged": (17, 5)}[name]
    cam = synth.make_camera(W, H)
    kw = dict(gaussian_dim=3, rot_4d=False)
    if name == "stack":
        sc = synth.make_scene(200, cam, seed, zmin=4.0, zmax=8.0, frustum=0.2, opacity_lo=0.95, opacity_hi=0.989, **kw)
        lo, hi = 4.0, 9.0
    elif name == "tail":
        sc = synth.make_scene(40, cam, seed, frustum=1.0, opacity_lo=0.3, opacity_hi=0.9, **kw)
        lo, hi = 3.0, 8.0
    elif name == "far":
        sc = synth.make_scene(61, cam, seed, frustum=1.0, **kw)
        lo, hi = 1.0, 3.0
    else:
        sc = synth.make_scene(120, cam, seed, frustum=1.1, **kw)
        lo, hi = 1.0, 4.0
    z = sc.means3D[:, 2]
    sc.scales = (regimes._px_world(cam, z)[:, None] * (lo + (hi - lo) * torch.rand(sc.P, 3, generator=g))).contiguous()
    if name == "far":
        z0 = float(z[0])
        P00, P11 = float(cam.full_proj_transform[0, 0]), float(cam.full_proj_transform[1, 1])
        sc.means3D[0, 0] = ((2 * -300.0 + 1) / W - 1.0) * (z0 + 1e-7) / P00
        sc.means3D[0, 1] = ((2 * -300.0 + 1) / H - 1.0) * (z0 + 1e-7) / P11
        sc.scales[0] = 250.0 * regimes._px_world(cam, z[0])
        sc.opacities[0] = 0.9
    return regimes._finish(name, dict(W=W, H=H, seed=seed), cam, sc, bg=(0.2, 0.5, 0.1))


EDGE_SCENES = ["blend:" + k for k in ("stack", "tail", "far", "ragged")]
_cache = {}


def build_case(case, device="cpu"):
    """(cfg, cam, sc, st, prefilter_var) of a gauss_f64 case or 'blend:<edge_scene>'"""
    import gauss_f64 as G
    if not case.startswith("blend:"):
        return G.build_case(case, device=device)
    from fdgs import synth
    if case not in _cache:
        _cache[case] = edge_scene(case[6:])
    cfg, cam, sc, st = _cache[case]
    if device != "cpu":
        sc = sc.to(device)
        st = synth.raster_settings(cam, sc, bg=torch.tensor(cfg["bg"]), device=device)
    return cfg, cam, sc, st, -1.0


def edge_reached(case, st, dec):
    """each edge scene reaches its edge in the forward's state st (decide's stats); also the regime scenes that carry
    one: `huge` (means far from the warp rectangle) and `needle` (instances past the exact flag's bound 128)"""
    s = dec["stats"]
    if case == "blend:stack":
        assert s["terminated"] > 0 and s["open"] > 0, ("stack: terminating and open pixels", s)
    elif case == "blend:tail":
        assert set(range(1, 8)) <= set(s["tail_mods"]), ("tail: column counts mod 8", s["tail_mods"])
    elif case in ("blend:far", "regime:huge"):
        assert s["far_max"] >= 200.0, ("far: offset from the warp rectangle", s["far_max"])
    elif case == "regime:needle":
        assert s["flag_max"] >= 128.0, ("needle: the exact flag", s["flag_max"])
    elif case == "blend:ragged":
        assert st["W"] % 8 and st["H"] % 4
