"""Float64 restatement of the per-Gaussian backward (preprocess_bwd.cu: sh_bwd_body, and geom_bwd_body from the
covariance chain on) with a first-order bound on the error an fp32 evaluation of the same expressions may carry.

The inputs are what the backward itself consumed, read back from what it returned, so no upstream gradient has to be
re-derived from the blend (whose atomics make it differ from run to run): dL_dcov3D and dL_dmeans3D are the values the
chain started from (the latter including the SH direction part), dL_dopacity / marginal is the blend's opacity
gradient, dL_dcolors with the forward's clamp bits feeds the SH backward, and the SH direction is the shifted mean the
forward returned minus the camera position.  dL_dmeans3D itself is checked whole: its EWA part restated from the
blend gradients geom_bwd_body converted and wrote back (dL_dmeans2D, dL_dconic), plus the SH direction part.

Every value is an E: the float64 value of the expression and a bound on |fp32 result - float64 value|.  Each
operation adds the propagated input errors and U |result| for its own rounding (U = 2^-24); sums of products use the
order-free bound (n - 1) U sum |terms|, so any association or FMA contraction the fp32 code chose is covered.  A
kernel value passes when |ours - value| <= K err + TINY: cancellation, 1/cov_t^2 and needles widen exactly the rows
that need it.  TEST INFRASTRUCTURE."""
import math

import numpy as np
import torch

U = 2.0 ** -24
K = 4.0           # the one slack factor of every check (the bound is first order; intrinsics are a few ulp)
TINY = 1e-30      # absolute floor: exact zeros stay exact, denormal noise passes
CUT = 0.05        # temporal marginal cut (forward.cu:333 / preprocess_fwd.cu)
MY_PI = 3.14159265
f32 = lambda x: float(np.float32(x))
C0 = f32(0.28209479177387814)
C1 = f32(0.4886025119029199)
C2 = [f32(c) for c in (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792,
                       0.5462742152960396)]
C3 = [f32(c) for c in (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154,
                       -0.4570457994644658, 1.445305721320277, -0.5900435899266435)]


class E:
    """float64 value v with error bound e of the fp32 evaluation"""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = v if torch.is_tensor(v) else torch.tensor(float(v), dtype=torch.float64)
        self.e = torch.zeros_like(self.v) if e is None else e

    @staticmethod
    def lift(x):
        return x if isinstance(x, E) else E(x)   # python constants are exact fp32 values here

    def __add__(a, b):
        b = E.lift(b)
        v = a.v + b.v
        return E(v, a.e + b.e + U * v.abs())

    __radd__ = __add__

    def __sub__(a, b):
        b = E.lift(b)
        v = a.v - b.v
        return E(v, a.e + b.e + U * v.abs())

    def __rsub__(a, b):
        return E.lift(b) - a

    def __neg__(a):
        return E(-a.v, a.e)

    def __mul__(a, b):
        b = E.lift(b)
        v = a.v * b.v
        return E(v, a.e * b.v.abs() + b.e * a.v.abs() + a.e * b.e + U * v.abs())

    __rmul__ = __mul__

    def __truediv__(a, b):
        b = E.lift(b)
        v = a.v / b.v
        lo = (b.v.abs() - b.e).clamp_min(1e-300)
        return E(v, (a.e + v.abs() * b.e) / lo + U * v.abs())

    def __rtruediv__(a, b):
        return E.lift(b) / a

    def sqrt(a):
        v = a.v.sqrt()
        lo = (a.v - a.e).clamp_min(0.0).sqrt()
        return E(v, a.e / (v + lo).clamp_min(1e-300) + U * v.abs())

    def exp(a, ulps=2.0):
        """expf: `ulps` of its own; __expf (ex2.approx of x log2 e) passes ulps=None: 2 ulp + the rounding of x log2 e"""
        v = a.v.exp()
        own = (2.0 + 2.0 * a.v.abs()) if ulps is None else ulps
        return E(v, v * torch.expm1(a.e) + own * U * v)

    def f32(a):
        """a double-precision island rounded to float"""
        return E(a.v, a.e + U * a.v.abs())


def esum(terms):
    """sum in any order: sum of the terms' errors + (n - 1) U sum |terms|"""
    terms = [t for t in terms if t is not None]
    v = sum(t.v for t in terms)
    a = sum(t.v.abs() for t in terms)
    return E(v, sum(t.e for t in terms) + (len(terms) - 1) * U * a)


def col(x, i):
    return E(x[:, i].double())


def stack(es, dim=-1):
    return E(torch.stack([e.v for e in es], dim), torch.stack([e.e for e in es], dim))


# ---- 4D covariance chain (preprocess_bwd.cu geom_bwd_body, rot_4d branch) --------------------------------------------
def _mat4(A, B):
    """glm (A*B)[c][r] = sum_k A[k][r] B[c][k]"""
    return [[esum([A[k][r] * B[c][k] for k in range(4)]) for r in range(4)] for c in range(4)]


def _ml_mr(q, p):
    a, b, c, d = q
    pp, qq, r, s = p
    Ml = [[a, b, -c, d], [-b, a, d, c], [c, -d, a, b], [-d, -c, -b, a]]
    Mr = [[pp, qq, -r, -s], [-qq, pp, s, -r], [r, -s, pp, -qq], [s, r, qq, pp]]
    return Ml, Mr


def chain_rot4d(sc, rot, rotr, t, opac, timestamp, prefilter_var, g_cov, g_mean, dopm):
    """sc: 4 E (modified scales); rot, rotr: 4 E each (normalised quaternions); t, opac: E; g_cov: 6 E (dL_dcov3D);
    g_mean: 3 E (dL_dmeans3D, total); dopm: E, the blend's opacity gradient times the marginal (what the backward
    returns as dL_dopacity).  Returns the chain's gradients and the marginal."""
    dt = E(f32(timestamp)) - t
    Ml, Mr = _ml_mr(rot, rotr)
    R = _mat4(Mr, Ml)
    M = [[sc[r] * R[c][r] for r in range(4)] for c in range(4)]
    cd = lambda i, j: esum([M[i][k] * M[j][k] for k in range(4)])
    cov_t = cd(3, 3)
    c12 = [cd(3, 0), cd(3, 1), cd(3, 2)]
    ctp = cov_t + f32(prefilter_var) if prefilter_var > 0 else cov_t
    arg = E((dt.v * -0.5) * dt.v / ctp.v, (dt.v.abs() * dt.e + 0.5 * dt.v * dt.v * ctp.e / ctp.v) / ctp.v)
    marginal = arg.f32().exp(ulps=None)
    dop = dopm / marginal
    d = g_cov
    dc12 = [-esum([d[0] * c12[0], d[1] * c12[1] * 0.5, d[2] * c12[2] * 0.5]) * 2.0 / cov_t,
            -esum([d[1] * c12[0] * 0.5, d[3] * c12[1], d[4] * c12[2] * 0.5]) * 2.0 / cov_t,
            -esum([d[2] * c12[0] * 0.5, d[4] * c12[1] * 0.5, d[5] * c12[2]]) * 2.0 / cov_t]
    dcovt = esum([c12[0] * c12[0] * d[0], c12[0] * c12[1] * d[1], c12[0] * c12[2] * d[2], c12[1] * c12[1] * d[3],
                  c12[1] * c12[2] * d[4], c12[2] * c12[2] * d[5]]) / (cov_t * cov_t)
    dmarg = dop * opac
    dcovt = dcovt + marginal * dt * dt / 2.0 / (ctp * ctp) * dmarg
    dL_dt = dmarg * (marginal * dt / ctp)
    dc12 = [dc12[i] + g_mean[i] / cov_t * dt for i in range(3)]
    ddot = esum([g_mean[i] * c12[i] for i in range(3)])
    dcovt = dcovt + (-ddot) / (cov_t * cov_t) * dt
    dL_dt = dL_dt + (-ddot) / cov_t
    # cov4_bwd (fdgs_common.cuh)
    h = lambda x: x * 0.5
    dS = [[d[0], h(d[1]), h(d[2]), h(dc12[0])], [h(d[1]), d[3], h(d[4]), h(dc12[1])],
          [h(d[2]), h(d[4]), d[5], h(dc12[2])], [h(dc12[0]), h(dc12[1]), h(dc12[2]), dcovt]]
    dM = _mat4([[m * 2.0 for m in row] for row in M], dS)
    gs = [esum([R[c][i] * dM[c][i] for c in range(4)]) for i in range(4)]
    N = [[sc[i] * dM[c][i] for c in range(4)] for i in range(4)]
    X, Y = _mat4(N, Mr), _mat4(Ml, N)
    g_rot = [esum([X[0][0], X[1][1], X[2][2], X[3][3]]), esum([-X[0][1], X[1][0], -X[2][3], X[3][2]]),
             esum([X[0][2], -X[1][3], -X[2][0], X[3][1]]), esum([-X[0][3], -X[1][2], X[2][1], X[3][0]])]
    g_rotr = [esum([Y[0][0], Y[1][1], Y[2][2], Y[3][3]]), esum([-Y[0][1], Y[1][0], Y[2][3], -Y[3][2]]),
              esum([Y[0][2], Y[1][3], -Y[2][0], -Y[3][1]]), esum([Y[0][3], -Y[1][2], Y[2][1], -Y[3][0]])]
    return dict(scales=gs[:3], scale_t=gs[3], rot=g_rot, rot_r=g_rotr, dt=dL_dt, marginal=marginal)


def chain_3d(sc, q, g_cov):
    """3D and non-rot 4D branch (quirk 5: no marginal gradient, no dL_dts / dL_dscale_t from it).  sc: 3 E; q: 4 E"""
    r, x, y, z = q
    R = [[1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - r * z), 2.0 * (x * z + r * y)],
         [2.0 * (x * y + r * z), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - r * x)],
         [2.0 * (x * z - r * y), 2.0 * (y * z + r * x), 1.0 - 2.0 * (x * x + y * y)]]
    M2 = [[2.0 * sc[rr] * R[c][rr] for rr in range(3)] for c in range(3)]
    d = g_cov
    dS = [[d[0], 0.5 * d[1], 0.5 * d[2]], [0.5 * d[1], d[3], 0.5 * d[4]], [0.5 * d[2], 0.5 * d[4], d[5]]]
    dM = [[esum([M2[k][rr] * dS[c][k] for k in range(3)]) for rr in range(3)] for c in range(3)]
    gs = [esum([R[c][i] * dM[c][i] for c in range(3)]) for i in range(3)]
    Nt = [[sc[i] * dM[c][i] for c in range(3)] for i in range(3)]
    g = [esum([2.0 * z * (Nt[0][1] - Nt[1][0]), 2.0 * y * (Nt[2][0] - Nt[0][2]), 2.0 * x * (Nt[1][2] - Nt[2][1])]),
         esum([2.0 * y * (Nt[1][0] + Nt[0][1]), 2.0 * z * (Nt[2][0] + Nt[0][2]), 2.0 * r * (Nt[1][2] - Nt[2][1]),
               -(4.0 * x * (Nt[2][2] + Nt[1][1]))]),
         esum([2.0 * x * (Nt[1][0] + Nt[0][1]), 2.0 * r * (Nt[2][0] - Nt[0][2]), 2.0 * z * (Nt[1][2] + Nt[2][1]),
               -(4.0 * y * (Nt[2][2] + Nt[0][0]))]),
         esum([2.0 * r * (Nt[0][1] - Nt[1][0]), 2.0 * x * (Nt[2][0] + Nt[0][2]), 2.0 * y * (Nt[1][2] + Nt[2][1]),
               -(4.0 * z * (Nt[1][1] + Nt[0][0]))])]
    return dict(scales=gs, rot=g)


# ---- raw-parameter activations (exp, F.normalize, sigmoid) ------------------------------------------------------------
def normalize_bwd(q, g):
    """act_normalize_bwd: gradient w.r.t. the raw quaternion q (4 E) given g w.r.t. the normalised one"""
    n = esum([q[0] * q[0], q[2] * q[2], q[1] * q[1], q[3] * q[3]]).sqrt()
    inv = 1.0 / n
    dot = esum([g[i] * q[i] for i in range(4)])
    coef = -dot * inv * inv / n
    return [g[i] * inv + coef * q[i] for i in range(4)]


# ---- SH backward (sh_bwd_body / sh_row_inplace) -----------------------------------------------------------------------
def sh_basis(x, y, z, deg):
    """the 16 basis values as E (None: identically zero), fp32 constants, the kernel's expressions"""
    l = [E(C0)] + [None] * 15
    if deg > 0:
        l[1], l[2], l[3] = -C1 * y, C1 * z, -C1 * x
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        l[4], l[5], l[6] = C2[0] * xy, C2[1] * yz, C2[2] * (2.0 * zz - xx - yy)
        l[7], l[8] = C2[3] * xz, C2[4] * (xx - yy)
        if deg > 2:
            l[9] = C3[0] * y * (3.0 * xx - yy)
            l[10] = C3[1] * xy * z
            l[11] = C3[2] * y * (4.0 * zz - xx - yy)
            l[12] = C3[3] * z * (2.0 * zz - 3.0 * xx - 3.0 * yy)
            l[13] = C3[4] * x * (4.0 * zz - xx - yy)
            l[14] = C3[5] * z * (xx - yy)
            l[15] = C3[6] * x * (xx - 3.0 * yy)
    return l


def sh_basis_deriv(x, y, z, deg):
    """d basis / d (x, y, z) of the normalised direction, three lists of 16 E (None: identically zero)"""
    dx, dy, dz = [None] * 16, [None] * 16, [None] * 16
    if deg > 0:
        dy[1], dz[2], dx[3] = E(-C1), E(C1), E(-C1)
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        dx[4], dy[4] = C2[0] * y, C2[0] * x
        dy[5], dz[5] = C2[1] * z, C2[1] * y
        dx[6], dy[6], dz[6] = -2.0 * C2[2] * x, -2.0 * C2[2] * y, 4.0 * C2[2] * z
        dx[7], dz[7] = C2[3] * z, C2[3] * x
        dx[8], dy[8] = 2.0 * C2[4] * x, -2.0 * C2[4] * y
        if deg > 2:
            dx[9], dy[9] = C3[0] * y * 6.0 * x, C3[0] * (3.0 * xx - 3.0 * yy)
            dx[10], dy[10], dz[10] = C3[1] * yz, C3[1] * xz, C3[1] * xy
            dx[11], dy[11], dz[11] = -C3[2] * y * 2.0 * x, C3[2] * (4.0 * zz - xx - 3.0 * yy), C3[2] * y * 8.0 * z
            dx[12], dy[12] = -C3[3] * z * 6.0 * x, -C3[3] * z * 6.0 * y
            dz[12] = C3[3] * (6.0 * zz - 3.0 * xx - 3.0 * yy)
            dx[13], dy[13], dz[13] = C3[4] * (4.0 * zz - 3.0 * xx - yy), -C3[4] * x * 2.0 * y, C3[4] * x * 8.0 * z
            dx[14], dy[14], dz[14] = C3[5] * z * 2.0 * x, -C3[5] * z * 2.0 * y, C3[5] * (xx - yy)
            dx[15], dy[15] = C3[6] * (3.0 * xx - 3.0 * yy), -C3[6] * x * 6.0 * y
    return dx, dy, dz


def dnormvdv(v, dv):
    """auxiliary.h dnormvdv: the gradient through v / |v|"""
    sum2 = esum([v[0] * v[0], v[1] * v[1], v[2] * v[2]])
    inv = 1.0 / (sum2 * sum2 * sum2).sqrt()
    return [esum([(sum2 - v[i] * v[i]) * dv[i]] + [-(v[j] * v[i] * dv[j]) for j in range(3) if j != i]) * inv
            for i in range(3)]


def time_blocks(ts, timestamp, duration, deg, deg_t, sh4d):
    """temporal weight tw and the reference's derivative dtw per 16-coefficient block (double angle, cast to float)"""
    nblk = (3 if deg_t > 1 else 2) if (sh4d and deg > 2 and deg_t > 0) else 1
    dir_t = ts - E(f32(timestamp))
    tw, dtw = [E(1.0)], [E(0.0)]
    for n in range(1, nblk):
        k = 2 * MY_PI * n / f32(duration)
        w = dir_t.v * k
        we = dir_t.e * k
        tw.append(E(torch.cos(w), torch.sin(w).abs() * we + we * we + U * torch.cos(w).abs()))
        dv = torch.sin(w) * k
        dtw.append(E(dv, k * (torch.cos(w).abs() * we + we * we) + U * dv.abs()))
    return nblk, tw, dtw


def sh_backward(shs, dcol, clamped, means, campos, ts, timestamp, duration, deg, deg_t, sh4d):
    """shs [P,M,3]; dcol [P,3] dL_dcolors; clamped [P,3] bool; means [P,3] the SHIFTED means (SURVEY quirk 1); campos [3];
    ts [P] (None in 3D).  Returns (dL_dsh as E [P,M,3], the SH part of dL_dts as E [P], the SH part of dL_dmeans3D as
    3 E [P]: the basis derivatives weighted by the temporal weights, through dnormvdv)."""
    P, M = shs.shape[0], shs.shape[1]
    dev = shs.device
    d = [col(means, i) - float(campos[i]) for i in range(3)]
    ln = esum([d[0] * d[0], d[1] * d[1], d[2] * d[2]]).sqrt()
    x, y, z = (d[i] / ln for i in range(3))
    l = sh_basis(x, y, z, deg)
    dl = sh_basis_deriv(x, y, z, deg)
    drgb = [E(torch.where(clamped[:, c], torch.zeros((), dtype=torch.float64, device=dev), dcol[:, c].double()))
            for c in range(3)]
    nblk, tw, dtw = time_blocks(E(ts.double()) if ts is not None else E(torch.zeros(P, dtype=torch.float64, device=dev)),
                                timestamp, duration, deg, deg_t, sh4d)
    ncoef = (deg + 1) ** 2
    v = torch.zeros(P, M, 3, dtype=torch.float64, device=dev)
    e = torch.zeros_like(v)
    dtt = E(torch.zeros(P, dtype=torch.float64, device=dev))
    ddir = [[], [], []]
    for blk in range(nblk):
        if 16 * blk >= M:
            continue              # a block the row does not hold: the kernel skips it
        for k in range(ncoef):
            c = 16 * blk + k
            if c >= M:
                continue
            w = (l[0] if (sh4d and k == 1) else l[k]) if blk == 0 else tw[blk] * l[k]
            for ch in range(3):
                o = w * drgb[ch]
                v[:, c, ch], e[:, c, ch] = o.v, o.e
                shc = E(shs[:, c, ch].double())
                for a in range(3):
                    if dl[a][k] is not None:
                        ddir[a].append((dl[a][k] if blk == 0 else tw[blk] * dl[a][k]) * shc * drgb[ch])
        if blk > 0:
            sl = esum([l[k] * E(shs[:, 16 * blk + k, ch].double()) * drgb[ch]
                       for k in range(ncoef) if 16 * blk + k < M for ch in range(3)])
            dtt = dtw[blk] * sl       # overwrites: backward.cu:403
    zero = E(torch.zeros(P, dtype=torch.float64, device=dev))
    dm = dnormvdv(d, [esum(t) if t else zero for t in ddir])
    return E(v, e), (dtt if sh4d else zero), dm


# ---- EWA part of dL_dmeans3D (geom_bwd_body: computeCov2DCUDA and the projection) -------------------------------------
def ewa_consts(st, exact=False):
    """The camera constants of computeCov2DCUDA and the projection: the fp32 values the kernels compute (focal lengths
    W / (2 tan fov), the clamp limits 1.3 tan fov, the 0.3 low-pass and the 1e-7 guards), or with `exact` the float64
    values blend_f64 / camera_f64 use, so that a float64 restatement can be compared with their autograd to 1e-12."""
    H, W = np.float32(st["image_height"]), np.float32(st["image_width"])
    tanx, tany = np.float32(st["tanfovx"]), np.float32(st["tanfovy"])
    if exact:
        return dict(fx=float(W) / (2.0 * float(tanx)), fy=float(H) / (2.0 * float(tany)), limx=1.3 * float(tanx),
                    limy=1.3 * float(tany), lowpass=0.3, eps=1e-7)
    return dict(fx=float(W / (np.float32(2.0) * tanx)), fy=float(H / (np.float32(2.0) * tany)),
                limx=float(np.float32(1.3) * tanx), limy=float(np.float32(1.3) * tany), lowpass=f32(0.3),
                eps=f32(0.0000001))


def ewa_chain(means, cov3D, dmean2D, dconic, st, exact=False, flip=None):
    """computeCov2DCUDA and the projection's backward (geom_bwd_body) as E values, from the blend gradients in the form
    the reference's computeCov2DCUDA consumes: dmean2D [P,3] (x, y and the depth gradient), dconic [P,4] (0, 1, 3 used);
    means [P,3] the shifted means, cov3D [P,6] the forward's conditional covariances.  flip: None, or two [P] bool masks
    (x, y) of rows on which the frustum clamp takes the other branch (with a positive field of view only: a negative
    one clamps every row whatever the value).  Returns a dict of the intermediates: g (the EWA part of dL_dmeans3D, 3 E),
    near (rows whose view-space x/z or y/z lies within 1e-5 of the 1.3 tan(fov) clamp, where fp32 and float64 may take
    different branches), nx / ny, and the view-space point's gradient (vx, vy, vz; vz0 without the depth gradient dz),
    the Jacobian (j00, j11, j02, j12), dL/dT (dT0, dT1), the projection's m_w, mul1, mul2 and d2x, d2y."""
    V = [float(x) for x in st["viewmatrix"].reshape(-1).cpu()]
    Pm = [float(x) for x in st["projmatrix"].reshape(-1).cpu()]
    k = ewa_consts(st, exact)
    fx, fy, limx, limy = k["fx"], k["fy"], k["limx"], k["limy"]
    m = [col(means, i) for i in range(3)]
    c3 = [col(cov3D, i) for i in range(6)]
    row = lambda a, b, c, d: esum([m[0] * a, m[1] * b, m[2] * c, E(d)])
    tx0, ty0, tz = row(V[0], V[4], V[8], V[12]), row(V[1], V[5], V[9], V[13]), row(V[2], V[6], V[10], V[14])
    txtz, tytz = tx0 / tz, ty0 / tz

    def clamp(r, lim, f):
        """min(lim, max(-lim, r)) and the gradient mask (lim < 0 with a negative field of view: always clamped)"""
        v = torch.clamp(torch.clamp(r.v, min=-lim), max=lim)
        kept = v == r.v
        out = (r.v < -lim) | (r.v > lim)
        if f is not None and lim > 0:
            f = f.to(r.v.device)
            out = out ^ f
            one = torch.ones_like(r.v)
            v = torch.where(f, torch.where(out, torch.where(r.v < 0, -one, one) * lim, r.v), v)
            kept = torch.where(f, ~out, kept)
        return E(v, torch.where(kept, r.e, torch.zeros_like(r.e))), (~out).double(), \
            (r.v.abs() / abs(lim) - 1.0).abs() <= 1e-5

    cx, xgm, nx = clamp(txtz, limx, None if flip is None else flip[0])
    cy, ygm, ny = clamp(tytz, limy, None if flip is None else flip[1])
    tx, ty = cx * tz, cy * tz
    tz2 = tz * tz
    j00, j11 = fx / tz, fy / tz
    j02, j12 = (fx * -tx) / tz2, (fy * -ty) / tz2
    T00, T01, T02 = V[2] * j02 + V[0] * j00, V[6] * j02 + V[4] * j00, V[10] * j02 + V[8] * j00
    T10, T11, T12 = V[2] * j12 + V[1] * j11, V[6] * j12 + V[5] * j11, V[10] * j12 + V[9] * j11
    d3 = lambda a0, b0, a1, b1, a2, b2: esum([a0 * b0, a1 * b1, a2 * b2])
    X00, X01 = d3(T00, c3[0], T01, c3[1], T02, c3[2]), d3(T10, c3[0], T11, c3[1], T12, c3[2])
    X10, X11 = d3(T00, c3[1], T01, c3[3], T02, c3[4]), d3(T10, c3[1], T11, c3[3], T12, c3[4])
    X20, X21 = d3(T00, c3[2], T01, c3[4], T02, c3[5]), d3(T10, c3[2], T11, c3[4], T12, c3[5])
    A = d3(T00, X00, T01, X10, T02, X20) + k["lowpass"]
    B = d3(T00, X01, T01, X11, T02, X21)
    C = d3(T10, X01, T11, X11, T12, X21) + k["lowpass"]
    dcx, dcy, dcz = col(dconic, 0), col(dconic, 1), col(dconic, 3)
    denom = esum([A * C, -(B * B)])
    d2i = 1.0 / (denom * denom + k["eps"])
    dL_da = d2i * esum([-C * C * dcx, 2.0 * B * C * dcy, (denom - A * C) * dcz])
    dL_dc = d2i * esum([-A * A * dcz, 2.0 * A * B * dcy, (denom - A * C) * dcx])
    dL_db = d2i * 2.0 * esum([B * C * dcx, -((denom + 2.0 * B * B) * dcy), A * B * dcz])
    dT0 = [esum([2.0 * r0 * dL_da, r1 * dL_db]) for r0, r1 in ((X00, X01), (X10, X11), (X20, X21))]
    dT1 = [esum([2.0 * r1 * dL_dc, r0 * dL_db]) for r0, r1 in ((X00, X01), (X10, X11), (X20, X21))]
    dJ00 = esum([V[0] * dT0[0], V[4] * dT0[1], V[8] * dT0[2]])
    dJ02 = esum([V[2] * dT0[0], V[6] * dT0[1], V[10] * dT0[2]])
    dJ11 = esum([V[1] * dT1[0], V[5] * dT1[1], V[9] * dT1[2]])
    dJ12 = esum([V[2] * dT1[0], V[6] * dT1[1], V[10] * dT1[2]])
    tzi = 1.0 / tz
    t2 = tzi * tzi
    t3 = t2 * tzi
    vx = E(xgm) * (-fx * t2 * dJ02)
    vy = E(ygm) * (-fy * t2 * dJ12)
    vz0 = esum([-fx * t2 * dJ00, -(fy * t2 * dJ11), (2.0 * fx * tx) * t3 * dJ02, (2.0 * fy * ty) * t3 * dJ12])
    dz = col(dmean2D, 2)
    vz = vz0 + dz
    g = [esum([V[0] * vx, V[1] * vy, V[2] * vz]), esum([V[4] * vx, V[5] * vy, V[6] * vz]),
         esum([V[8] * vx, V[9] * vy, V[10] * vz])]
    m_w = 1.0 / (row(Pm[3], Pm[7], Pm[11], Pm[15]) + k["eps"])
    mul1 = row(Pm[0], Pm[4], Pm[8], Pm[12]) * m_w * m_w
    mul2 = row(Pm[1], Pm[5], Pm[9], Pm[13]) * m_w * m_w
    d2x, d2y = col(dmean2D, 0), col(dmean2D, 1)
    for i in range(3):
        g[i] = esum([g[i], (Pm[4 * i] * m_w - Pm[4 * i + 3] * mul1) * d2x, (Pm[4 * i + 1] * m_w - Pm[4 * i + 3] * mul2) * d2y])
    return dict(g=g, near=nx | ny, nx=nx, ny=ny, m=m, tx=tx, ty=ty, tz=tz, cx=cx, cy=cy, xgm=xgm, ygm=ygm, fx=fx, fy=fy,
                t2=t2, dJ02=dJ02, dJ12=dJ12, j00=j00, j11=j11, j02=j02, j12=j12, dT0=dT0, dT1=dT1, vx=vx, vy=vy, vz=vz,
                vz0=vz0, dz=dz, m_w=m_w, mul1=mul1, mul2=mul2, d2x=d2x, d2y=d2y)


def ewa_mean_grad(means, cov3D, dmean2D, dconic, st):
    """The part of dL_dmeans3D that does not come from the SH colour (ewa_chain).  Returns (3 E, rows whose view-space
    x/z or y/z lies within 1e-5 of the 1.3 tan(fov) clamp, where fp32 and float64 may take different branches)."""
    r = ewa_chain(means, cov3D, dmean2D, dconic, st)
    return r["g"], r["near"]


# ---- the whole per-Gaussian backward of one view ----------------------------------------------------------------------
def per_gaussian(sc, st, prefilter_var, out, clamped, means_out, raw=None, has_sh=True):
    """The float64 restatement of everything the per-Gaussian backward returns from the covariance chain on.

    sc: the activated parameters as fp32 tensors (means3D, ts, scales, scales_t, rotations, rotations_r, opacities, shs),
        with rot_4d / gaussian_dim / force_sh_3d / sh_degree(_t) / time_duration;
    st: raster settings (timestamp, campos, scale_modifier);
    out: dict of what the backward returned (dL_dcov3D, dL_dmeans3D, dL_dopacity, dL_dcolors) -- the chain's inputs --
         and the EWA part's inputs: dL_dmeans2D and dL_dconic as computeCov2DCUDA consumes them, and the forward's cov3D;
    clamped [P,3] bool: the forward's clamp bits; means_out [P,3]: the forward's shifted means;
    raw: None, or dict(log_scales, log_scales_t, rotations, rotations_r) of the raw entry (rotations un-normalised).

    Returns a dict name -> E over all rows (the rows the kernel does not render are not meaningful), plus 'marginal'
    (rot_4d), 'recovered' (rows whose opacity gradient could be recovered), 'near_cut' and 'near_clamp'."""
    P = sc.means3D.shape[0]
    dev = sc.means3D.device
    mod = f32(st["scale_modifier"])
    timestamp = st["timestamp"]
    sh4d = not (sc.gaussian_dim == 3 or sc.force_sh_3d)
    res = {}
    if has_sh:
        dsh, dts_sh, dm_sh = sh_backward(sc.shs, out["dL_dcolors"], clamped, means_out, st["campos"].cpu().double(),
                                  sc.ts[:, 0] if sc.gaussian_dim == 4 else None, timestamp, sc.time_duration,
                                  sc.sh_degree, sc.sh_degree_t, sh4d)
        res["dL_dsh"] = dsh
    else:
        dts_sh = E(torch.zeros(P, dtype=torch.float64, device=dev))
        dm_sh = [E(torch.zeros(P, dtype=torch.float64, device=dev))] * 3
    ewa, res["near_clamp"] = ewa_mean_grad(means_out, out["cov3D"], out["dL_dmeans2D"], out["dL_dconic"], st)
    res["dL_dmeans3D"] = [ewa[i] + dm_sh[i] for i in range(3)]
    g_cov = [col(out["dL_dcov3D"], i) for i in range(6)]
    zero = E(torch.zeros(P, dtype=torch.float64, device=dev))
    s = [E(mod) * col(sc.scales, i) for i in range(3)]
    dop_out = out["dL_dopacity"].reshape(-1).double()
    opac = E(sc.opacities.reshape(-1).double())
    recovered = torch.ones(P, dtype=torch.bool, device=dev)
    if raw is not None:
        # dL_dopacity came back as dop * marginal * (1 - o) * o; o = 1.0f leaves nothing to recover dop from
        o = opac
        den = (1.0 - o) * o
        recovered = den.v != 0
        dop = E(dop_out) / E(torch.where(recovered, den.v, torch.ones_like(den.v)), den.e)
    else:
        dop = E(dop_out)
    if sc.rot_4d:
        st4 = s + [E(mod) * col(sc.scales_t, 0)]
        q = [col(sc.rotations, i) for i in range(4)]
        qr = [col(sc.rotations_r, i) for i in range(4)]
        r = chain_rot4d(st4, q, qr, col(sc.ts, 0), opac, timestamp, prefilter_var, g_cov,
                        [col(out["dL_dmeans3D"], i) for i in range(3)], dop)
        res["dL_dscales"] = r["scales"]
        res["dL_dscales_t"] = [r["scale_t"]]
        res["dL_drot"], res["dL_drot_r"] = r["rot"], r["rot_r"]
        res["dL_dts"] = [dts_sh + r["dt"]]
        m = r["marginal"].v
        res["marginal"] = r["marginal"]
        # test_gpu_regimes.time_cut_rows, with the scale modifier and the prefilter variance the chain applies
        res["near_cut"] = (m / CUT - 1.0).abs() <= 1e-5
    else:
        r = chain_3d(s, [col(sc.rotations, i) for i in range(4)], g_cov)
        res["dL_dscales"], res["dL_drot"] = r["scales"], r["rot"]
        res["dL_dscales_t"] = [zero]
        res["dL_drot_r"] = [zero] * 4
        res["dL_dts"] = [dts_sh]
        res["near_cut"] = torch.zeros(P, dtype=torch.bool, device=dev)
    if raw is not None:
        res["dL_dscales"] = [res["dL_dscales"][i] * E(sc.scales[:, i].double()) for i in range(3)]
        if sc.gaussian_dim == 4:
            res["dL_dscales_t"] = [res["dL_dscales_t"][0] * E(sc.scales_t[:, 0].double())]
        res["dL_drot"] = normalize_bwd([col(raw["rotations"], i) for i in range(4)], res["dL_drot"])
        if sc.rot_4d:
            res["dL_drot_r"] = normalize_bwd([col(raw["rotations_r"], i) for i in range(4)], res["dL_drot_r"])
    res["recovered"] = recovered
    return res


def compare(name, got, want, rows):
    """Every element of `got` (tensor [P,...]) on `rows` within K err + TINY of `want` (E [P,...] or list of E [P]).
    Returns (worst |got - value| / bar, number of elements checked)."""
    if isinstance(want, list):
        want = stack(want, 1)
    g = got.reshape(want.v.shape).double().to(want.v.device)
    rows = rows.to(want.v.device)
    err = (g - want.v).abs()[rows]
    bar = (K * want.e + TINY)[rows]
    if err.numel() == 0:
        return 0.0, 0
    assert torch.isfinite(g[rows]).all(), (name, "non-finite")
    ratio = err / bar
    worst = float(ratio.max())
    if worst > 1.0:
        r, j = torch.nonzero(ratio.reshape(ratio.shape[0], -1) > 1.0)[0].tolist()
        idx = torch.nonzero(rows).reshape(-1)[r].item()
        at = lambda x: x[idx].reshape(-1)[j].item()
        raise AssertionError("%s: %d elements beyond K err + tiny (worst err/bar %.3g); first at row %d, element %d: "
                             "got %r, float64 %r, error bound %.3g" % (name, int((ratio > 1).sum()), worst, idx, j,
                                                                       at(g), at(want.v), at(want.e)))
    return worst, int(err.numel())


# ---- scenes at the edges of the per-Gaussian backward -----------------------------------------------------------------
def _near(n, g, axis):
    """unit quaternions within ~1e-3 of `axis` (identity: (1,0,0,0); 180 degrees about x: (0,1,0,0))"""
    q = torch.tensor(axis, dtype=torch.float32).expand(n, 4) + 1e-3 * torch.randn(n, 4, generator=g)
    return torch.nn.functional.normalize(q, dim=1).contiguous()


def edge_scene(name):
    """(cfg, cam, sc, st) of one edge scene, CPU tensors:
      scale_t  scales_t log-uniform in [1e-4, 10], timestamps within ~1 temporal sigma, a third of the right quaternions
               near the identity and a third near 180 degrees, a quarter of the left ones near the identity (so
               Sigma_tt ~ scale_t^2: the 1/cov_t^2 terms at their largest);
      clamp    the SH DC term drives exactly one colour channel negative on three rows of four (each channel in turn);
      p<N>[a]  N Gaussians (1, the SH kernel's CTA size +- 1, a multiple plus one of its shared-memory row slots), all
               in view, or with 'a' every other one behind the camera."""
    from fdgs import synth
    seed = {"scale_t": 9201, "clamp": 9202}.get(name, 9300 + len(name))
    if name.startswith("p"):
        alt = name.endswith("a")
        P = int(name[1:].rstrip("a"))
        cam = synth.make_camera(96, 64)
        sc = synth.make_scene(P, cam, seed + P, zmin=3.0, zmax=6.0, frustum=0.7, scale_t_mean=0.5)
        sc.ts[:] = cam.timestamp
        if alt:
            sc.means3D[1::2, 2] = -sc.means3D[1::2, 2]
        cfg = dict(W=96, H=64, seed=seed + P, P=P)
    else:
        cam = synth.make_camera(160, 112)
        g = torch.Generator().manual_seed(seed)
        sc = synth.make_scene(3000, cam, seed)
        P = sc.P
        if name == "scale_t":
            sc.scales_t = torch.exp(math.log(1e-4) + math.log(1e5) * torch.rand(P, 1, generator=g)).contiguous()
            third = torch.arange(P) % 3
            sc.rotations_r[third == 0] = _near(int((third == 0).sum()), g, (1.0, 0.0, 0.0, 0.0))
            sc.rotations_r[third == 1] = _near(int((third == 1).sum()), g, (0.0, 1.0, 0.0, 0.0))
            quarter = torch.arange(P) % 4 == 0
            sc.rotations[quarter] = _near(int(quarter.sum()), g, (1.0, 0.0, 0.0, 0.0))
            sc.ts = (cam.timestamp + sc.scales_t * torch.randn(P, 1, generator=g)).contiguous()
        elif name == "clamp":
            ch = torch.arange(P) % 4
            for c in range(3):
                sc.shs[ch == c, 0, c] = -2.5 / 0.28209479177387814
        else:
            raise KeyError(name)
        cfg = dict(W=160, H=112, seed=seed, P=P)
    st = synth.raster_settings(cam, sc)
    return cfg, cam, sc, st


EDGE_SCENES = ["scale_t", "clamp", "p1", "p127", "p129", "p385", "p127a", "p129a", "p385a"]


# ---- the check of one backward ------------------------------------------------------------------------------------------
CHECKED = ("dL_dsh", "dL_dmeans3D", "dL_dscales", "dL_dscales_t", "dL_drot", "dL_drot_r", "dL_dts")


def check_backward(label, sc, st, prefilter_var, out, clamped, means_out, vis, raw=None):
    """All of CHECKED on the rendered rows against the restatement, every row the backward did not render exactly zero.
    out: name -> what the backward returned (dL_dsh [P,M,3] whole, also for split rows), with dL_dconic and cov3D (see
    per_gaussian); clamped [P,3] bool;
    vis [P] bool: rows the backward rendered.  Returns name -> worst err / bar."""
    has_sh = out.get("dL_dsh") is not None and out["dL_dsh"].numel() > 0
    res = per_gaussian(sc, st, prefilter_var, out, clamped, means_out, raw=raw, has_sh=has_sh)
    vis = vis.to(res["near_cut"].device)
    keep = vis & ~res["near_cut"]
    chain_rows = keep & res["recovered"]
    worst = {}
    for name in CHECKED:
        if name not in res:
            continue
        rows = keep if name == "dL_dsh" else (keep & ~res["near_clamp"]) if name == "dL_dmeans3D" else chain_rows
        worst[name], _ = compare("%s %s" % (label, name), out[name], res[name], rows)
    unrendered = ~vis
    for name in CHECKED + ("dL_dopacity", "dL_dcov3D", "dL_dmeans3D", "dL_dcolors"):
        t = out.get(name)
        if t is None or t.numel() == 0:
            continue
        t = t.reshape(t.shape[0], -1)[unrendered.to(t.device)]
        assert int(torch.count_nonzero(t)) == 0, (label, name, "non-zero on a row the backward did not render")
    saturated = vis & ~res["recovered"]
    if bool(saturated.any()):
        d = out["dL_dopacity"].reshape(-1)[saturated.to(out["dL_dopacity"].device)]
        assert int(torch.count_nonzero(d)) == 0, (label, "dL_dopacity on a saturated-sigmoid row")
    print("%-34s rows %6d checked, %d near the temporal cut, %d near the frustum clamp (dL_dmeans3D unchecked), %d with a "
          "saturated sigmoid (chain unchecked); worst err/bar: %s"
          % (label, int(keep.sum()), int((vis & res["near_cut"]).sum()), int((keep & res["near_clamp"]).sum()),
             int(saturated.sum()),
             "  ".join("%s %.3f" % (k[4:], v) for k, v in worst.items())))
    return worst


# ---- the cases both tests run ---------------------------------------------------------------------------------------------
CASES = (["small", "dim3", "norot4d", "sh3d", "deg1", "deg1m4", "m16", "prefilter", "dur10", "smod05", "smod2", "rotcam",
          "n3v", "tiny", "flowbg", "negfov", "ragged"]
         + ["regime:" + k for k in ("time_edge", "needle", "huge", "opaque", "threshold")]
         + ["edge:" + k for k in EDGE_SCENES])


def build_case(case, device="cpu"):
    """(cfg, cam, sc, st, prefilter_var) of a helpers.CONFIGS name, 'regime:<regimes.SCENES>' or 'edge:<EDGE_SCENES>'"""
    import helpers
    import regimes
    if case.startswith("regime:"):
        cfg, cam, sc, st = regimes.build(case[7:], device=device)
    elif case.startswith("edge:"):
        cfg, cam, sc, st = edge_scene(case[5:])
        if device != "cpu":
            from fdgs import synth
            sc = sc.to(device)
            st = synth.raster_settings(cam, sc, device=device)
    else:
        cfg, cam, sc, st = helpers.build(case, device=device)
    return cfg, cam, sc, st, cfg.get("prefilter_var", -1.0)
