"""The camera gradient of the 3D rasterizer (precomputed colours and covariances) in float64: blend_f64's projection,
EWA splatting and blend, with the view and projection matrices as differentiable float64 tensors, so that autograd
gives dL/dviewmatrix and dL/dprojmatrix in the layout of the torch tensors the rasterizer takes (element [c][r] is the
gradient of element [c][r]).  The projection is blend_f64.project's arithmetic with the camera as an argument; the blend
is blend_f64.walk_tile.  Rows under the frustum clamp follow the textbook clamp here, not the reference's (whose
backward drops the clamp's depth term), so comparisons take scenes without such rows.
TEST INFRASTRUCTURE."""
import numpy as np
import torch

import blend_f64 as BF

F64 = torch.float64


def project(st, means3D, cov3D, viewmatrix, projmatrix):
    """blend_f64.project with viewmatrix / projmatrix ([4,4] float64 tensors in the rasterizer's layout) as inputs."""
    W, H = int(st["image_width"]), int(st["image_height"])
    view, proj = viewmatrix.t(), projmatrix.t()
    tanx = float(np.float32(st["tanfovx"]))
    tany = float(np.float32(st["tanfovy"]))
    fx, fy = W / (2.0 * tanx), H / (2.0 * tany)
    mh = torch.cat([means3D, torch.ones(means3D.shape[0], 1, dtype=F64)], 1)
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
                     torch.stack([z, fy / tz, -fy * ty / (tz * tz)], 1)], 1)
    Tm = J @ view[:3, :3]
    c = cov3D
    S = torch.stack([torch.stack([c[:, 0], c[:, 1], c[:, 2]], 1), torch.stack([c[:, 1], c[:, 3], c[:, 4]], 1),
                     torch.stack([c[:, 2], c[:, 4], c[:, 5]], 1)], 1)
    cov2 = Tm @ S @ Tm.transpose(1, 2)
    cx, cy, cz = BF._Conic.apply(cov2[:, 0, 0] + 0.3, cov2[:, 0, 1], cov2[:, 1, 1] + 0.3)
    return pix, ndc, depth, torch.stack([cx, cy, cz], 1), clamped


def loss(st, lists, t, grads, viewmatrix, projmatrix, means3D=None):
    """sum over the images of image * upstream gradient (blend_f64.render's blend over `lists`), with the camera given.
    t: the twin's float32 arrays (blend_f64.forward_backward); grads: float32 upstream images, None = no gradient.
    Returns (loss, the frustum-clamp mask, the ambiguous-pixel mask)."""
    W, H = int(st["image_width"]), int(st["image_height"])
    f = lambda k: torch.as_tensor(np.asarray(t[k], np.float32)).to(F64)
    m = f("means3D") if means3D is None else means3D
    pix, ndc, depth, conic, fclamp = project(st, m, f("cov3D"), viewmatrix, projmatrix)
    colors, opacity, flows = f("colors"), f("opacity").reshape(-1), f("flows")
    bg = torch.as_tensor(st["bg"]).detach().cpu().to(F64)
    ranges = np.asarray(lists["ranges"]).reshape(-1, 2).astype(np.int64)
    plist = torch.from_numpy(np.asarray(lists["point_list"]).astype(np.int64))
    gx = (W + 15) // 16
    feats = torch.cat([colors, depth[:, None], flows], 1)
    out = torch.zeros(H * W, 6, dtype=F64)
    T_img = torch.ones(H * W, dtype=F64)
    amb = np.zeros(H * W, bool)
    pieces, tpieces, pids = [], [], []
    for k in range(ranges.shape[0]):
        lo, hi = ranges[k]
        if hi <= lo:
            continue
        ids = plist[lo:hi]
        w, Tf, pid, rec = BF.walk_tile(pix, conic, opacity, ids, (k % gx) * 16, (k // gx) * 16, W, H)
        pieces.append(w @ feats[ids])
        tpieces.append(Tf)
        pids.append(pid)
        amb[pid.numpy()] = rec["ambiguous"]
    if pids:
        pid = torch.cat(pids)
        out = out.index_put((pid,), torch.cat(pieces))
        T_img = T_img.index_put((pid,), torch.cat(tpieces))
    imgs = dict(color=(out[:, :3] + T_img[:, None] * bg[None, :]).t().reshape(3, H, W), depth=out[:, 3].reshape(1, H, W),
                alpha=(1.0 - T_img).reshape(1, H, W), flow=out[:, 4:6].t().reshape(2, H, W))
    L = 0.0
    for g, key in zip(grads, ("color", "depth", "alpha", "flow")):
        if g is not None:
            L = L + (imgs[key] * torch.as_tensor(np.asarray(g, np.float32)).to(F64)).sum()
    return L, fclamp.numpy(), amb.reshape(H, W)


def camera_grads(st, lists, t, grads):
    """float64 dL/dviewmatrix [4,4], dL/dprojmatrix [4,4] and dL/dmeans3D [P,3] of loss() at the settings' camera"""
    V = torch.as_tensor(st["viewmatrix"]).detach().cpu().to(F64).requires_grad_(True)
    Pm = torch.as_tensor(st["projmatrix"]).detach().cpu().to(F64).requires_grad_(True)
    m = torch.as_tensor(np.asarray(t["means3D"], np.float32)).to(F64).requires_grad_(True)
    L, fclamp, amb = loss(st, lists, t, grads, V, Pm, means3D=m)
    L.backward()
    return dict(view=V.grad.numpy(), proj=Pm.grad.numpy(), means3D=m.grad.numpy(), frustum_clamp=fclamp, ambiguous=amb)
