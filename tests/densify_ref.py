"""Test infrastructure: the reference's densification surgery restated with PyTorch ops (the semantics of
scene/gaussian_model.py:371-589 and train.py:168-183, 233-237 of the original 4D Gaussian splatting code), plus a
seeded model whose statistics reach every branch of it.

The restatement keeps the reference's op sequence where the bits depend on it: clone and split are applied as two
concatenations, the split's selected originals are dropped, then the prune mask is evaluated on every row; samples come
from torch.normal(mean=0, std) in the reference's shapes and order; positions go through torch.bmm.
"""
import math

import torch
from torch import nn

GROUPS_3D = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
ATTR = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
        "scaling": "_scaling", "rotation": "_rotation", "t": "_t", "scaling_t": "_scaling_t", "rotation_r": "_rotation_r"}


def exact_extent(percent_dense, extent, device):
    """An extent near `extent` whose thresholds fp32(percent_dense * extent) and fp32(0.1 * extent) are both exp of an
    fp32 log-scale on this device, and those two log-scales: rows can then sit exactly on either threshold."""
    def step(x, k):
        t = torch.tensor([x], dtype=torch.float32, device=device)
        for _ in range(abs(k)):
            t = torch.nextafter(t, torch.full_like(t, math.copysign(1e9, k)))
        return t
    base = torch.tensor([math.log(percent_dense * extent)], dtype=torch.float32, device=device)
    cand = base.item()
    for _ in range(400):
        dense_v = float(torch.exp(torch.tensor([cand], dtype=torch.float32, device=device)))
        ext = dense_v / percent_dense
        if float(torch.tensor(percent_dense * ext, dtype=torch.float32)) == dense_v:
            big_v = float(torch.tensor(0.1 * ext, dtype=torch.float32))
            c = step(math.log(big_v), -40)
            seq = [c]
            for _ in range(80):
                c = torch.nextafter(c, torch.full_like(c, 1e9))
                seq.append(c)
            seq = torch.cat(seq)
            hit = (torch.exp(seq) == big_v).nonzero()
            if hit.numel():
                return ext, cand, float(seq[hit[0, 0]])
        cand = float(step(cand, 1))
    raise RuntimeError("no extent with exactly representable thresholds found")


class Model:
    """The attributes of the reference's GaussianModel that densification touches."""

    def group_names(self):
        names = list(GROUPS_3D)
        if self.gaussian_dim == 4:
            names += ["t", "scaling_t"] + (["rotation_r"] if self.rot_4d else [])
        return names


def make_model(P, M=16, gaussian_dim=3, rot_4d=False, optim="torch", seed=0, device="cuda", extent=4.0,
               percent_dense=0.01):
    """A seeded model with one optimiser step taken (non-zero moments) and statistics that reach every branch:
    clones, splits, opacity and world-size prunes of originals and of children, denom = 0, rows exactly at the
    gradient and scale thresholds."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    m = Model()
    m.gaussian_dim, m.rot_4d, m.percent_dense = gaussian_dim, rot_4d, percent_dense
    extent, ls_dense, ls_big = exact_extent(percent_dense, extent, device)
    m.extent = extent
    dense = float(torch.tensor(percent_dense * extent, dtype=torch.float32))
    big = float(torch.tensor(0.1 * extent, dtype=torch.float32))
    r = lambda *s: torch.randn(*s, generator=g)
    u = lambda *s: torch.rand(*s, generator=g)
    # log-scales: a mix below / above the dense threshold, some above the world-size threshold, some whose split
    # children land above it, and rows whose largest scale is exactly on either threshold
    smax = torch.exp(torch.empty(P).uniform_(math.log(dense) - 2.0, math.log(big) + 0.6, generator=g))
    pick = u(P)
    on_dense, on_big = pick < 0.02, (pick >= 0.02) & (pick < 0.03)
    smax[on_dense], smax[on_big] = dense, big
    ls = torch.log(smax)[:, None] - 3.0 * u(P, 3) - 1e-3
    col = torch.randint(0, 3, (P,), generator=g)
    ls[torch.arange(P), col] = torch.log(smax)
    ls[on_dense, col[on_dense]] = ls_dense
    ls[on_big, col[on_big]] = ls_big
    ls = ls.to(device)
    m._scaling = ls
    m._xyz = r(P, 3) * 2.0
    m._features_dc = r(P, 1, 3) * 0.5
    m._features_rest = r(P, M - 1, 3) * 0.1
    m._opacity = r(P, 1) * 2.0 - 1.5
    m._rotation = r(P, 4)
    if gaussian_dim == 4:
        m._t = r(P, 1) * 0.3
        m._scaling_t = torch.log(u(P, 1) * 0.3 + 0.01)
        if rot_4d:
            m._rotation_r = r(P, 4)
    # statistics: gradients around max_grad = 2e-4, some rows exactly on it, denom = 0 rows (0/0 = NaN -> 0 and x/0 = inf)
    denom = torch.randint(0, 6, (P, 1), generator=g).float()
    grad = torch.exp(torch.empty(P, 1).uniform_(math.log(2e-5), math.log(2e-3), generator=g))
    on = u(P, 1) < 0.03
    grad[on] = 2e-4
    accum = grad * denom
    accum[on] = float(torch.tensor(2e-4, dtype=torch.float32)) * denom[on]
    accum[(denom == 0) & (u(P, 1) < 0.3)] = 1e-3          # x / 0 = inf: selected
    m.xyz_gradient_accum = accum
    m.denom = denom
    m.max_radii2D = torch.randint(0, 40, (P,), generator=g).float()
    if gaussian_dim == 4:
        m.t_gradient_accum = u(P, 1) * denom
    for k in list(vars(m)):
        v = getattr(m, k)
        if isinstance(v, torch.Tensor):
            setattr(m, k, v.to(device).contiguous())
    names = m.group_names()
    for n in names:
        setattr(m, ATTR[n], nn.Parameter(getattr(m, ATTR[n]).requires_grad_(True)))
    groups = [{"params": [getattr(m, ATTR[n])], "lr": 1e-3, "name": n} for n in names]
    if optim == "torch":
        m.optimizer = torch.optim.Adam(groups, lr=0.0, eps=1e-15)
    else:
        from fdgs.optim import FusedAdam
        m.optimizer = FusedAdam(groups, lr=0.0, eps=1e-15)
    for n in names:
        p = getattr(m, ATTR[n])
        p.grad = torch.randn(p.shape, generator=g).to(device) * 1e-2
    before = [getattr(m, ATTR[n]).detach().clone() for n in names]
    m.optimizer.step()
    for n, b in zip(names, before):        # moments from the step, parameters as constructed (exact threshold rows)
        getattr(m, ATTR[n]).data.copy_(b)
        getattr(m, ATTR[n]).grad = None
    return m


def clone_model(m, optim=None):
    """A deep copy whose optimiser is the same kind (or `optim`: 'torch' / 'fused') with the same state."""
    c = Model()
    for k, v in vars(m).items():
        if k == "optimizer":
            continue
        setattr(c, k, v.detach().clone() if isinstance(v, torch.Tensor) else v)
    names = m.group_names()
    for n in names:
        setattr(c, ATTR[n], nn.Parameter(getattr(m, ATTR[n]).detach().clone().requires_grad_(True)))
    kind = optim or ("torch" if isinstance(m.optimizer, torch.optim.Adam) else "fused")
    groups = [{"params": [getattr(c, ATTR[g["name"]])], "lr": g["lr"], "name": g["name"]} for g in m.optimizer.param_groups]
    if kind == "torch":
        c.optimizer = torch.optim.Adam(groups, lr=0.0, eps=1e-15)
    else:
        from fdgs.optim import FusedAdam
        c.optimizer = FusedAdam(groups, lr=0.0, eps=1e-15)     # the copied state carries each tensor's "step"
    for g_old, g_new in zip(m.optimizer.param_groups, c.optimizer.param_groups):
        st = m.optimizer.state.get(g_old["params"][0])
        if st is not None:
            c.optimizer.state[g_new["params"][0]] = {k: v.clone() for k, v in st.items()}
    return c


# ---- the surgery, restated ------------------------------------------------------------------------------------------
def _swap(m, name, tensor, state_fn):
    """Replace group `name`'s leaf by `tensor`, its moments by state_fn(old moment)."""
    opt = m.optimizer
    grp = next(g for g in opt.param_groups if g["name"] == name)
    old = grp["params"][0]
    st = opt.state.pop(old, None)
    new = nn.Parameter(tensor.requires_grad_(True))
    if st is not None:
        st["exp_avg"] = state_fn(st["exp_avg"])
        st["exp_avg_sq"] = state_fn(st["exp_avg_sq"])
        opt.state[new] = st
    grp["params"][0] = new
    setattr(m, ATTR[name], new)


def _append(m, extra):
    for name, t in extra.items():
        _swap(m, name, torch.cat((getattr(m, ATTR[name]), t), 0), lambda s, t=t: torch.cat((s, torch.zeros_like(t)), 0))
    P = m._xyz.shape[0]
    m.xyz_gradient_accum = torch.zeros((P, 1), device="cuda")
    m.denom = torch.zeros((P, 1), device="cuda")
    m.max_radii2D = torch.zeros((P,), device="cuda")
    if m.gaussian_dim == 4:
        m.t_gradient_accum = torch.zeros((P, 1), device="cuda")


def _keep(m, mask):
    for name in m.group_names():
        _swap(m, name, getattr(m, ATTR[name])[mask], lambda s: s[mask])
    m.xyz_gradient_accum = m.xyz_gradient_accum[mask]
    m.denom = m.denom[mask]
    m.max_radii2D = m.max_radii2D[mask]
    if m.gaussian_dim == 4:
        m.t_gradient_accum = m.t_gradient_accum[mask]


def _rot3(q):
    n = torch.sqrt(q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1] + q[:, 2] * q[:, 2] + q[:, 3] * q[:, 3])
    w, x, y, z = (q / n[:, None]).unbind(1)
    rows = [1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
            2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
            2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]
    return torch.stack(rows, 1).view(-1, 3, 3)


def _rot4(l, r):
    a, b, c, d = (l / torch.norm(l, dim=-1, keepdim=True)).unbind(-1)
    p, q, u, s = (r / torch.norm(r, dim=-1, keepdim=True)).unbind(-1)
    L = torch.stack([a, -b, -c, -d, b, a, -d, c, c, d, a, -b, d, -c, b, a]).view(4, 4, -1).permute(2, 0, 1)
    R = torch.stack([p, q, u, s, -q, p, -s, u, -u, s, p, -q, -s, -u, q, p]).view(4, 4, -1).permute(2, 0, 1)
    return (L @ R).flip(1, 2)


def ref_densify_and_prune(m, max_grad, min_opacity, extent, max_screen_size, prune_only=False, N=2, record=None):
    """The reference's densify_and_prune.  `record` (a dict) receives the split's inputs for a float64 evaluation."""
    if not prune_only:
        grads = m.xyz_gradient_accum / m.denom
        grads[grads.isnan()] = 0.0
        # clone
        sel = torch.norm(grads, dim=-1) >= max_grad
        sel = sel & (torch.max(torch.exp(m._scaling), dim=1).values <= m.percent_dense * extent)
        _append(m, {n: getattr(m, ATTR[n])[sel] for n in m.group_names()})
        # split (over the rows after the clone; clones have a padded gradient of 0)
        P0 = m._xyz.shape[0]
        g = torch.zeros((P0,), device="cuda")
        g[:grads.shape[0]] = grads.squeeze()
        sel = (g >= max_grad) & (torch.max(torch.exp(m._scaling), dim=1).values > m.percent_dense * extent)
        S = int(sel.sum())
        scale = torch.exp(m._scaling)[sel].repeat(N, 1)
        extra = {"scaling": torch.log(scale / (0.8 * N)),
                 "rotation": m._rotation[sel].repeat(N, 1),
                 "f_dc": m._features_dc[sel].repeat(N, 1, 1),
                 "f_rest": m._features_rest[sel].repeat(N, 1, 1),
                 "opacity": m._opacity[sel].repeat(N, 1)}
        if not m.rot_4d:
            smp = torch.normal(mean=torch.zeros((S * N, 3), device="cuda"), std=scale)
            R = _rot3(m._rotation[sel]).repeat(N, 1, 1)
            extra["xyz"] = torch.bmm(R, smp.unsqueeze(-1)).squeeze(-1) + m._xyz[sel].repeat(N, 1)
            if record is not None:
                record.update(samples=smp, std=scale, q=m._rotation[sel].repeat(N, 1), mean=m._xyz[sel].repeat(N, 1))
            if m.gaussian_dim == 4:
                st = torch.exp(m._scaling_t)[sel].repeat(N, 1)
                smp_t = torch.normal(mean=torch.zeros((S * N, 1), device="cuda"), std=st)
                extra["t"] = smp_t + m._t[sel].repeat(N, 1)
                extra["scaling_t"] = torch.log(st / (0.8 * N))
                if record is not None:
                    record.update(samples_t=smp_t, std_t=st, mean_t=m._t[sel].repeat(N, 1))
        else:
            std = torch.exp(torch.cat([m._scaling, m._scaling_t], 1))[sel].repeat(N, 1)
            smp = torch.normal(mean=torch.zeros((S * N, 4), device="cuda"), std=std)
            R = _rot4(m._rotation[sel], m._rotation_r[sel]).repeat(N, 1, 1)
            mean = torch.cat([m._xyz, m._t], 1)[sel].repeat(N, 1)
            xyzt = torch.bmm(R, smp.unsqueeze(-1)).squeeze(-1) + mean
            extra["xyz"], extra["t"] = xyzt[..., 0:3], xyzt[..., 3:4]
            extra["scaling_t"] = torch.log(torch.exp(m._scaling_t)[sel].repeat(N, 1) / (0.8 * N))
            extra["rotation_r"] = m._rotation_r[sel].repeat(N, 1)
            if record is not None:
                record.update(samples=smp, std=std, ql=m._rotation[sel].repeat(N, 1),
                              qr=m._rotation_r[sel].repeat(N, 1), mean=mean)
        _append(m, extra)
        _keep(m, ~torch.cat((sel, torch.zeros(N * S, device="cuda", dtype=bool))))
    prune = (torch.sigmoid(m._opacity) < min_opacity).squeeze()
    if max_screen_size:
        prune = prune | (m.max_radii2D > max_screen_size) | (torch.exp(m._scaling).max(dim=1).values > 0.1 * extent)
    if record is not None and not prune_only:
        record["child_keep"] = ~prune[prune.shape[0] - record["samples"].shape[0]:]
    _keep(m, ~prune)


def ref_reset_opacity(m):
    x = torch.min(torch.sigmoid(m._opacity), torch.ones_like(m._opacity) * 0.01)
    _swap(m, "opacity", torch.log(x / (1 - x)), lambda s: torch.zeros_like(s))


def ref_stats(m, point_grads, radii_list, t_grad):
    """train.py:164-183 + :233-237 for a batch of len(point_grads) views (point_grads: each view's viewspace grad)."""
    B = len(point_grads)
    norms = [torch.norm(pg[:, :2], dim=-1) for pg in point_grads]
    if B > 1:
        count = torch.stack([r > 0 for r in radii_list], 1).sum(1)
        vis = count > 0
        radii = torch.stack(radii_list, 1).max(1)[0]
        gsum = torch.stack(norms, 1).sum(1)
        gsum[vis] = gsum[vis] * B / count[vis]
        gsum = gsum.unsqueeze(1)
        tg = None
        if m.gaussian_dim == 4:
            tg = t_grad.clone()[:, 0]
            tg[vis] = tg[vis] * B / count[vis]
            tg = tg.unsqueeze(1)
    else:
        radii = radii_list[0]
        vis = radii > 0
        tg = t_grad.clone() if m.gaussian_dim == 4 else None
    m.max_radii2D[vis] = torch.max(m.max_radii2D[vis], radii[vis])
    if B == 1:
        m.xyz_gradient_accum[vis] += torch.norm(point_grads[0][vis, :2], dim=-1, keepdim=True)
    else:
        m.xyz_gradient_accum[vis] += gsum[vis]
    m.denom[vis] += 1
    if m.gaussian_dim == 4:
        m.t_gradient_accum[vis] += tg[vis]
    return torch.stack(norms, 1).sum(1) if B > 1 else None
