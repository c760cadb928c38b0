"""GPU (-m gpu): fdgs.optim.FusedAdam's semantics over long runs, against torch.optim.Adam(eps=1e-15) (the reference's
optimiser, scene/gaussian_model.py:357) and a float64 restatement of the same update:

  * 2000 steps with the xyz learning rate's exponential schedule changing every step: every 100 steps ours is within
    2x torch fp32's distance from float64 (per tensor, relative L2 and max), and the moments within 4 ulps of torch's;
  * gradients of 1e-20 (squares are fp32 denormals) and 1e20 (squares overflow), and rows exactly zero for hundreds of
    steps;
  * per-parameter step counts: a parameter whose .grad is None skips a step without advancing its count, a group
    added mid-run starts at step 1, the count survives a densification, and a run resumed at step 29 990 uses that
    step's bias correction;
  * the sparse mode over many steps: listed rows follow the dense update of a model whose unlisted rows are frozen
    (float64 restatement), unlisted rows stay bit-identical, and unsorted rows covering every row equal the dense step."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
B1, B2, EPS = 0.9, 0.999, 1e-15


class Adam64:
    """torch.optim.Adam's update (amsgrad off, no weight decay) in float64, one step count per tensor; rows=None is
    dense, otherwise only the listed rows move (the step count still advances for the whole tensor)"""

    def __init__(self, params):
        self.p = [p.detach().double().clone() for p in params]
        self.m = [torch.zeros_like(p) for p in self.p]
        self.v = [torch.zeros_like(p) for p in self.p]
        self.t = [0] * len(self.p)

    def step(self, grads, lrs, rows=None):
        for i, (g, lr) in enumerate(zip(grads, lrs)):
            if g is None:
                continue
            self.t[i] += 1
            t = self.t[i]
            g = g.double()
            sel = slice(None) if rows is None else rows
            m, v = self.m[i][sel], self.v[i][sel]
            m = B1 * m + (1 - B1) * g[sel]
            v = B2 * v + (1 - B2) * g[sel] * g[sel]
            bc1, bc2 = 1 - B1 ** t, 1 - B2 ** t
            self.p[i][sel] = self.p[i][sel] - lr / bc1 * m / (v.sqrt() / math.sqrt(bc2) + EPS)
            self.m[i][sel], self.v[i][sel] = m, v


def _ulp(t):
    a = t.abs().float()
    return torch.nextafter(a, torch.full_like(a, float("inf"))) - a


def _moments_close(sa, sb, ulps=4):
    for key in ("exp_avg", "exp_avg_sq"):
        a, b = sa[key], sb[key]
        d = torch.where(a == b, 0.0, (a - b).abs())                    # equal infinities (overflowed g * g) match
        assert bool((d <= ulps * _ulp(b)).all()), (key, float(d.max()), float(b.abs().max()))


def _dist(p32, p64):
    d = p32.double() - p64
    return float(d.norm() / max(float(p64.norm()), 1e-300)), float(d.abs().max())


def _xyz_lr(step, lr_init=1.6e-4 * 1.3, lr_final=1.6e-6 * 1.3, max_steps=30_000):
    """the xyz schedule of the reference (utils/general_utils.py get_expon_lr_func, no delay)"""
    t = min(max(step / max_steps, 0.0), 1.0)
    return math.exp(math.log(lr_init) * (1 - t) + math.log(lr_final) * t)


def _three(params, lrs):
    from fdgs.optim import FusedAdam
    pa = [p.clone().requires_grad_(True) for p in params]
    pb = [p.clone().requires_grad_(True) for p in params]
    ta = torch.optim.Adam([{"params": [p], "lr": lr} for p, lr in zip(pa, lrs)], lr=0.0, eps=EPS)
    fb = FusedAdam([{"params": [p], "lr": lr} for p, lr in zip(pb, lrs)], lr=0.0, eps=EPS)
    return pa, pb, ta, fb, Adam64(params)


def _assert_bars(pa, pb, ref, label):
    for i, (a, b) in enumerate(zip(pa, pb)):
        ro, mo = _dist(b.detach(), ref.p[i])
        rt, mt = _dist(a.detach(), ref.p[i])
        assert ro <= 2 * rt + 1e-300 and mo <= 2 * mt + 1e-300, (label, i, ro, rt, mo, mt)


# ---- long run ------------------------------------------------------------------------------------------------------------
def test_long_run_with_schedule():
    g = torch.Generator().manual_seed(1)
    P = 3001
    shapes = [(P, 3), (P, 1), (P, 16, 3), (P, 4)]
    params = [torch.randn(*s, generator=g).to(DEV) for s in shapes]
    base_lrs = [None, 1.6e-4, 2.5e-3 / 20, 1e-3]
    pa, pb, ta, fb, ref = _three(params, [0.0] * 4)
    zero_rows = torch.arange(0, P, 7, device=DEV)                          # exactly zero for steps 200..899
    for step in range(1, 2001):
        lrs = [_xyz_lr(step)] + base_lrs[1:]
        for opt in (ta, fb):
            for grp, lr in zip(opt.param_groups, lrs):
                grp["lr"] = lr
        grads = []
        for s in shapes:
            gr = (torch.randn(*s, generator=g) * (0.1 + torch.rand(s[0], *[1] * (len(s) - 1), generator=g))).to(DEV)
            if 200 <= step < 900:
                gr[zero_rows] = 0.0
            grads.append(gr)
        for a, b, gr in zip(pa, pb, grads):
            a.grad, b.grad = gr.clone(), gr.clone()
        ta.step()
        fb.step()
        ref.step(grads, lrs)
        if step % 100 == 0:
            _assert_bars(pa, pb, ref, step)
            for a, b in zip(pa, pb):
                _moments_close(ta.state[a], fb.state[b])
                assert int(fb.state[b]["step"]) == step == int(ta.state[a]["step"])
    assert float(fb.state[pb[0]]["exp_avg_sq"][zero_rows].abs().max()) > 0     # the zero rows resumed
    print("2000 steps: every 100 within 2x torch fp32's distance from float64")


@pytest.mark.parametrize("scale", [1e-20, 1e20])
def test_extreme_gradients(scale):
    """1e-20: g*g is a fp32 denormal, which the kernel must not flush; 1e20: g*g overflows to inf in fp32, as in torch
    (the update is then m / inf = 0)"""
    g = torch.Generator().manual_seed(2)
    P = 2048
    params = [torch.randn(P, 3, generator=g).to(DEV)]
    pa, pb, ta, fb, ref = _three(params, [1e-3])
    for step in range(50):
        gr = (scale * torch.randn(P, 3, generator=g)).to(DEV)
        pa[0].grad, pb[0].grad = gr.clone(), gr.clone()
        ta.step()
        fb.step()
        ref.step([gr], [1e-3])
    v = fb.state[pb[0]]["exp_avg_sq"]
    if scale < 1:
        assert bool(((v > 0) & (v < torch.finfo(torch.float32).tiny)).any())    # denormal second moments
        _assert_bars(pa, pb, ref, scale)
        _moments_close(ta.state[pa[0]], fb.state[pb[0]])
    else:
        # g * g overflows in the kernel's order (the square first, then * (1 - beta2)): the second moment is inf and the
        # update m / inf = 0 from then on, and everything stays finite (torch's addcmul keeps v finite here and moves them)
        inf = torch.isinf(v)
        assert bool(inf.float().mean() > 0.5)
        assert bool(torch.isfinite(pb[0]).all()) and bool(torch.isfinite(fb.state[pb[0]]["exp_avg"]).all())


# ---- step counts ---------------------------------------------------------------------------------------------------------
def test_intermittent_gradients_and_added_group():
    """B's .grad is None on every third step; group C joins at step 40.  torch counts steps per parameter"""
    g = torch.Generator().manual_seed(3)
    P = 1500
    params = [torch.randn(P, 3, generator=g).to(DEV) for _ in range(3)]
    lrs = [1e-3, 2e-3, 5e-3]
    from fdgs.optim import FusedAdam
    pa = [p.clone().requires_grad_(True) for p in params]
    pb = [p.clone().requires_grad_(True) for p in params]
    ta = torch.optim.Adam([{"params": [pa[0]], "lr": lrs[0]}, {"params": [pa[1]], "lr": lrs[1]}], lr=0.0, eps=EPS)
    fb = FusedAdam([{"params": [pb[0]], "lr": lrs[0]}, {"params": [pb[1]], "lr": lrs[1]}], lr=0.0, eps=EPS)
    ref = Adam64(params)
    for step in range(1, 121):
        if step == 40:
            ta.add_param_group({"params": [pa[2]], "lr": lrs[2]})
            fb.add_param_group({"params": [pb[2]], "lr": lrs[2]})
        grads = []
        for i in range(3):
            skip = (i == 1 and step % 3 == 0) or (i == 2 and step < 40)
            grads.append(None if skip else torch.randn(P, 3, generator=g).to(DEV))
        for a, b, gr in zip(pa, pb, grads):
            a.grad = None if gr is None else gr.clone()
            b.grad = None if gr is None else gr.clone()
        ta.step()
        fb.step()
        ref.step(grads, lrs)
    assert [int(fb.state[b]["step"]) for b in pb] == [120, 80, 81] == [int(ta.state[a]["step"]) for a in pa]
    _assert_bars(pa, pb, ref, "intermittent")
    for a, b in zip(pa, pb):
        _moments_close(ta.state[a], fb.state[b])


def test_resumed_at_a_late_step():
    """bias corrections near the end of a 30 000-step run: state loaded at step 29 990 (torch's format) continues
    with that step's correction"""
    g = torch.Generator().manual_seed(4)
    P = 1000
    params = [torch.randn(P, 3, generator=g).to(DEV)]
    pa, pb, ta, fb, ref = _three(params, [1.6e-6])
    m0 = (1e-3 * torch.randn(P, 3, generator=g)).to(DEV)
    v0 = (1e-6 * torch.rand(P, 3, generator=g)).to(DEV)
    ta.state[pa[0]] = {"step": torch.tensor(29990.0), "exp_avg": m0.clone(), "exp_avg_sq": v0.clone()}
    fb.state[pb[0]] = {"step": torch.tensor(29990.0), "exp_avg": m0.clone(), "exp_avg_sq": v0.clone()}
    ref.m[0], ref.v[0], ref.t[0] = m0.double(), v0.double(), 29990
    for _ in range(10):
        gr = (1e-3 * torch.randn(P, 3, generator=g)).to(DEV)
        pa[0].grad, pb[0].grad = gr.clone(), gr.clone()
        ta.step()
        fb.step()
        ref.step([gr], [1.6e-6])
    assert int(fb.state[pb[0]]["step"]) == 30000
    _assert_bars(pa, pb, ref, "late")
    _moments_close(ta.state[pa[0]], fb.state[pb[0]])


def test_step_count_survives_densification():
    """a densification between steps re-keys the state with its "step" (fdgs.densify, as the reference's
    cat_tensors_to_optimizer does): the next step uses the carried count"""
    import densify_ref as R
    from fdgs import densify
    nat = R.make_model(20_000, 16, 4, True, optim="fused")
    ref = R.clone_model(nat, optim="torch")
    g = torch.Generator().manual_seed(6)
    for it in range(4):
        for name in nat.group_names():
            a, b = getattr(nat, R.ATTR[name]), getattr(ref, R.ATTR[name])
            gr = (torch.randn(a.shape, generator=g) * 1e-2).to(DEV)
            if name == "opacity" and it % 2:
                a.grad = b.grad = None                                 # a parameter without a gradient this step
            else:
                a.grad, b.grad = gr.clone(), gr.clone()
        nat.optimizer.step()
        ref.optimizer.step()
    state = torch.cuda.get_rng_state()
    densify.densify_and_prune(nat, 2e-4, 0.005, 1.0, 20)
    torch.cuda.set_rng_state(state)
    densify.densify_and_prune(ref, 2e-4, 0.005, 1.0, 20)
    for name in nat.group_names():
        a, b = getattr(nat, R.ATTR[name]), getattr(ref, R.ATTR[name])
        assert a.shape == b.shape
        assert int(nat.optimizer.state[a]["step"]) == int(ref.optimizer.state[b]["step"]) == (3 if name == "opacity" else 5)
        gr = (torch.randn(a.shape, generator=g) * 1e-2).to(DEV)
        a.grad, b.grad = gr.clone(), gr.clone()
    nat.optimizer.step()
    ref.optimizer.step()
    for name in nat.group_names():
        a, b = getattr(nat, R.ATTR[name]), getattr(ref, R.ATTR[name])
        d = (a - b).abs()
        assert float(d.max()) <= 1e-5 * 1e-3 * 6 + 2e-7 * float(b.abs().max()), (name, float(d.max()))
        _moments_close(nat.optimizer.state[a], ref.optimizer.state[b])


# ---- sparse mode ---------------------------------------------------------------------------------------------------------
def test_sparse_over_many_steps():
    """300 steps, each over a random 30 % of the rows (rows move in and out of the rendered set; moments non-zero after
    the first step): listed rows follow the frozen-rows model's dense update in float64, unlisted rows are bit-identical"""
    from fdgs.optim import FusedAdam
    g = torch.Generator().manual_seed(7)
    P = 4000
    shapes = [(P, 3), (P, 16, 3), (P, 1)]
    lrs = [1e-3, 2.5e-3 / 20, 5e-2]
    params = [torch.randn(*s, generator=g).to(DEV) for s in shapes]
    pb = [p.clone().requires_grad_(True) for p in params]
    fb = FusedAdam([{"params": [p], "lr": lr} for p, lr in zip(pb, lrs)], eps=EPS)
    ref = Adam64(params)
    worst = 0.0
    count = torch.zeros(P, dtype=torch.float64, device=DEV)               # updates each row has had
    for step in range(1, 301):
        vis = torch.rand(P, generator=g) < 0.3
        rows = torch.nonzero(vis).squeeze(1).to(DEV)
        before = [p.detach().clone() for p in pb]
        mv = [(fb.state[p]["exp_avg"].clone(), fb.state[p]["exp_avg_sq"].clone()) if p in fb.state else None for p in pb]
        grads = [torch.randn(*s, generator=g).to(DEV) for s in shapes]   # unlisted rows' gradients are ignored
        for b, gr in zip(pb, grads):
            b.grad = gr.clone()
        fb.step(rows=rows)
        ref.step(grads, lrs, rows=rows)
        count[rows] += 1
        off = ~vis.to(DEV)
        for b, p0, st, s0 in zip(pb, before, (fb.state[p] for p in pb), mv):
            assert torch.equal(b.detach()[off], p0[off])
            if s0 is not None:
                assert torch.equal(st["exp_avg"][off], s0[0][off]) and torch.equal(st["exp_avg_sq"][off], s0[1][off])
        if step % 50 == 0:
            for i, b in enumerate(pb):
                d = (b.detach().double() - ref.p[i]).abs()
                # per update at most one rounding of p (an ulp of the larger of |p| before and after) and ~1e-6 of the
                # step (<= a few lr): a wrong bias correction is off by O(10 %) of lr per update
                cnt = count.view(-1, *[1] * (b.dim() - 1))
                mag = torch.maximum(params[i].abs(), b.detach().abs())
                bar = cnt * (_ulp(mag).double() + 1e-5 * lrs[i])
                assert bool((d <= bar).all()), (step, i, float((d - bar).max()))
                worst = max(worst, float(d.max() / (ref.p[i] - params[i].double()).abs().max()))
    print("sparse 300 steps: worst max |ours - f64| / max displacement = %.2e" % worst)


def test_sparse_with_every_row_unsorted_equals_dense():
    from fdgs.optim import FusedAdam
    g = torch.Generator().manual_seed(8)
    P = 3000
    params = [torch.randn(P, 3, generator=g).to(DEV), torch.randn(P, 16, 3, generator=g).to(DEV)]
    pd = [p.clone().requires_grad_(True) for p in params]
    ps = [p.clone().requires_grad_(True) for p in params]
    od = FusedAdam([{"params": [p], "lr": 1e-3} for p in pd], eps=EPS)
    osp = FusedAdam([{"params": [p], "lr": 1e-3} for p in ps], eps=EPS)
    for _ in range(20):
        for a, b in zip(pd, ps):
            gr = torch.randn(a.shape, generator=g).to(DEV)
            a.grad, b.grad = gr.clone(), gr.clone()
        od.step()
        osp.step(rows=torch.randperm(P, generator=g).to(DEV))
    for a, b in zip(pd, ps):
        assert torch.equal(a, b)
        assert torch.equal(od.state[a]["exp_avg"], osp.state[b]["exp_avg"])
        assert torch.equal(od.state[a]["exp_avg_sq"], osp.state[b]["exp_avg_sq"])
