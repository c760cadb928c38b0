"""GPU (-m gpu): the whole training iteration as one CUDA graph -- GraphedStep(..., optimizer=FusedAdam) with
densify_stats=True captures the densification statistics and a staged fused Adam step after the step's backward.

  1. Adam: over 200 iterations with the xyz learning rate changing every step, tensors of different step counts,
     hold=True and hold={"opacity"} iterations and a re-capture, the graphed step equals eager FusedAdam.step() bit for
     bit in parameters, moments and step counts (the image enters the loss times 0, so the gradients are a
     deterministic expression of the leaves and the ground truth);
  2. statistics: for B = 1, 2 and 24 the in-graph statistics equal ViewBatchStats + add_densification_stats computed
     eagerly from the replay's own pkg, bit for bit;
  3. overflow and warm-up: the first call and a call whose replay overflowed each apply exactly one Adam step and one
     statistics update;
  4. rigidity: the rigidity loss with its neighbour list built inside fn equals the eager loss and step bit for bit
     while Adam moves the positions;
  5. synchronisation: the status read is a call's only host synchronisation;
  6. training: a lego-shaped loop (lr schedule, statistics, two densifications, one opacity reset) tracks the eager
     loop run in the reference's order (statistics -> densify / reset -> Adam).
"""
import copy
import math
import warnings

import pytest
import torch
from torch import nn

import helpers

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _lego(P=20000, W=256, H=256):
    from test_gpu_densify_train import _lego_model
    return _lego_model(P, W, H, DEV)


def _leaves(m):
    return [p for g in m.optimizer.param_groups for p in g["params"]]


def _clone(m):
    """An independent copy of the model: parameters, FusedAdam state (counts and moments) and statistics."""
    import densify_ref as R
    from fdgs.optim import FusedAdam
    c = copy.copy(m)
    groups = []
    state = {}
    for g in m.optimizer.param_groups:
        p = g["params"][0]
        q = nn.Parameter(p.detach().clone().requires_grad_(True))
        setattr(c, R.ATTR[g["name"]], q)
        groups.append({"params": [q], "lr": g["lr"], "name": g["name"]})
        st = m.optimizer.state.get(p)
        if st is not None:
            state[q] = {k: v.clone() for k, v in st.items()}
    c.optimizer = FusedAdam(groups, lr=0.0, betas=m.optimizer.betas, eps=m.optimizer.eps)
    c.optimizer.state = state
    for n in ("xyz_gradient_accum", "t_gradient_accum", "denom", "max_radii2D"):
        setattr(c, n, getattr(m, n).clone())
    return c


def _state(m):
    """name -> (parameter, exp_avg, exp_avg_sq, step) and the statistics, for comparisons."""
    out = {}
    for g in m.optimizer.param_groups:
        p = g["params"][0]
        st = m.optimizer.state.get(p, {})
        out[g["name"]] = (p.detach(), st.get("exp_avg"), st.get("exp_avg_sq"), float(st["step"]) if st else None)
    stats = {n: getattr(m, n) for n in ("xyz_gradient_accum", "t_gradient_accum", "denom", "max_radii2D")}
    return out, stats


def _assert_equal(a, b, what):
    sa, ta = _state(a)
    sb, tb = _state(b)
    for name in sa:
        for i, kind in enumerate(("param", "exp_avg", "exp_avg_sq")):
            x, y = sa[name][i], sb[name][i]
            assert (x is None and y is None) or torch.equal(x, y), (what, name, kind)
        assert sa[name][3] == sb[name][3], (what, name, sa[name][3], sb[name][3])
    for n in ta:
        assert torch.equal(ta[n], tb[n]), (what, n)


def _pipe():
    from test_gpu_densify_train import _Pipe
    return _Pipe()


def _exact_loss(m, pkg, gt):
    """The image times 0 (the blend backward adds exact zeros) plus a deterministic expression of every leaf and gt."""
    c = gt.mean()
    loss = pkg["render"].sum() * 0.0
    for i, p in enumerate(_leaves(m)):
        loss = loss + (0.1 * (i + 1)) * ((p - c) ** 2).sum()
    return loss


def _fn(m, loss_fn, bg):
    from gaussian_renderer import render_batch

    def fn(views, gt):
        pkg = render_batch(views, m, _pipe(), bg)
        loss = loss_fn(m, pkg, gt)
        loss.backward()
        return loss, pkg
    return fn


def _eager_grads(m, cams, gt, loss_fn, bg):
    from gaussian_renderer import render_batch
    for p in _leaves(m):
        p.grad = None
    pkg = render_batch(cams, m, _pipe(), bg)
    loss = loss_fn(m, pkg, gt)
    loss.backward()
    return loss, pkg


def _eager_step(m, hold):
    """FusedAdam.step() as the reference's loop sees it: a held (replaced) leaf has no gradient."""
    held = m.optimizer.held(hold)
    for p in _leaves(m):
        if id(p) in held:
            p.grad = None
    m.optimizer.step()


def _gt(cams, s):
    g = torch.Generator().manual_seed(100 + s)
    return torch.rand(len(cams), 3, int(cams[0].image_height), int(cams[0].image_width), generator=g).to(DEV)


# ---- 1. Adam ------------------------------------------------------------------------------------------------------
def test_graphed_adam_equals_eager_fused_adam_bit_for_bit():
    from fdgs.graph import GraphedStep
    m, cams, _ = _lego(P=8000, W=128, H=128)
    bg = torch.zeros(3, device=DEV)
    # different step counts to start with: some groups have stepped before
    for p in _leaves(m):
        p.grad = torch.full_like(p, 1e-3)
    _eager_step(m, {"opacity", "t", "f_rest"})
    m.optimizer.zero_grad()
    e = _clone(m)
    step = GraphedStep(_fn(m, _exact_loss, bg), m, optimizer=m.optimizer)
    xyz_g = [g for g in m.optimizer.param_groups if g["name"] == "xyz"][0]
    exyz_g = [g for g in e.optimizer.param_groups if g["name"] == "xyz"][0]
    for it in range(200):
        views = [cams[(2 * it + k) % len(cams)] for k in range(2)]
        gt = _gt(views, it)
        lr = 1.6e-4 * 0.01 ** (it / 200)          # the xyz schedule changes every iteration
        xyz_g["lr"] = exyz_g["lr"] = lr
        hold = True if it % 37 == 5 else ({"opacity"} if it % 23 == 7 else ())
        if it == 120:                               # a new SH degree re-captures; the optimiser state carries on
            m.active_sh_degree = e.active_sh_degree = 2
        step(views, gt, hold=hold)
        _eager_grads(e, views, gt, _exact_loss, bg)
        _eager_step(e, hold)
        _assert_equal(m, e, it)
    # one capture, one for the SH degree, and one per overflow (R varies with the views; the overflowed replays must
    # have changed nothing for the comparison above to hold)
    assert step.info["captures"] == 2 + step.info["overflows"], step.info
    counts = {g["name"]: float(m.optimizer.state[g["params"][0]]["step"]) for g in m.optimizer.param_groups}
    assert len(set(counts.values())) >= 3, counts


# ---- 2. statistics ------------------------------------------------------------------------------------------------
class _Acc:
    def __init__(self, m):
        self.gaussian_dim = m.gaussian_dim
        for n in ("xyz_gradient_accum", "t_gradient_accum", "denom", "max_radii2D"):
            setattr(self, n, getattr(m, n).clone())


@pytest.mark.parametrize("B", [1, 2, 24])
def test_graphed_statistics_equal_the_eager_statistics_of_the_replay(B):
    import fdgs.densify as D
    from fdgs.dist import ViewBatchStats
    from fdgs.graph import GraphedStep
    from test_gpu_graph import _train_step
    m, cams, gts = _lego(P=20000, W=200, H=200)
    bg = torch.zeros(3, device=DEV)
    step = GraphedStep(_train_step(m, bg), m)
    for s in range(3):
        views = [cams[(s * B + k) % len(cams)] for k in range(B)]
        gt = torch.stack([gts[(s * B + k) % len(cams)] for k in range(B)])
        ref = _Acc(m)
        _, pkg = step(views, gt, densify_stats=True)
        vs, radii = pkg["viewspace_points"].grad, pkg["radii"]
        if B == 1:
            D.add_densification_stats(ref, vs[0], radii[0], t_grad=m._t.grad)
        else:
            st = ViewBatchStats(m._xyz.shape[0], DEV)
            for k in range(B):
                st.add_view(vs[k], radii[k])
            D.add_densification_stats(ref, t_grad=m._t.grad, batch_stats=st, batch_size=B)
        for n in ("xyz_gradient_accum", "t_gradient_accum", "denom", "max_radii2D"):
            assert torch.equal(getattr(m, n), getattr(ref, n)), (B, s, n)
    assert step.info["captures"] == 1 and float(m.denom.max()) >= 1


# ---- 3. overflow and warm-up --------------------------------------------------------------------------------------
def test_warm_up_and_overflow_apply_one_step_and_one_statistics_update():
    from fdgs.graph import GraphedStep
    from test_gpu_graph import _train_step
    m, cams, gts = _lego(P=20000, W=200, H=200)
    bg = torch.zeros(3, device=DEV)
    step = GraphedStep(_train_step(m, bg), m, optimizer=m.optimizer)
    views, gt = cams[:2], torch.stack(gts[:2])

    def check(call):
        before = _clone(m)
        _, pkg = call()
        # one eager step of the copy with the replay's gradients, one statistics update from its pkg
        from fdgs.dist import ViewBatchStats
        import fdgs.densify as D
        st = ViewBatchStats(m._xyz.shape[0], DEV)
        for k in range(2):
            st.add_view(pkg["viewspace_points"].grad[k], pkg["radii"][k])
        D.add_densification_stats(before, t_grad=m._t.grad, batch_stats=st, batch_size=2)
        for p, q in zip(_leaves(before), _leaves(m)):
            p.grad = q.grad.clone()
        before.optimizer.step()
        _assert_equal(m, before, "one step")

    check(lambda: step(views, gt, densify_stats=True))           # the first call: warm-up, capture, replay
    assert step.info["captures"] == 1 and step.info["overflows"] == 0
    step.views.capacity, step._key = 1, None                     # the next call captures at capacity 1 and overflows
    check(lambda: step(views, gt, densify_stats=True))
    assert step.info["captures"] == 3 and step.info["overflows"] == 1, step.info
    status = step._out[1]["status"].tolist()
    assert status[2] == 0 and step.info["capacity"] == math.ceil(1.25 * status[0])
    check(lambda: step(views, gt, densify_stats=True))
    assert step.info["captures"] == 3


# ---- 4. rigidity --------------------------------------------------------------------------------------------------
def _rigid_loss(m, pkg, gt):
    from fdgs import regularize as fr
    nb = fr.neighbours(m.get_xyz)              # rebuilt every step: Adam moves the positions between replays
    return (pkg["render"].sum() * 0.0 + fr.rigidity_loss(m, neighbours=nb)
            + 1e-3 * ((m._xyz - gt.mean()) ** 2).sum())


def test_rigidity_loss_with_its_neighbours_captured_equals_eager():
    from fdgs.graph import GraphedStep
    m, cams, _ = _lego(P=20000, W=128, H=128)
    e = _clone(m)
    bg = torch.zeros(3, device=DEV)
    step = GraphedStep(_fn(m, _rigid_loss, bg), m, optimizer=m.optimizer)
    x0 = m._xyz.detach().clone()
    for it in range(12):
        views = [cams[(2 * it + k) % len(cams)] for k in range(2)]
        gt = _gt(views, it)
        loss, _ = step(views, gt)
        loss_e, _ = _eager_grads(e, views, gt, _rigid_loss, bg)
        assert torch.equal(loss, loss_e), it
        for p, q in zip(_leaves(m), _leaves(e)):
            assert (p.grad is None) == (q.grad is None) and (p.grad is None or torch.equal(p.grad, q.grad)), it
        _eager_step(e, ())
        _assert_equal(m, e, it)
    assert not torch.equal(m._xyz.detach(), x0)
    assert step.info["captures"] == 1


# ---- 5. synchronisation -------------------------------------------------------------------------------------------
def test_the_status_read_is_the_only_synchronisation():
    from fdgs.graph import GraphedStep
    from test_gpu_graph import _train_step
    m, cams, gts = _lego(P=20000, W=200, H=200)
    bg = torch.zeros(3, device=DEV)
    step = GraphedStep(_train_step(m, bg), m, optimizer=m.optimizer)
    views, gt = cams[:2], torch.stack(gts[:2])
    for _ in range(2):
        step(views, gt, densify_stats=True)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            step(views, gt, densify_stats=True, hold={"opacity"})
        finally:
            torch.cuda.set_sync_debug_mode(0)
    syncs = [w for w in caught if "called a synchronizing CUDA operation" in str(w.message)]
    assert len(syncs) == 1, [str(w.message) for w in syncs]
    assert step.info["captures"] == 1


# ---- 6. training --------------------------------------------------------------------------------------------------
def _rel(a, b):
    return helpers.l2_rel(helpers.to_np(a), helpers.to_np(b))


def test_training_loop_with_the_graphed_iteration_tracks_the_eager_loop():
    import fdgs.densify as D
    from fdgs.dist import ViewBatchStats
    from fdgs.graph import GraphedStep
    from test_gpu_densify_train import _max_grad
    from test_gpu_graph import _train_step
    m, cams, gts = _lego(P=20000, W=400, H=400)
    bg = torch.zeros(3, device=DEV)
    batch, iters = 2, 60
    densify_at, reset_at = (20, 40), 30
    step = GraphedStep(_train_step(m, bg), m, optimizer=m.optimizer)
    xyz_lr = lambda it: 1.6e-4 * (1.6e-6 / 1.6e-4) ** (it / iters)     # noqa: E731  (expon_lr_func's log-linear decay)

    def eager(c, views, gt, reset, densify):
        """The reference's order: statistics -> reset / densify -> Adam (a replaced leaf has no gradient)."""
        loss, pkg = _eager_grads(c, views, gt, lambda mm, pk, g: sum((pk["render"][j] - g[j]).abs().mean()
                                                                    for j in range(g.shape[0])), bg)
        st = ViewBatchStats(c._xyz.shape[0], DEV)
        for j in range(len(views)):
            st.add_view(pkg["viewspace_points"].grad[j], pkg["radii"][j])
        D.add_densification_stats(c, t_grad=c._t.grad, batch_stats=st, batch_size=len(views))
        if reset:
            D.reset_opacity(c)
        if not densify:                      # densify_and_prune replaces every leaf: Adam steps nothing
            c.optimizer.step()
        return c

    for it in range(iters):
        for g in m.optimizer.param_groups:
            if g["name"] == "xyz":
                g["lr"] = xyz_lr(it)
        views = [(it * batch + k) % len(cams) for k in range(batch)]
        vc, gt = [cams[k] for k in views], torch.stack([gts[k] for k in views])
        reset, densify = it == reset_at, it in densify_at or it == iters - 1
        e1 = eager(_clone(m), vc, gt, reset, densify)
        e2 = eager(_clone(m), vc, gt, reset, densify)
        hold = True if densify else ({"opacity"} if reset else ())
        step(vc, gt, densify_stats=True, hold=hold)
        if reset:
            D.reset_opacity(m)
        (sg, tg), (s1, t1), (s2, t2) = _state(m), _state(e1), _state(e2)
        for name in sg:
            assert sg[name][3] == s1[name][3], (it, name)
            # floors: the gradient's (test_gpu_graph.py), twice that for the squared gradients of exp_avg_sq
            for i, floor in ((0, 1e-5), (1, 1e-3), (2, 4e-3)):
                err, noise = _rel(sg[name][i], s1[name][i]), _rel(s2[name][i], s1[name][i])
                assert err <= max(floor, 4 * noise), (it, name, i, err, noise)
        for n in tg:
            err, noise = _rel(tg[n], t1[n]), _rel(t2[n], t1[n])
            assert err <= max(1e-3, 4 * noise), (it, n, err, noise)
        if it in densify_at:
            P0 = m._xyz.shape[0]
            D.densify_and_prune(m, _max_grad(m), 0.005, 1.2, None)
            assert m._xyz.shape[0] != P0
    assert step.info["captures"] >= 4 and step.info["overflows"] == 0, step.info
