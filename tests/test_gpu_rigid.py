"""H100: the native rigidity and motion regularisers (fdgs.regularize over csrc/regularize.cu) against the reference's
expressions restated in tests/rigid_ref.py.

Scenes: the lego initialisation (tests/lego.py's distributions) at 100k and 2M, clustered points, n < k (n = 7,
padded entries of weight 0), and a hub of 2000 exact duplicates of one row (half with perturbed quaternions, half
identical: zero-norm edges and in-degrees far above k).

  - the weights are bit-identical to torch.exp(-100 * dist), the transpose is the stable argsort of the neighbours
  - velocity, both losses and the four gradients are within 2 x the float32 restatement's distance from the float64
    restatement, plus a floor of a few ulp, on relative L2 and on the row-wise maximum (row error over the largest
    reference row), with an upstream gradient != 1
  - no NaN / Inf in the hub scene; two calls give torch.equal values and gradients
  - forward and backward with a given neighbour list never synchronise the host
A 30-iteration lego-shaped training loop (batch 2, render() raw entry + L1 + both regularisers) checks the losses and
every gradient at every iteration against the restatement with per-view kNN, then steps on the native gradients.
"""
import math

import pytest
import torch

import rigid_ref

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FLOOR = 8 * 2.0 ** -24          # a few fp32 ulp, relative to the reference's scale
LAMBDA_RIGID, LAMBDA_MOTION, BATCH = 1.0, 0.1, 2
NAMES = ("_scaling", "_scaling_t", "_rotation", "_rotation_r")


class Model:
    """The attributes of the reference's GaussianModel the regularisers read (rot_4d, raw parameters)."""
    rot_4d, gaussian_dim = True, 4

    def __init__(self, _xyz, _t, _scaling, _scaling_t, _rotation, _rotation_r):
        self._xyz, self._t = _xyz, _t
        self._scaling, self._scaling_t, self._rotation, self._rotation_r = _scaling, _scaling_t, _rotation, _rotation_r

    get_xyz = property(lambda s: s._xyz)
    get_t = property(lambda s: s._t)


def _leaves(p):
    return {k: v.detach().clone().contiguous().requires_grad_(k in NAMES) for k, v in p.items()}


def lego_scene(n, seed=0):
    """tests/lego.py lego_setup's initial distributions (gaussian_model.py:280-281 for scaling_t)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    u = lambda *s: torch.rand(*s, generator=g, device=DEV)
    nn_ = lambda *s: torch.randn(*s, generator=g, device=DEV)
    return dict(_xyz=u(n, 3) * 2.6 - 1.3, _t=u(n, 1), _scaling=torch.log(0.012 * (0.5 + u(n, 3))),
                _scaling_t=math.log(math.sqrt(1.0 / 5)) + 0.1 * nn_(n, 1),
                _rotation=torch.nn.functional.normalize(nn_(n, 4), dim=1),
                _rotation_r=torch.nn.functional.normalize(nn_(n, 4), dim=1))


def clustered_scene(seed=1):
    g = torch.Generator(device=DEV).manual_seed(seed)
    p = lego_scene(40_000, seed)
    centres = torch.rand(40, 3, generator=g, device=DEV) * 2 - 1
    p["_xyz"] = centres[torch.arange(40_000, device=DEV) % 40] + 0.02 * torch.randn(40_000, 3, generator=g, device=DEV)
    p["_rotation"] = torch.randn(40_000, 4, generator=g, device=DEV)          # raw, un-normalised
    return p


def small_scene():
    return lego_scene(7, seed=2)


def hub_scene(seed=3):
    """2000 exact duplicates of row 0 (densification clones onto identical positions); rows 0..999 keep its
    quaternions (identical velocities: zero-norm edges), rows 1000..1999 get perturbed ones; plus 3000 others."""
    p = lego_scene(5000, seed)
    g = torch.Generator(device=DEV).manual_seed(seed + 100)
    for k in p:
        p[k][1:2000] = p[k][0]
    p["_rotation"][1000:2000] += 0.05 * torch.randn(1000, 4, generator=g, device=DEV)
    p["_rotation_r"][1000:2000] += 0.05 * torch.randn(1000, 4, generator=g, device=DEV)
    p["_xyz"][2000:] = p["_xyz"][0] + 0.3 * torch.randn(3000, 3, generator=g, device=DEV)
    return p


SCENES = {"lego100k": lambda: lego_scene(100_000), "lego2M": lambda: lego_scene(2_000_000), "clustered": clustered_scene,
          "n_lt_k": small_scene, "hub": hub_scene}


def _native(p, nb, k=20):
    from fdgs import regularize as R
    q = _leaves(p)
    lr, lm = R.rigidity_and_motion_loss(Model(**q), k, nb)
    (LAMBDA_RIGID * lr / BATCH + LAMBDA_MOTION * lm / BATCH).backward()
    return lr.detach(), lm.detach(), {n: q[n].grad for n in NAMES}


def _restated(p, idx, dist, dtype, k=20):
    q = {n: v.detach().to(dtype).clone().requires_grad_(n in NAMES) for n, v in p.items()}
    args = [q[n] for n in NAMES] + [q["_t"]]
    vel = rigid_ref.velocity(*args)
    lr = rigid_ref.rigid_from_velocity(vel, idx, dist.to(dtype), k)
    lm = rigid_ref.motion_from_velocity(vel)
    (LAMBDA_RIGID * lr / BATCH + LAMBDA_MOTION * lm / BATCH).backward()
    assert q["_t"].grad is None or torch.equal(q["_t"].grad, torch.zeros_like(q["_t"].grad))
    return vel.detach(), lr.detach(), lm.detach(), {n: q[n].grad for n in NAMES}


def _metrics(a, ref):
    """(relative L2, largest row error over the largest reference row); a scalar is one row"""
    a, ref = a.double().reshape(max(ref.shape[:1] or (1,)), -1), ref.double().reshape(max(ref.shape[:1] or (1,)), -1)
    l2 = float((a - ref).norm() / ref.norm().clamp_min(1e-300))
    rowmax = float((a - ref).norm(dim=1).max() / ref.norm(dim=1).max().clamp_min(1e-300))
    return l2, rowmax


def _within_bars(name, ours, f32, f64):
    (o_l2, o_row), (t_l2, t_row) = _metrics(ours, f64), _metrics(f32, f64)
    assert o_l2 <= 2 * t_l2 + FLOOR, (name, "relative L2", o_l2, t_l2)
    assert o_row <= 2 * t_row + FLOOR, (name, "row-wise max", o_row, t_row)
    return o_l2, t_l2, o_row, t_row


@pytest.mark.parametrize("scene", list(SCENES))
def test_against_the_float64_restatement(scene):
    from fdgs import regularize as R
    import fdgs
    k = 20
    p = SCENES[scene]()
    n = p["_xyz"].shape[0]
    nb = R.neighbours(p["_xyz"], k)
    # weights bit-identical to the reference's expression; the transpose is the stable sort by destination
    assert torch.equal(nb.weight, torch.exp(-100 * nb.dist2))
    order = torch.argsort(nb.idx.flatten().long(), stable=True)
    assert torch.equal(nb.in_edges.long(), order)
    counts = torch.bincount(nb.idx.flatten().long(), minlength=n)
    assert torch.equal(nb.in_offsets.long(), torch.cat([counts.new_zeros(1), counts.cumsum(0)]))
    if scene == "n_lt_k":
        assert torch.equal(nb.weight[:, n:], torch.zeros_like(nb.weight[:, n:]))
    if scene == "hub":
        assert int(counts.max()) > 10 * k

    idx, dist = nb.idx.long(), nb.dist2
    v32, r32, m32, g32 = _restated(p, idx, dist, torch.float32)
    v64, r64, m64, g64 = _restated(p, idx, dist, torch.float64)
    params = [p[a].contiguous() for a in ("_t", "_scaling", "_scaling_t", "_rotation", "_rotation_r")]
    vel = fdgs.ext().rigid_forward(params, k, nb.idx, nb.weight, False, False)[0]
    lr, lm, g = _native(p, nb, k)
    report = {"velocity": _within_bars("velocity", vel, v32, v64),
              "L_rigid": _within_bars("L_rigid", lr, r32, r64), "L_motion": _within_bars("L_motion", lm, m32, m64)}
    for name in NAMES:
        report[name] = _within_bars(name, g[name], g32[name], g64[name])
    print(scene, {a: "L2 %.2e (fp32 %.2e) row %.2e (fp32 %.2e)" % b for a, b in report.items()})
    if scene == "hub":
        for t in [vel, lr, lm] + list(g.values()):
            assert torch.isfinite(t).all()
    # run to run: bit-identical
    lr2, lm2, g2 = _native(p, nb, k)
    assert torch.equal(lr, lr2) and torch.equal(lm, lm2)
    assert all(torch.equal(g[a], g2[a]) for a in NAMES)


def test_combined_call_equals_the_separate_ones():
    from fdgs import regularize as R
    p = lego_scene(20_000, seed=7)
    nb = R.neighbours(p["_xyz"])
    q = _leaves(p)
    m = Model(**q)
    lr, lm = R.rigidity_loss(m, neighbours=nb), R.motion_loss(m)
    lr2, lm2 = R.rigidity_and_motion_loss(m, neighbours=nb)
    assert torch.equal(lr, lr2) and torch.equal(lm, lm2)
    lr3 = R.rigidity_loss(m)                       # neighbours=None: recomputed, the same list
    assert torch.equal(lr, lr3)
    (lr + lm).backward()
    sep = {a: q[a].grad.clone() for a in NAMES}
    for a in NAMES:
        q[a].grad = None
    (lr2 + lm2).backward()
    for a in NAMES:      # one chain of dv_rigid + dv_motion vs two chains added by autograd: rounding only
        assert float((q[a].grad - sep[a]).norm()) <= 1e-6 * float(sep[a].norm()), a
    assert q["_xyz"].grad is None and q["_t"].grad is None


def test_no_host_synchronisation_with_a_given_list():
    from fdgs import regularize as R
    p = lego_scene(50_000, seed=8)
    nb = R.neighbours(p["_xyz"])
    q = _leaves(p)
    m = Model(**q)
    g = torch.full((), 0.5, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        lr, lm = R.rigidity_and_motion_loss(m, neighbours=nb)
        (g * lr + g * lm).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(q["_scaling"].grad).all()
