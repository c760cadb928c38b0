"""H100: native densify-and-prune, reset_opacity and the statistics update against the reference's surgery restated
in tests/densify_ref.py, run from the same generator state.  Everything is bit-identical except the split children's
positions and times, which are held against a float64 evaluation of the same formula on the same samples."""
import pytest
import torch

import densify_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
VARIANTS = [(3, False), (4, False), (4, True)]
IDS = ["3d", "4d", "4d_rot4d"]
# (max_grad, min_opacity, max_screen_size, prune_only)
CASES = {
    "densify": (2e-4, 0.05, 20, False),             # clones, splits, opacity and world-size prunes of originals and children
    "densify_no_screen": (2e-4, 0.05, None, False),
    "nothing_selected": (1e9, 0.05, 20, False),     # S = 0 and C = 0
    "prune_only": (2e-4, 0.05, 20, True),          # live max_radii2D over max_screen_size
    "all_pruned": (2e-4, 1.5, None, False),
}


def _native(m, case, N=2, generator=None):
    from fdgs import densify as D
    mg, mo, mss, po = CASES[case]
    return D.densify_and_prune(m, mg, mo, m.extent, mss, prune_only=po, N=N, generator=generator)


def _reference(m, case, N=2, record=None):
    mg, mo, mss, po = CASES[case]
    with torch.no_grad():
        R.ref_densify_and_prune(m, mg, mo, m.extent, mss, prune_only=po, N=N, record=record)


def _ulp(x):
    a = x.abs()
    return torch.nextafter(a, torch.full_like(a, float("inf"))) - a


def _positions_f64(rec, raw, raw_t, rot_4d):
    """xyz (and t) of every split child in float64 from the raw normal draws and the fp32 std / quaternions / means."""
    d = torch.float64
    std = rec["std"].to(d)
    smp = raw.to(d) * std
    if rot_4d:
        Rm = R._rot4(rec["ql"].to(d), rec["qr"].to(d))
        xyzt = torch.bmm(Rm, smp.unsqueeze(-1)).squeeze(-1) + rec["mean"].to(d)
        return xyzt[:, :3], xyzt[:, 3:4]
    Rm = R._rot3(rec["q"].to(d))
    xyz = torch.bmm(Rm, smp.unsqueeze(-1)).squeeze(-1) + rec["mean"].to(d)
    t = None
    if raw_t is not None:
        t = raw_t.to(d) * rec["std_t"].to(d) + rec["mean_t"].to(d)
    return xyz, t


def _compare(nat, ref, rec=None, N=2, label=""):
    """Bit-identical everything; split children's xyz / t within 2x torch's distance from float64 + 1 ulp."""
    P = ref._xyz.shape[0]
    assert nat._xyz.shape[0] == P, (label, nat._xyz.shape[0], P)
    kids = 0
    if rec is not None and "samples" in rec:
        kids = int(rec["child_keep"].sum())
    for name in ref.group_names():
        a, b = getattr(nat, R.ATTR[name]), getattr(ref, R.ATTR[name])
        assert a.shape == b.shape, (label, name)
        if name in ("xyz", "t") and kids:
            assert torch.equal(a[:P - kids], b[:P - kids]), (label, name, "copied rows")
        else:
            assert torch.equal(a, b), (label, name, int((a != b).sum()))
        sa, sb = nat.optimizer.state.get(a), ref.optimizer.state.get(b)
        assert (sa is None) == (sb is None), (label, name)
        if sa is not None:
            assert torch.equal(sa["exp_avg"], sb["exp_avg"]), (label, name, "exp_avg")
            assert torch.equal(sa["exp_avg_sq"], sb["exp_avg_sq"]), (label, name, "exp_avg_sq")
            if "step" in sb:
                assert torch.equal(torch.as_tensor(sa["step"]), torch.as_tensor(sb["step"])), (label, name)
    for s in ["xyz_gradient_accum", "denom", "max_radii2D"] + (["t_gradient_accum"] if ref.gaussian_dim == 4 else []):
        assert torch.equal(getattr(nat, s), getattr(ref, s)), (label, s)
    return kids


def _check_positions(nat, ref, rec, raw, raw_t, kids, label):
    keep = rec["child_keep"]
    xyz64, t64 = _positions_f64(rec, raw, raw_t, ref.rot_4d)
    pairs = [("xyz", xyz64[keep])] + ([("t", t64[keep])] if t64 is not None else [])
    worst = 0.0
    for name, want in pairs:
        a = getattr(nat, R.ATTR[name]).detach()[-kids:].double()
        b = getattr(ref, R.ATTR[name]).detach()[-kids:].double()
        ours, torchs = (a - want).abs(), (b - want).abs()
        bar = 2 * torchs + _ulp(want.float()).double()
        assert bool((ours <= bar).all()), (label, name, float((ours - bar).max()))
        worst = max(worst, float(ours.max().detach()))
    return worst


def _run_case(P, M, dim, rot_4d, optim, case, seed=0, N=2):
    m = R.make_model(P, M, dim, rot_4d, optim=optim, seed=seed)
    ref = R.clone_model(m)
    state = torch.cuda.get_rng_state()
    rec = {}
    _reference(ref, case, N=N, record=rec)
    torch.cuda.set_rng_state(state)
    P_new = _native(m, case, N=N)
    assert P_new == ref._xyz.shape[0]
    kids = _compare(m, ref, rec, N=N, label=(dim, rot_4d, optim, case))
    if kids:
        # the raw normal draws of both: the reference's torch.normal is normal_(0, 1) * std
        torch.cuda.set_rng_state(state)
        S = rec["samples"].shape[0]
        raw = torch.randn((S, 4 if rot_4d else 3), device=DEV)
        raw_t = torch.randn((S, 1), device=DEV) if (dim == 4 and not rot_4d) else None
        assert torch.equal(raw * rec["std"], rec["samples"])
        _check_positions(m, ref, rec, raw, raw_t, kids, (dim, rot_4d, optim, case))
    return m, ref, rec


@pytest.mark.parametrize("optim", ["fused", "torch"])
@pytest.mark.parametrize("dim,rot_4d", VARIANTS, ids=IDS)
@pytest.mark.parametrize("case", list(CASES))
def test_densify_matches_reference_50k(case, dim, rot_4d, optim):
    m, ref, rec = _run_case(50_000, 16, dim, rot_4d, optim, case)
    if case == "densify":
        n_kids = int(rec["child_keep"].sum())
        assert 0 < n_kids < rec["child_keep"].numel(), "children both kept and pruned"
        assert ref._xyz.shape[0] > 0


def test_branches_are_reached():
    """The seeded statistics reach every branch the issue lists (counted on the restatement's inputs)."""
    m = R.make_model(50_000, 16, 4, True, optim="torch")
    dense = torch.tensor(m.percent_dense * m.extent, dtype=torch.float32).item()
    big = torch.tensor(0.1 * m.extent, dtype=torch.float32).item()
    smax = torch.exp(m._scaling.detach()).max(1).values
    g = m.xyz_gradient_accum / m.denom
    assert int((smax == dense).sum()) > 100 and int((smax == big).sum()) > 50
    assert int(g.isnan().sum()) > 100 and int(g.isinf().sum()) > 100
    assert int((g == torch.tensor(2e-4, dtype=torch.float32).item()).sum()) > 100
    g = torch.nan_to_num(g, nan=0.0).squeeze(1)
    clone = (g >= 2e-4) & (smax <= dense)
    split = (g >= 2e-4) & (smax > dense)
    assert int(clone.sum()) > 1000 and int(split.sum()) > 1000
    assert int((torch.sigmoid(m._opacity.detach()).squeeze(1) < 0.05).sum()) > 1000
    assert int((smax > big).sum()) > 1000


@pytest.mark.parametrize("optim", ["fused", "torch"])
@pytest.mark.parametrize("dim,rot_4d", VARIANTS, ids=IDS)
def test_densify_matches_reference_cfg3_size(dim, rot_4d, optim):
    """2M Gaussians with 48 SH coefficients (cfg3 size)."""
    m, ref, rec = _run_case(2_000_000, 48, dim, rot_4d, optim, "densify", seed=3)
    del m, ref
    torch.cuda.empty_cache()


@pytest.mark.parametrize("optim", ["fused", "torch"])
def test_reset_opacity_matches_reference(optim):
    from fdgs import densify as D
    m = R.make_model(50_000, 16, 4, True, optim=optim)
    with torch.no_grad():
        m._opacity.data[:7, 0] = torch.tensor([-30.0, -4.59512, -4.59511, 0.0, 30.0, 8.0, -4.5951198])
    ref = R.clone_model(m)
    with torch.no_grad():
        R.ref_reset_opacity(ref)
    D.reset_opacity(m)
    _compare(m, ref, label="reset_opacity")
    assert torch.equal(m.optimizer.state[m._opacity]["exp_avg"], torch.zeros_like(m._opacity))


@pytest.mark.parametrize("batch", [1, 4])
@pytest.mark.parametrize("dim", [3, 4])
def test_stats_match_reference(batch, dim):
    from fdgs import densify as D
    from fdgs.dist import ViewBatchStats
    P = 50_000
    m = R.make_model(P, 4, dim, False, optim="torch")
    ref = R.clone_model(m)
    g = torch.Generator(device="cpu").manual_seed(7)
    grads = [(torch.randn(P, 3, generator=g) * 1e-3).to(DEV) for _ in range(batch)]
    radii = [(torch.randint(-3, 30, (P,), generator=g).clamp_min(0)).int().to(DEV) for _ in range(batch)]
    t_grad = (torch.randn(P, 1, generator=g) * 1e-3).to(DEV) if dim == 4 else None
    with torch.no_grad():
        gsum = R.ref_stats(ref, grads, radii, t_grad)
    if batch == 1:
        D.add_densification_stats(m, grads[0], radii[0], t_grad=t_grad)
    else:
        st = ViewBatchStats(P, DEV)
        st.grad_norm_sum = gsum.unsqueeze(1).contiguous()
        st.visibility_count = torch.stack([r > 0 for r in radii], 1).sum(1).float().unsqueeze(1)
        st.max_radii = torch.stack(radii, 1).max(1)[0].int()
        D.add_densification_stats(m, t_grad=t_grad, batch_stats=st, batch_size=batch)
    for s in ["xyz_gradient_accum", "denom", "max_radii2D"] + (["t_gradient_accum"] if dim == 4 else []):
        assert torch.equal(getattr(m, s), getattr(ref, s)), s


def test_same_seed_same_model_other_seed_moves_only_split_positions():
    from fdgs import densify as D
    base = R.make_model(50_000, 16, 4, True, optim="fused")
    out = []
    for seed in (11, 11, 12):
        m = R.clone_model(base)
        gen = torch.Generator(device=DEV).manual_seed(seed)
        D.densify_and_prune(m, 2e-4, 0.05, m.extent, 20, generator=gen)
        out.append(m)
    a, b, c = out
    _compare(a, b, label="same seed")
    for name in a.group_names():
        x, z = getattr(a, R.ATTR[name]), getattr(c, R.ATTR[name])
        if name in ("xyz", "t"):
            assert not torch.equal(x, z)
            diff_rows = (x != z).reshape(x.shape[0], -1).any(1).nonzero().squeeze(1)
            kids = x.shape[0] - int(diff_rows.min())
            assert kids > 0
        else:
            assert torch.equal(x, z), name


def test_next_step_after_native_surgery_matches_torch_adam():
    """FusedAdam after the native surgery vs torch.optim.Adam after the reference surgery: within the bars of
    test_fused_adam_dense_matches_torch_adam."""
    base = R.make_model(50_000, 16, 4, True, optim="torch")
    nat = R.clone_model(base, optim="fused")
    ref = R.clone_model(base, optim="torch")
    state = torch.cuda.get_rng_state()
    _reference(ref, "densify")
    torch.cuda.set_rng_state(state)
    _native(nat, "densify")
    g = torch.Generator(device="cpu").manual_seed(5)
    for name in ref.group_names():
        a, b = getattr(nat, R.ATTR[name]), getattr(ref, R.ATTR[name])
        gr = (torch.randn(a.shape, generator=g) * 1e-2).to(DEV)
        a.grad, b.grad = gr.clone(), gr.clone()
    nat.optimizer.step()
    ref.optimizer.step()
    lr = 1e-3
    for name in ref.group_names():
        a, b = getattr(nat, R.ATTR[name]), getattr(ref, R.ATTR[name])
        d = (a - b).abs()
        assert float(d.max()) <= 1e-5 * lr + 2e-7 * float(b.abs().max()), (name, float(d.max()))
        sa, sb = nat.optimizer.state[a], ref.optimizer.state[b]
        assert torch.allclose(sa["exp_avg"], sb["exp_avg"], rtol=2e-6, atol=2e-7)
        assert torch.allclose(sa["exp_avg_sq"], sb["exp_avg_sq"], rtol=2e-6, atol=1e-9)
