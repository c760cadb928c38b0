"""GPU (-m gpu): the SH gradient's zero rows written by the forward's blend (include/fdgs.h: fdgs_forward_zero_sh).

In training the autograd forward allocates the dense SH gradient and the blend kernel zeroes the rows of the Gaussians
the view does not render; the backward then writes only the rendered rows.  Checked here with the caching allocator's
blocks poisoned with NaN, so a row nobody wrote shows up: every non-rendered row is exactly zero and every rendered row
matches the path that writes the whole gradient in the backward (the reference-layout entries), up to the blend
backward's atomic accumulation order."""
import pytest
import torch

import helpers

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _poison(numel, n=4):
    """fill n freed blocks of the caching allocator of this size with NaN: the next allocations of the size reuse them"""
    ts = [torch.full((numel,), float("nan"), device=DEV) for _ in range(n)]
    torch.cuda.synchronize()
    del ts


def _scene(name, n=None, shift=0.0):
    cfg, cam, sc, st = helpers.build(name, device=DEV)
    t = {k: v for k, v in sc.tensors().items()}
    if n is not None:
        t = {k: v[:n].contiguous() for k, v in t.items()}
        cfg = dict(cfg, P=n)
    if shift:
        t["means3D"] = t["means3D"] + torch.tensor([shift, 0.0, 0.0], device=DEV)
    return cfg, st, sc, t


def _render(st, t, raw):
    from gaussian_renderer import GaussianRasterizationSettings, GaussianRasterizer
    rast = GaussianRasterizer(GaussianRasterizationSettings(**st))
    means2D = torch.zeros_like(t["means3D"], requires_grad=True)
    if raw:
        p = dict(means3D=t["means3D"], opacity_logits=torch.logit(t["opacities"]), features_dc=t["shs"][:, :1],
                 features_rest=t["shs"][:, 1:], log_scales=torch.log(t["scales"]), rotations_raw=t["rotations"],
                 ts=t["ts"], log_scales_t=torch.log(t["scales_t"]), rotations_r_raw=t["rotations_r"])
        p = {k: v.detach().clone().requires_grad_(True) for k, v in p.items()}
        out = rast.forward_raw(means2D=means2D, flow_2d=t["flow_2d"], **p)
        return p, out, ("features_dc", "features_rest")
    p = {k: t[k].detach().clone().requires_grad_(True) for k in
         ("means3D", "opacities", "shs", "ts", "scales", "scales_t", "rotations", "rotations_r")}
    out = rast(means2D=means2D, flow_2d=t["flow_2d"], **p)
    return p, out, ("shs",)


def _dense_sh_grad(cfg, st, t, raw, gc, gd, ga):
    """the SH gradient as the entries without the forward's zero rows write it (every row in the backward)"""
    import fdgs
    C = fdgs.ext()
    sc = type("S", (), dict(t, gaussian_dim=st["gaussian_dim"], rot_4d=st["rot_4d"]))
    e = torch.empty(0, device=DEV)
    if raw:
        sc.scales, sc.scales_t = torch.log(t["scales"]), torch.log(t["scales_t"])
        sc.opacities = torch.logit(t["opacities"])
        sc.shs = t["shs"][:, :1].contiguous()
        rest = t["shs"][:, 1:].contiguous()
        fw = C.rasterize_gaussians_ext(*helpers.fwd_args(st, sc, cfg), rest, True, e)
        g = C.rasterize_gaussians_backward_ext(*helpers.bwd_args(st, sc, cfg, fw, (gc, gd, ga, e)), rest, True, e,
                                               False, False)
        return g[5], g[13]
    fw = C.rasterize_gaussians(*helpers.fwd_args(st, sc, cfg))
    return (C.rasterize_gaussians_backward(*helpers.bwd_args(st, sc, cfg, fw, (gc, gd, ga, e)))[5],)


CASES = [("tiny", None, 0.0), ("small", None, 0.0), ("ragged", None, 0.0),
         ("tiny", 30, 0.0),        # fewer Gaussians than tiles: stripes of one row, most CTAs own none
         ("tiny", 1999, 0.0),      # P not a multiple of the stripe
         ("tiny", None, 1e4)]      # a view that renders nothing: every row is a zero row


@pytest.mark.parametrize("raw", [False, True], ids=["dense", "split"])
@pytest.mark.parametrize("name,n,shift", CASES, ids=["tiny", "small", "ragged", "p_lt_tiles", "ragged_stripe", "empty"])
def test_unrendered_rows_zero_rendered_rows_match(name, n, shift, raw):
    cfg, st, sc, t = _scene(name, n, shift)
    P = t["means3D"].shape[0]
    _poison(P * t["shs"].shape[1] * 3)
    _poison(P * 3)
    _poison(P * (t["shs"].shape[1] - 1) * 3)
    p, (color, radii, depth, alpha, flow, covs), sh_names = _render(st, t, raw)
    gc, gd, ga, _ = helpers.pixel_grads(cfg, device=DEV)
    ((color * gc).sum() + (depth * gd).sum() + (alpha * ga).sum()).backward()
    torch.cuda.synchronize()
    ref = _dense_sh_grad(cfg, st, t, raw, gc, gd, ga)
    rendered = radii > 0
    if shift:
        assert not rendered.any()
    for name_, want in zip(sh_names, ref):
        got = p[name_].grad
        assert got is not None and got.shape == want.shape, name_
        assert not torch.isnan(got).any(), name_
        assert torch.count_nonzero(got[~rendered]) == 0, name_
        assert torch.count_nonzero(want[~rendered]) == 0, name_
        if rendered.any():
            err = helpers.l2_rel(got[rendered].cpu().numpy(), want[rendered].cpu().numpy())
            assert err < 1e-5, (name_, err)


def test_no_grad_forward_allocates_no_gradient():
    cfg, st, sc, t = _scene("small")
    from gaussian_renderer import GaussianRasterizationSettings, GaussianRasterizer
    rast = GaussianRasterizer(GaussianRasterizationSettings(**st))

    def peak(requires_grad):
        p = {k: t[k].detach().clone().requires_grad_(requires_grad) for k in
             ("means3D", "opacities", "shs", "ts", "scales", "scales_t", "rotations", "rotations_r")}
        means2D = torch.zeros_like(p["means3D"])
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        with torch.no_grad():
            out = rast(means2D=means2D, flow_2d=t["flow_2d"], **p)
        torch.cuda.synchronize()
        del out
        return torch.cuda.max_memory_allocated() - base

    peak(False)   # warm the allocator's pools
    sh_bytes = t["shs"].numel() * 4
    assert peak(True) < peak(False) + sh_bytes // 2


def test_forward_zero_sh_rejects_inconsistent_rows():
    import ctypes
    import fdgs
    lib = fdgs.lib()
    lib.fdgs_forward_zero_sh.restype = ctypes.c_int
    lib.fdgs_backward_zero_sh.restype = ctypes.c_int
    assert lib.fdgs_forward_zero_sh(None, None, None, None, None, None, None, None, None, None, None, None) == 1
    assert b"null" in lib.fdgs_last_error()
    assert lib.fdgs_backward_zero_sh(None, None, None, 1, None) == 1
