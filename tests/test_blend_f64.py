"""CPU: the regime scenes of regimes.py reach their regimes, and the float64 restatement of the blend (blend_f64.py)
agrees with the CPU oracle on every scene's 3D twin -- images to 1e-5 and the six gradients to 1e-4 (relative L2)
outside the ambiguous pixels and the rows under the frustum clamp."""
import numpy as np
import pytest

import blend_f64
import helpers
import oracle_py
import regimes


@pytest.fixture(scope="module", params=list(regimes.SCENES))
def scene(request):
    name = request.param
    cfg, cam, sc, st = regimes.build(name)
    f = oracle_py.forward(helpers.oracle_inputs(st, sc, cfg))
    return name, cfg, sc, st, f


def test_preconditions(scene):
    name, cfg, sc, st, f = scene
    print(name, regimes.preconditions(name, cfg, sc, st, f))


@pytest.mark.parametrize("aux", [False, True], ids=["colour", "all"])
def test_f64_restatement_vs_oracle(scene, aux):
    name, cfg, sc, st, f = scene
    rows, st3, t = regimes.twin(cfg, sc, st, f)
    inp = regimes.twin_oracle_inputs(st3, t)
    ft = oracle_py.forward(inp)
    # the twin projects to the same screen-space Gaussians as the original
    assert helpers.bitdiff(ft["means2D"], f["means2D"][rows]) == 0
    assert helpers.bitdiff(ft["conic_opacity"], f["conic_opacity"][rows]) == 0
    gc, gd, ga, gf = (helpers.to_np(x) for x in helpers.pixel_grads(cfg))
    up = (gc, gd, ga, gf) if aux else (gc, None, None, None)
    # fp32 inverts the dilated 2D covariance with det = a c - b^2: a needle (det << a c) loses log2(a c / det) bits there,
    # and every fp32 implementation inherits that.  Pixels where such a row may blend are masked like the ambiguous ones;
    # their images are compared with an allowance of the worst loss among those rows, everything else at the plain bars
    ill, loss_rows = blend_f64.ill_conditioned(ft["conic_opacity"])
    r = blend_f64.forward_backward(st3, regimes.f64_lists(ft), t, up, ill=ill)
    keep = ~(r["ambiguous"] | r["ill"])
    loss = float(loss_rows[ill].max(initial=1.0))
    print("%s: %d of %d pixels ambiguous, %d where one of %d ill-conditioned conics blends (loss x%.1f), %d rows under "
          "the frustum clamp" % (name, int(r["ambiguous"].sum()), keep.size, int(r["ill"].sum()), int(ill.sum()), loss,
                                 int(r["frustum_clamp"].sum())))
    illp = r["ill"] & ~r["ambiguous"]
    for key, img in (("color", ft["color"]), ("depth", ft["depth"]), ("alpha", ft["alpha"]), ("flow", ft["flow"])):
        e = helpers.l2_rel(img[..., keep], r["images"][key][..., keep])
        e_ill = helpers.l2_rel(img[..., illp], r["images"][key][..., illp]) if illp.any() else 0.0
        print("  image %-6s l2 %.2e (bar 1e-5); at ill-conditioned pixels %.2e (bar %.1e)" % (key, e, e_ill, 1e-5 * loss))
        assert e < 1e-5, (key, e)
        assert e_ill < 1e-5 * loss, (key, e_ill)
    z = lambda g: np.zeros_like(gd) if g is None else g
    gi = r["grads_in"]
    go = oracle_py.backward(inp, ft, gi[0], z(gi[1]), z(gi[2]), z(gi[3]) if gi[3] is not None else np.zeros_like(gf))
    ok = ~r["frustum_clamp"]
    for key in ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dflows"):
        e = helpers.l2_rel(go[key][ok], r["grads"][key][ok])
        print("  %-12s l2 %.2e (bar 1e-4)" % (key, e))
        assert e < 1e-4, (key, e)
