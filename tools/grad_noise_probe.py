"""Error of our gradients against the mean of K reference reruns, in units of the reference's own run-to-run spread.
usage: python tools/grad_noise_probe.py <config> [aux|colour]   (env: FDGS_TILE_CULL)"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "4d-gaussian-splatting_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch
import helpers
import oracle_py
import fdgs

name = sys.argv[1] if len(sys.argv) > 1 else "mid_rotcam"
aux = (sys.argv[2] if len(sys.argv) > 2 else "aux") == "aux"
K = 8
C, ref = fdgs.ext(), oracle_py.ref_module()
cfg, cam, sc, st = helpers.build(name, device="cuda:0")
gc, gd, ga, gf = helpers.pixel_grads(cfg, device="cuda:0")
up = (gc, gd, ga, gf) if aux else (gc, 0 * gd, 0 * ga, 0 * gf)
e = torch.empty(0, device="cuda:0")
fw = C.rasterize_gaussians(*helpers.fwd_args(st, sc, cfg))
rf = ref.rasterize_gaussians(*helpers.fwd_args(st, sc, cfg))
ours = [C.rasterize_gaussians_backward(*helpers.bwd_args(st, sc, cfg, fw, up if aux else (gc, e, e, e))) for _ in range(3)]
runs = [ref.rasterize_gaussians_backward(*helpers.bwd_args(st, sc, cfg, rf, up)) for _ in range(K)]
print("%s %s tile_cull=%s R=%d (ref %d)" % (name, "aux" if aux else "colour", os.environ.get("FDGS_TILE_CULL", "1"),
                                            fw[0], rf[0]))
for k, g in enumerate(helpers.GRAD_NAMES):
    if runs[0][k].numel() == 0:
        continue
    m = torch.stack([r[k].double() for r in runs]).mean(0)
    nm = m.norm().item()
    if nm == 0:
        continue
    spread = (sum(((r[k].double() - m).norm().item() / nm) ** 2 for r in runs) / K) ** 0.5
    errs = [((o[k].double() - m).norm().item() / nm) for o in ours]
    print("  %-14s ours-vs-mean %s   ref spread %.2e   ratio %.1f" % (g, " ".join("%.2e" % x for x in errs), spread, errs[0] / max(spread, 1e-30)))
