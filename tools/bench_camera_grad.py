"""The cost of the camera gradient: the rasterizer backward with and without dL/dviewmatrix, dL/dprojmatrix and dL/dcampos.

    python tools/bench_camera_grad.py [--steps 30] [--warmup 5] [--only cfg3,dynerf]

For each workload one seeded scene is rendered once; then the two arms run its backward, alternating call by call:
  plain    the backward the rasterizer runs when the camera needs no gradient (rasterize_gaussians_backward_ext /
           rasterize_gaussians_backward_batch)
  camera   the same call with the camera gradients (rasterize_gaussians_backward_camera / _batch_camera)
The time is the median of CUDA-event times over --steps calls of each arm.  One JSON line per workload, then the GPU's
name, power limit and max SM clock read in the same process.  Writes nothing into the tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "4d-gaussian-splatting_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

DEV = "cuda:0"
WORKLOADS = {
    "cfg3": dict(P=2000000, W=1352, H=1014, seed=1237, B=1),
    "dynerf": dict(P=300000, W=1352, H=1014, seed=14, B=4, time_duration=10.0, timestamp=4.3, scale_t_mean=1.2),
}


def _gpu_info():
    info = dict(device=torch.cuda.get_device_name(0))
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        pl, clk = [s.strip() for s in r.stdout.strip().split(",")]
        info.update(power_limit=pl, max_sm_clock=clk)
    except Exception as e:       # reported, not fatal: the timings stand with the device name
        info["nvidia_smi"] = "unavailable: %s" % e
    return info


def _arms(cfg):
    """the two backward calls of one workload, as closures over the same forward state"""
    import fdgs
    import helpers
    from fdgs import synth
    from test_gpu_batch import _batch, _inputs, _single
    from test_gpu_view_parallel import _views
    C = fdgs.ext()
    _, cam, sc, st = helpers.build(cfg, device=DEV)
    g = _inputs(sc, False, False)
    e = torch.Tensor([]).to(DEV)
    gc, gd, ga, _ = helpers.pixel_grads(cfg, device=DEV)
    if cfg["B"] == 1:
        fw = _single(st, sc, cfg, g, False, None)
        args = (st["bg"], sc.means3D, fw[10], fw[5], e, sc.flow_2d, g["opacity"], g["ts"], g["scales"], g["scales_t"],
                g["rotations"], g["rotations_r"], 1.0, e, -1.0, st["viewmatrix"], st["projmatrix"], st["tanfovx"],
                st["tanfovy"], gc, gd, ga, e, g["sh"], st["sh_degree"], st["sh_degree_t"], st["campos"], st["timestamp"],
                st["time_duration"], st["rot_4d"], st["gaussian_dim"], st["force_sh_3d"], fw[6], fw[0], fw[7], fw[8],
                False, g["sh_rest"], False, e, False, False, e, e)
        return (lambda: C.rasterize_gaussians_backward_ext(*args)), (lambda: C.rasterize_gaussians_backward_camera(*args))
    cams = _views(cfg, cfg["B"], DEV)
    sts = [synth.raster_settings(c, sc, bg=torch.zeros(3), device=DEV) for c in cams]
    fw = _batch(sts, sc, cfg, g, False, None)
    f32 = lambda k: torch.tensor([s[k] for s in sts], dtype=torch.float32)
    B = cfg["B"]
    rep = lambda t: t.reshape(1, *t.shape).expand(B, *t.shape).contiguous()
    args = (sts[0]["bg"], sc.means3D, fw[9], fw[5], sc.flow_2d, g["opacity"], g["ts"], g["scales"], g["scales_t"],
            g["rotations"], g["rotations_r"], 1.0, -1.0, torch.stack([s["viewmatrix"] for s in sts]),
            torch.stack([s["projmatrix"] for s in sts]), torch.stack([s["campos"] for s in sts]), f32("timestamp"),
            f32("tanfovx"), f32("tanfovy"), rep(gc), rep(gd), rep(ga), e, g["sh"], g["sh_rest"], sts[0]["sh_degree"],
            sts[0]["sh_degree_t"], sts[0]["time_duration"], sts[0]["rot_4d"], sts[0]["gaussian_dim"],
            sts[0]["force_sh_3d"], fw[6], fw[0], fw[7], fw[8], False, False, e, False)
    return (lambda: C.rasterize_gaussians_backward_batch(*args)), (lambda: C.rasterize_gaussians_backward_batch_camera(*args))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_camera_grad needs a GPU")
    names = [n for n in WORKLOADS if not a.only or n in a.only.split(",")]
    for name in names:
        cfg = WORKLOADS[name]
        plain, camera = _arms(cfg)
        for _ in range(a.warmup):
            plain(); camera()
        times = {"plain": [], "camera": []}
        for _ in range(a.steps):
            for arm, fn in (("plain", plain), ("camera", camera)):
                s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                fn()
                t.record()
                torch.cuda.synchronize()
                times[arm].append(s.elapsed_time(t))
        p, c = statistics.median(times["plain"]), statistics.median(times["camera"])
        print(json.dumps(dict(workload=name, P=cfg["P"], W=cfg["W"], H=cfg["H"], B=cfg["B"], steps=a.steps,
                              backward_ms=round(p, 4), backward_camera_ms=round(c, 4), extra_ms=round(c - p, 4),
                              spread_ms=dict(plain=[round(min(times["plain"]), 4), round(max(times["plain"]), 4)],
                                             camera=[round(min(times["camera"]), 4), round(max(times["camera"]), 4)]))))
    print(json.dumps(_gpu_info()))


if __name__ == "__main__":
    main()
