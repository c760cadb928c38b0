"""Environment-map sky: the native path (sky kernel + composition inside the rasterizer) against the PyTorch composition
it replaced (Camera.get_rays + grid_sample + `rendered + (1 - alpha) * sky`), on the cfg5 workload -- 300k Gaussians,
1352x1014, duration [0,10], posed N3V-style camera -- with a 500x500 environment map, render() + a colour-only loss +
backward per step.

The two arms alternate inside one process (warm-up, then timed steps with CUDA events).  A separate torch.profiler run
of each arm names the blend-backward instantiation it ran and the kernel times of the sky; a third run times the
sky sampler's kernels alone.  Prints the card name and power limit with the numbers.

    python tools/bench_sky.py --steps 50 --warmup 10 [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "4d-gaussian-splatting_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import helpers  # noqa: E402
import sky_ref  # noqa: E402
from fdgs import synth  # noqa: E402
from raw_model import RawModel, Pipe  # noqa: E402

DEV = "cuda:0"


class SkyPipe(Pipe):
    env_map_res = 500


class NoSkyPipe(Pipe):
    env_map_res = 0


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still reported, with the query's failure beside them
        q = "unknown (%s)" % e
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_sky.py measures on a GPU"
    from gaussian_renderer import render

    cfg, _, sc, _ = helpers.build("cfg5", device=DEV)
    R, T = synth.pose_from_euler(*cfg["pose"])
    cam = sky_ref.SkyCamera(cfg["W"], cfg["H"], R=R, T=T, timestamp=cfg["timestamp"], device=DEV)
    model = RawModel(sc, seed=1, requires_grad=True)
    model.env_map = torch.rand(3, 500, 500, generator=torch.Generator().manual_seed(5)).to(DEV).requires_grad_(True)
    G = torch.randn(3, cfg["H"], cfg["W"], generator=torch.Generator().manual_seed(77)).to(DEV)
    bg = torch.zeros(3, device=DEV)
    leaves = list(model.leaves().values()) + [model.env_map]

    def native():
        pkg = render(cam, model, SkyPipe(), bg)
        (pkg["render"] * G).sum().backward()

    def torch_sky():
        pkg = render(cam, model, NoSkyPipe(), bg)
        img = sky_ref.torch_composition(pkg["render"], pkg["alpha"], sky_ref.torch_sky(model.env_map, cam))
        (img * G).sum().backward()

    arms = {"native": native, "torch": torch_sky}

    def step(fn):
        for t in leaves:
            t.grad = None
        fn()

    for _ in range(args.warmup):
        for fn in arms.values():
            step(fn)
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(args.steps):
        for k, fn in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step(fn)
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b))

    # profiler runs of their own: which blend backward ran, and the sky's kernels
    kernels = {}
    for k, fn in arms.items():
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                step(fn)
            torch.cuda.synchronize()
        per = {}
        for e in prof.key_averages():
            if e.device_type == torch.autograd.DeviceType.CUDA or getattr(e, "self_device_time_total", 0) > 0:
                per[e.key] = (getattr(e, "device_time_total", 0.0) / 3.0 / 1000.0, e.count // 3)
        kernels[k] = {
            "blend_bwd": sorted(n for n in per if "blend_bwd" in n),
            "ms_per_step": {n: round(v[0], 4) for n, v in per.items()
                            if any(s in n for s in ("blend_bwd", "blend_fwd", "sky_", "grid_sampler", "linalg", "atan2", "acos"))},
        }
    # the sky sampler alone, forward and backward
    from fdgs.sky import sky_background
    g = torch.randn(3, cfg["H"], cfg["W"], generator=torch.Generator().manual_seed(3)).to(DEV)
    env = model.env_map.detach().clone().requires_grad_(True)
    for _ in range(5):
        (sky_background(env, cam) * g).sum().backward()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            (sky_background(env, cam) * g).sum().backward()
        torch.cuda.synchronize()
    sky_bwd = {e.key: round(getattr(e, "device_time_total", 0.0) / 20.0 / 1000.0, 4)
               for e in prof.key_averages() if "sky_" in e.key}

    name, limit = card()
    res = {"workload": "cfg5 + env_map 500x500, render + colour-only loss + backward", "card": name,
           "power_limit_and_max_sm_clock": limit, "steps": args.steps, "warmup": args.warmup}
    for k, v in times.items():
        res[k + "_ms_median"] = round(statistics.median(v), 3)
        res[k + "_ms_mean"] = round(statistics.fmean(v), 3)
        res[k + "_ms_min"] = round(min(v), 3)
    res["speedup_median"] = round(res["torch_ms_median"] / res["native_ms_median"], 4)
    res["kernels"] = kernels
    res["sky_backward_ms"] = sky_bwd
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_sky.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
