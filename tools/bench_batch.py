"""Batched views against the sequential view loop: one training step's rasterizer work at the reference's batch shapes.

    python tools/bench_batch.py [--steps 30] [--warmup 5] [--only lego-800,trex]

For each workload the same seeded scene and cameras are rendered by two arms, alternating step by step:
  loop   for every view: render() -> fused L1/SSIM loss -> backward()      (the reference's train.py:104-166)
  batch  render_batch() -> the B per-view losses -> one backward()
The step time is the median of CUDA-event times over --steps steps.  Per step the script also reports the kernels the
library launched (fdgs_launch_count), the host synchronisations (one per forward call by construction: B for the loop,
1 for the batch) and each arm's peak memory above the resident scene.  One JSON line per workload, then the GPU's name,
power limit and max SM clock read in the same process.  Writes nothing into the tree.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "4d-gaussian-splatting_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

DEV = "cuda:0"

# the reference's training shapes (configs/*: batch_size, resolution) on synthetic scenes of its Gaussian counts
WORKLOADS = {
    "lego-800": dict(P=100000, W=800, H=800, B=2, seed=11),
    "lego-400": dict(P=100000, W=400, H=400, B=2, seed=11),
    "hook": dict(P=300000, W=400, H=400, B=8, seed=12),
    "trex": dict(P=300000, W=400, H=400, B=24, seed=13),
    "dynerf": dict(P=300000, W=1352, H=1014, B=4, seed=14, time_duration=10.0, timestamp=4.3, scale_t_mean=1.2),
    "dynerf-sky": dict(P=300000, W=1352, H=1014, B=4, seed=14, time_duration=10.0, timestamp=4.3, scale_t_mean=1.2,
                       sky=True),
}


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False

    def __init__(self, sky):
        self.env_map_res = 500 if sky else 0


class _RawModel:
    """The reference GaussianModel's raw parameters (the configuration train.py renders through the raw entry)."""

    def __init__(self, sc, env=None):
        leaf = lambda t: t.detach().clone().contiguous().requires_grad_(True)
        self._xyz, self._t = leaf(sc.means3D), leaf(sc.ts)
        self._scaling, self._scaling_t = leaf(sc.scales.log()), leaf(sc.scales_t.log())
        self._rotation, self._rotation_r = leaf(sc.rotations), leaf(sc.rotations_r)
        self._opacity = leaf(torch.logit(sc.opacities))
        self._features_dc, self._features_rest = leaf(sc.shs[:, :1]), leaf(sc.shs[:, 1:])
        self.scaling_activation, self.opacity_activation, self.rotation_activation = torch.exp, torch.sigmoid, F.normalize
        self.active_sh_degree, self.active_sh_degree_t = sc.sh_degree, sc.sh_degree_t
        self.time_duration = [0.0, sc.time_duration]
        self.rot_4d, self.gaussian_dim, self.force_sh_3d, self.prefilter_var = sc.rot_4d, sc.gaussian_dim, sc.force_sh_3d, -1.0
        self.env_map = leaf(env) if env is not None else None

    @property
    def get_xyz(self):
        return self._xyz

    def leaves(self):
        out = [self._xyz, self._t, self._scaling, self._scaling_t, self._rotation, self._rotation_r, self._opacity,
               self._features_dc, self._features_rest]
        return out + ([self.env_map] if self.env_map is not None else [])


def _setup(w):
    from fdgs import synth
    import sky_ref
    cam0 = synth.make_camera(w["W"], w["H"], timestamp=w.get("timestamp", 0.5))
    sc = synth.make_scene(w["P"], cam0, w["seed"], time_duration=w.get("time_duration", 1.0),
                          scale_t_mean=w.get("scale_t_mean", 0.15)).to(DEV)
    env = torch.rand(3, 500, 500, generator=torch.Generator().manual_seed(5)).to(DEV) if w.get("sky") else None
    cams, gts = [], []
    dur = w.get("time_duration", 1.0)
    for v in range(w["B"]):
        R, T = synth.pose_from_euler(2.0 * v, -1.0 * v, 0.0, 0.05 * v, 0.0, -0.03 * v)
        ts = w.get("timestamp", 0.5) + 0.07 * dur * (v - 0.5 * w["B"]) / max(1, w["B"] / 4)
        if w.get("sky"):
            cams.append(sky_ref.SkyCamera(w["W"], w["H"], R=R, T=T, timestamp=ts, device=DEV))
        else:
            cams.append(synth.make_camera(w["W"], w["H"], timestamp=ts, R=R, T=T).to(DEV))
        gts.append(torch.rand(3, w["H"], w["W"], generator=torch.Generator().manual_seed(100 + v)).to(DEV))
    return _RawModel(sc, env), cams, gts


def _loop_step(pc, pipe, cams, gts, bg):
    from gaussian_renderer import render
    from fdgs.loss import l1_ssim_loss
    for cam, gt in zip(cams, gts):
        pkg = render(cam, pc, pipe, bg)
        l1_ssim_loss(pkg["render"], gt).backward()


def _batch_step(pc, pipe, cams, gts, bg):
    from gaussian_renderer import render_batch
    from fdgs.loss import l1_ssim_loss
    pkg = render_batch(cams, pc, pipe, bg)
    sum(l1_ssim_loss(pkg["render"][k], gt) for k, gt in enumerate(gts)).backward()


def _zero(pc):
    for p in pc.leaves():
        p.grad = None


def bench(name, w, steps, warmup):
    import fdgs
    lib = fdgs.lib()
    lib.fdgs_launch_count.restype = ctypes.c_longlong
    pc, cams, gts = _setup(w)
    pipe, bg = _Pipe(w.get("sky")), torch.zeros(3, device=DEV)
    arms = {"loop": _loop_step, "batch": _batch_step}
    out = {"workload": name, "P": w["P"], "W": w["W"], "H": w["H"], "B": w["B"]}
    for arm, fn in arms.items():      # warm-up, launches and peak memory, one arm at a time
        for _ in range(warmup):
            _zero(pc)
            fn(pc, pipe, cams, gts, bg)
        _zero(pc)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        n0 = lib.fdgs_launch_count()
        fn(pc, pipe, cams, gts, bg)
        torch.cuda.synchronize()
        out[arm + "_launches"] = int(lib.fdgs_launch_count() - n0)
        out[arm + "_peak_extra_MB"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
        out[arm + "_host_syncs"] = w["B"] if arm == "loop" else 1
    times = {a: [] for a in arms}
    for _ in range(steps):
        for arm, fn in arms.items():   # alternating: both arms see the same drift of the shared machine
            _zero(pc)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn(pc, pipe, cams, gts, bg)
            e1.record()
            e1.synchronize()
            times[arm].append(e0.elapsed_time(e1))
    for arm in arms:
        out[arm + "_ms"] = round(statistics.median(times[arm]), 3)
        q = sorted(times[arm])
        out[arm + "_ms_iqr"] = [round(q[len(q) // 4], 3), round(q[(3 * len(q)) // 4], 3)]
    out["speedup"] = round(out["loop_ms"] / out["batch_ms"], 3)
    return out


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        pl, clk = [s.strip() for s in r.stdout.strip().split(",")]
        info.update(power_limit=pl, max_sm_clock=clk)
    except Exception as e:       # reported, not fatal: the timings stand with the device name
        info["nvidia_smi"] = "unavailable: %s" % e
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_batch: no CUDA device")
    names = [n for n in WORKLOADS if not args.only or n in args.only.split(",")]
    info = gpu_info()
    for n in names:
        r = bench(n, WORKLOADS[n], args.steps, args.warmup)
        r.update(info)
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
