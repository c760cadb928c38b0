"""The evaluation metrics of training_report (train.py:312-334) per test view: the reference's path restated (torch on
the GPU for L1 / PSNR / SSIM, a host copy, MS-SSIM in float32 on the CPU -- torchmetrics itself when it imports, else
tests/metrics_ref.py's restatement of it) vs the native op (fdgs.metrics.image_metrics).

Workload: 3-channel image pairs (uniform noise and a perturbed copy) at 1352x1014 and 800x800.  Per size it reports,
as medians over --calls calls after --warmup, the two arms alternated call by call (host wall clock around the call and
a device synchronisation, since the reference's path ends on the host):
  - reference_ms / native_ms per view, and the speed-up
  - test_set_s: a --views-view test set end to end through MetricAccumulator (one synchronisation at the end);
    the reference's test set is estimated as views x its per-view median (running it would take minutes)
  - per-kernel device times from torch.profiler (a run of its own, --calls views) and the algorithmic bytes of each
    kernel counted from shapes, with the achieved rate
The card's name and power limit and the host's CPU count are read in the same run.  Prints one JSON line.

    python tools/bench_metrics.py [--sizes 1014x1352,800x800] [--calls 20] [--warmup 3] [--views 300] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "4d-gaussian-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import torch  # noqa: E402

import metrics_ref as M  # noqa: E402

POOL = 8     # distinct image pairs, cycled


def cpu_msssim():
    try:
        from torchmetrics import MultiScaleStructuralSimilarityIndexMeasure
        tm = MultiScaleStructuralSimilarityIndexMeasure(data_range=1.0)
        return "torchmetrics", lambda a, b: tm(a, b).item()
    except ImportError:
        return "tests/metrics_ref.py restatement", lambda a, b: M.torch_msssim(a, b).mean().item()


def pairs(H, W):
    g = torch.Generator(device="cuda").manual_seed(0)
    out = []
    for _ in range(POOL):
        y = torch.rand(3, H, W, generator=g, device="cuda")
        x = (y + 0.05 * torch.randn(3, H, W, generator=g, device="cuda")).contiguous()
        out.append((x, y))
    return out


def algorithmic_bytes(H, W):
    """bytes per view: level 1 reads both fp32 images and writes level 2 of both in float64; level s (2..5) reads its
    two float64 planes and writes the next level; partials and the finalize are counted too"""
    lv, h, w = [], H, W
    for _ in range(5):
        lv.append((h, w))
        h, w = h // 2, w // 2
    tiles = sum(((a + 31) // 32) * ((b + 31) // 32) for a, b in lv)
    first = 3 * (2 * 4 * H * W + 2 * 8 * lv[1][0] * lv[1][1])
    rest = sum(3 * (2 * 8 * lv[s][0] * lv[s][1] + (2 * 8 * lv[s + 1][0] * lv[s + 1][1] if s < 4 else 0)) for s in range(1, 5))
    part = 3 * tiles * 5 * 8
    return {"level1": first, "levels2to5": rest, "finalize": part + 4 * 8}


def bench_size(H, W, calls, warmup, views):
    from fdgs import metrics
    ms_name, ms_cpu = cpu_msssim()
    pool = pairs(H, W)

    def reference(i):
        x, y = pool[i % POOL]
        image = torch.clamp(x, 0.0, 1.0)
        l1 = (image - y).abs().mean().double()
        mse = ((image - y) ** 2).view(3, -1).mean(1, keepdim=True)
        psnr = (20 * torch.log10(1.0 / torch.sqrt(mse))).mean().double()
        ssim = M.torch_ssim(image[None], y[None]).mean().double()
        ms = ms_cpu(image[None].cpu(), y[None].cpu())
        return l1, psnr, ssim, ms

    def native(i):
        x, y = pool[i % POOL]
        return metrics.image_metrics(x, y, clamp=True)

    ref_t, nat_t = [], []
    with M.no_tf32():
        for i in range(warmup + calls):
            for fn, ts in ((reference, ref_t), (native, nat_t)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn(i)
                torch.cuda.synchronize()
                if i >= warmup:
                    ts.append((time.perf_counter() - t0) * 1e3)
    res = {"H": H, "W": W, "msssim_reference": ms_name,
           "reference_ms": statistics.median(ref_t), "native_ms": statistics.median(nat_t)}
    res["speedup"] = res["reference_ms"] / res["native_ms"]

    acc = metrics.MetricAccumulator()
    acc.add(*pool[0])
    acc.result()
    t0 = time.perf_counter()
    acc = metrics.MetricAccumulator()
    for i in range(views):
        acc.add(*pool[i % POOL])
    acc.result()
    res["views"] = views
    res["native_test_set_s"] = time.perf_counter() - t0
    res["reference_test_set_s_estimated"] = views * res["reference_ms"] / 1e3

    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        acc = metrics.MetricAccumulator()
        for i in range(calls):
            acc.add(*pool[i % POOL])
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        name = None
        if "ms_scale_kernel" in e.key:
            name = "level1" if "<true" in e.key or "ILb1E" in e.key else "levels2to5"
        elif "ms_finalize_kernel" in e.key:
            name = "finalize"
        elif "ms_accumulate_kernel" in e.key:
            name = "accumulate"
        if name:
            kern[name] = kern.get(name, 0.0) + us / 1e3 / calls
    ab = algorithmic_bytes(H, W)
    res["kernel_ms"] = {a: round(b, 4) for a, b in sorted(kern.items())}
    res["kernel_algorithmic_MB"] = {a: round(b / 2**20, 2) for a, b in ab.items()}
    res["kernel_GBps"] = {a: round(ab[a] / (kern[a] * 1e-3) / 1e9, 1) for a in ab if kern.get(a, 0) > 0}
    return {a: (round(b, 4) if isinstance(b, float) else b) for a, b in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1014x1352,800x800")
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--views", type=int, default=300)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_metrics needs a GPU")
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        card = torch.cuda.get_device_name(0) + ", power limit not read"
    sizes = [tuple(int(v) for v in s.split("x")) for s in args.sizes.split(",")]
    res = {"workload": "training_report metrics per view (L1, PSNR, SSIM, MS-SSIM), 3 channels, clamp on",
           "card": card, "host_cpus": os.cpu_count(), "torch_threads": torch.get_num_threads(), "calls": args.calls,
           "sizes": [bench_size(H, W, args.calls, args.warmup, args.views) for H, W in sizes]}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
