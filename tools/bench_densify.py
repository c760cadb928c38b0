"""Densify-and-prune at cfg3 size: the reference's PyTorch surgery (restated in tests/densify_ref.py) vs the native
compaction (fdgs.densify), on the same model and generator state.

Workload: 2M Gaussians, gaussian_dim 4 with rot_4d, M = 48 SH coefficients, Adam moments present; 1 % of the rows
are selected for cloning, 1 % for splitting (N = 2), 0.5 % have an opacity under the prune threshold -- roughly what a
densification step of a trained scene selects.  Every timed call runs on a fresh copy of the model (the copy is not
timed).  Reports per arm the median over --calls calls (CUDA events, after --warmup calls), the peak of
torch.cuda.max_memory_allocated above the model's own footprint, and for the native arm the achieved bandwidth over the
algorithmic bytes (every parameter and moment float of the P source rows read once and of the P_new result rows
written once) twice: over the whole op (plan, the totals' read, the samples, allocation, Python) and over the device
time of the compaction kernels alone (torch.profiler, one call of its own).  Prints one JSON line.

    python tools/bench_densify.py [--P 2000000] [--calls 20] [--warmup 3] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "4d-gaussian-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import torch  # noqa: E402
from torch import nn  # noqa: E402

import densify_ref as R  # noqa: E402

EXTENT, MAX_GRAD, MIN_OPACITY = 4.0, 2e-4, 0.005


def make(P, M, seed=0):
    from fdgs.optim import FusedAdam
    g = torch.Generator(device="cuda").manual_seed(seed)
    m = R.Model()
    m.gaussian_dim, m.rot_4d, m.percent_dense = 4, True, 0.01
    dense = m.percent_dense * EXTENT
    u = torch.rand(P, device="cuda", generator=g)
    clone, split, low = u < 0.01, (u >= 0.01) & (u < 0.02), (u >= 0.02) & (u < 0.025)
    smax = torch.where(split, 4.0 * dense, 0.5 * dense)
    m._scaling = (torch.log(smax)[:, None] - torch.rand(P, 3, device="cuda", generator=g)).contiguous()
    m._scaling[:, 0] = torch.log(smax)
    m._xyz = torch.randn(P, 3, device="cuda", generator=g)
    m._features_dc = torch.randn(P, 1, 3, device="cuda", generator=g)
    m._features_rest = torch.randn(P, M - 1, 3, device="cuda", generator=g) * 0.1
    m._opacity = torch.where(low, -8.0, 0.5)[:, None].contiguous()
    m._rotation = torch.randn(P, 4, device="cuda", generator=g)
    m._t = torch.randn(P, 1, device="cuda", generator=g)
    m._scaling_t = torch.full((P, 1), -2.0, device="cuda")
    m._rotation_r = torch.randn(P, 4, device="cuda", generator=g)
    m.denom = torch.ones(P, 1, device="cuda")
    m.xyz_gradient_accum = torch.where(clone | split, 1e-3, 1e-5)[:, None].contiguous()
    m.t_gradient_accum = torch.zeros(P, 1, device="cuda")
    m.max_radii2D = torch.zeros(P, device="cuda")
    names = m.group_names()
    for n in names:
        setattr(m, R.ATTR[n], nn.Parameter(getattr(m, R.ATTR[n]).requires_grad_(True)))
    m.optimizer = FusedAdam([{"params": [getattr(m, R.ATTR[n])], "lr": 1e-3, "name": n} for n in names], lr=0.0, eps=1e-15)
    for n in names:
        p = getattr(m, R.ATTR[n])
        p.grad = torch.full_like(p, 1e-3)
    m.optimizer.step()
    for n in names:
        getattr(m, R.ATTR[n]).grad = None
    return m


def floats_per_row(m):
    return sum(3 * getattr(m, R.ATTR[n])[0].numel() for n in m.group_names())   # parameter + two moments


def run(arm, base, calls, warmup):
    from fdgs import densify as D
    times, peaks, p_new = [], [], None
    for i in range(warmup + calls):
        m = R.clone_model(base)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        floor = torch.cuda.memory_allocated()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.manual_seed(1234)
        a.record()
        if arm == "reference":
            with torch.no_grad():
                R.ref_densify_and_prune(m, MAX_GRAD, MIN_OPACITY, EXTENT, None)
        else:
            D.densify_and_prune(m, MAX_GRAD, MIN_OPACITY, EXTENT, None)
        b.record()
        torch.cuda.synchronize()
        if i >= warmup:
            times.append(a.elapsed_time(b))
            peaks.append(torch.cuda.max_memory_allocated() - floor)
        p_new = m._xyz.shape[0]
        del m
    return statistics.median(times), max(peaks), p_new


def apply_kernel_ms(base):
    """Device time of the compaction kernels (densify_apply_kernel + densify_positions_kernel) in one native call,
    from torch.profiler in a run of its own."""
    from torch.profiler import ProfilerActivity, profile
    from fdgs import densify as D
    m = R.clone_model(base)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        D.densify_and_prune(m, MAX_GRAD, MIN_OPACITY, EXTENT, None)
        torch.cuda.synchronize()
    us = 0.0
    for e in prof.key_averages():
        if "densify_apply_kernel" in e.key or "densify_positions_kernel" in e.key:
            us += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
    return us / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=2_000_000)
    ap.add_argument("--M", type=int, default=48)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_densify needs a GPU")
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        card = torch.cuda.get_device_name(0) + ", power limit not read"
    base = make(args.P, args.M)
    t_ref, mem_ref, p_ref = run("reference", base, args.calls, args.warmup)
    t_nat, mem_nat, p_nat = run("native", base, args.calls, args.warmup)
    assert p_ref == p_nat, (p_ref, p_nat)
    t_kern = apply_kernel_ms(base)
    algo_bytes = 4 * floats_per_row(base) * (args.P + p_nat)
    res = {"workload": "densify_and_prune P=%d M=%d rot_4d, 1%% clone 1%% split 0.5%% prune" % (args.P, args.M),
           "card": card, "P_after": p_nat, "calls": args.calls,
           "reference_ms": round(t_ref, 3), "native_ms": round(t_nat, 3), "speedup": round(t_ref / t_nat, 2),
           "reference_peak_extra_MB": round(mem_ref / 2**20, 1), "native_peak_extra_MB": round(mem_nat / 2**20, 1),
           "native_algorithmic_GB": round(algo_bytes / 1e9, 3),
           "native_op_GBps": round(algo_bytes / (t_nat * 1e-3) / 1e9, 1),
           "compaction_kernels_ms": round(t_kern, 3),
           "compaction_kernels_GBps": round(algo_bytes / (t_kern * 1e-3) / 1e9, 1) if t_kern > 0 else None}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
