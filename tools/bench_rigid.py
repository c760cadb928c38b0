"""The rigidity + motion regularisers of train.py:132-159 at lego size (100k) and at 2M Gaussians, k = 20: the reference's
PyTorch expressions (restated in tests/rigid_ref.py, float32) vs the native op (fdgs.regularize), with the SAME
neighbour list in both arms.

Workload: tests/lego.py lego_setup's initial distributions (positions in (-1.3, 1.3)^3, lego's scales and
quaternions), lambda_rigid = 1, lambda_motion = 0.1, upstream gradient 1 / batch (batch 2).  Per size it reports, as
medians over --calls calls after --warmup (CUDA events):
  - reference_ms / native_ms: forward + backward of both losses (velocity, losses, gradients of the four raw tensors)
  - knn_ms: the neighbour search alone (fdgs.knn, grid); neighbours_ms: the list build on top of it (weights, stable
    radix sort by destination, CSR offsets)
  - per-call device times of the native pieces: velocity kernel alone, forward (velocity + loss + total), backward
  - per-kernel device times from torch.profiler (a run of its own, the same number of calls)
  - algorithmic bytes of every native kernel (counted from shapes, gathers counted per access) and the achieved rate
  - peak extra memory (torch.cuda.max_memory_allocated above the inputs) of both arms
The card's name and power limit are read in the same run.  Prints one JSON line.

    python tools/bench_rigid.py [--sizes 100000,2000000] [--calls 20] [--warmup 5] [--out FILE]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "4d-gaussian-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import torch  # noqa: E402

import rigid_ref  # noqa: E402

K, LAMBDA_RIGID, LAMBDA_MOTION, BATCH = 20, 1.0, 0.1, 2
NAMES = ("_scaling", "_scaling_t", "_rotation", "_rotation_r")


class Model:
    rot_4d, gaussian_dim = True, 4

    def __init__(self, p):
        for k, v in p.items():
            setattr(self, k, v)

    get_xyz = property(lambda s: s._xyz)


def make(n, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    u = lambda *s: torch.rand(*s, generator=g, device="cuda")
    nn_ = lambda *s: torch.randn(*s, generator=g, device="cuda")
    p = dict(_xyz=u(n, 3) * 2.6 - 1.3, _t=u(n, 1), _scaling=torch.log(0.012 * (0.5 + u(n, 3))),
             _scaling_t=math.log(math.sqrt(1.0 / 5)) + 0.1 * nn_(n, 1),
             _rotation=torch.nn.functional.normalize(nn_(n, 4), dim=1),
             _rotation_r=torch.nn.functional.normalize(nn_(n, 4), dim=1))
    return {k: v.contiguous().requires_grad_(k in NAMES) for k, v in p.items()}


def algorithmic_bytes(n, k):
    """bytes every native kernel reads and writes, from shapes (a gathered row counted at every access)"""
    params = 4 * (1 + 3 + 1 + 4 + 4)            # t, scaling, scaling_t, rotation, rotation_r
    return {"rigid_weight_kernel": n * k * (4 + 4 + 4),                       # dist2 in, weight + edge id out
            "rigid_offsets_kernel": n * k * 4 + (n + 1) * 4,
            "rigid_velocity_kernel": n * (params + 12),
            "rigid_loss_kernel": n * (12 + k * (4 + 4 + 12)),               # v_i; per edge idx, weight, v_j
            "rigid_bwd_kernel": n * (12 + k * (4 + 4 + 12) + 8 + k * (4 + 4 + 12) + params + 4 * (3 + 1 + 4 + 4))}


def timed(fn, calls, warmup):
    times = []
    for i in range(warmup + calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        if i >= warmup:
            times.append(a.elapsed_time(b))
    return statistics.median(times)


def peak_extra(fn):
    for q in range(2):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        floor = torch.cuda.memory_allocated()
        fn()
        torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - floor) / 2**20


def bench_size(n, calls, warmup):
    import fdgs
    from fdgs import regularize as R
    from fdgs.knn import knn
    C = fdgs.ext()
    p = make(n)
    m = Model(p)
    nb = R.neighbours(p["_xyz"], K)
    idx64 = nb.idx.long()
    params = [p[a].detach() for a in ("_t", "_scaling", "_scaling_t", "_rotation", "_rotation_r")]
    leaves = [p[a] for a in NAMES]

    def reference():
        vel = rigid_ref.velocity(p["_scaling"], p["_scaling_t"], p["_rotation"], p["_rotation_r"], p["_t"])
        lr = rigid_ref.rigid_from_velocity(vel, idx64, nb.dist2, K)
        lm = rigid_ref.motion_from_velocity(vel)
        torch.autograd.grad((LAMBDA_RIGID * lr + LAMBDA_MOTION * lm) / BATCH, leaves)

    def native():
        lr, lm = R.rigidity_and_motion_loss(m, K, nb)
        torch.autograd.grad((LAMBDA_RIGID * lr + LAMBDA_MOTION * lm) / BATCH, leaves)

    xyz = p["_xyz"].detach()
    idx, d2 = C.knn(xyz, K, False)
    vel, lr, lm = C.rigid_forward(params, K, nb.idx, nb.weight, True, True)
    g = torch.full((), LAMBDA_RIGID / BATCH, device="cuda")
    gm = torch.full((), LAMBDA_MOTION / BATCH, device="cuda")
    res = {"n": n, "k": K,
           "reference_ms": timed(reference, calls, warmup), "native_ms": timed(native, calls, warmup),
           "knn_ms": timed(lambda: knn(xyz[None], xyz[None], K), calls, warmup),
           "neighbours_ms": timed(lambda: C.rigid_neighbours(idx, d2), calls, warmup),
           "velocity_call_ms": timed(lambda: C.rigid_forward(params, K, nb.idx, nb.weight, False, False), calls, warmup),
           "forward_call_ms": timed(lambda: C.rigid_forward(params, K, nb.idx, nb.weight, True, True), calls, warmup),
           "backward_call_ms": timed(lambda: C.rigid_backward(params, K, vel, nb.idx, nb.weight, nb.in_offsets, nb.in_edges,
                                                              g, gm), calls, warmup),
           "reference_peak_extra_MB": peak_extra(reference), "native_peak_extra_MB": peak_extra(native),
           "neighbour_list_MB": (nb.weight.numel() * 4 + nb.in_offsets.numel() * 4 + nb.in_edges.numel() * 4) / 2**20,
           "max_in_degree": int(torch.bincount(idx64.flatten(), minlength=n).max())}
    res["speedup"] = res["reference_ms"] / res["native_ms"]

    # per-kernel device time, one profiled run of `calls` list builds and native forward + backward
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            C.rigid_neighbours(idx, d2)
            native()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        name = next((k for k in ("rigid_weight_kernel", "rigid_offsets_kernel", "rigid_velocity_kernel", "rigid_loss_kernel",
                                 "rigid_total_kernel", "rigid_bwd_kernel") if k in e.key), None)
        if name is None and ("Onesweep" in e.key or "RadixSort" in e.key or "radix" in e.key.lower()):
            name = "cub_radix_sort"
        if name:
            kern[name] = kern.get(name, 0.0) + us / 1e3 / calls
    ab = algorithmic_bytes(n, K)
    res["kernel_ms"] = {a: round(b, 4) for a, b in sorted(kern.items())}
    res["kernel_algorithmic_MB"] = {a: round(b / 2**20, 2) for a, b in ab.items()}
    res["kernel_GBps"] = {a: round(ab[a] / (kern[a] * 1e-3) / 1e9, 1) for a in ab if kern.get(a, 0) > 0}
    return {a: (round(b, 4) if isinstance(b, float) else b) for a, b in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100000,2000000")
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rigid needs a GPU")
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        card = torch.cuda.get_device_name(0) + ", power limit not read"
    sizes = [int(s) for s in args.sizes.split(",")]
    res = {"workload": "rigidity + motion regularisers, lego initialisation, k = %d, same neighbour list" % K,
           "card": card, "calls": args.calls, "sizes": [bench_size(n, args.calls, args.warmup) for n in sizes]}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
