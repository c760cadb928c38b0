"""The training step as one CUDA graph against the eager batched step, at tools/bench_batch.py's workloads.

    python tools/bench_graph.py [--steps 30] [--warmup 5] [--only lego-400,trex]

For each workload (lego-800, lego-400, hook, trex, dynerf, dynerf-sky: dynerf with a 500^2 environment map) the same
seeded scene and cameras run two arms, alternating step by step:
  eager  render_batch(cams) -> the B fused L1/SSIM losses -> one backward() (with a map: the per-view sky sampler)
  graph  fdgs.graph.GraphedStep around the same step over StaticViews: one graph replay + one status read
Reported per workload: the median CUDA-event step time of each arm, the median host time to enqueue a step (the host
clock from the call until it returns, without the graph's final status read, i.e. the time the host needs before the
GPU could start on the next step), the capture time, the graph's peak memory above the resident scene (its private
pool, including the capacity margin) against the eager step's, the re-captures and overflows, and the capacity.  Then
the eager tile_sort_pack stage time of the capacity path (both sort size classes always launched) against the exact
path at trex and cfg3.  One JSON line each, with the GPU's name, power limit and max SM clock read in the same process.
Writes nothing into the tree.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "4d-gaussian-splatting_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle"),
          os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_batch import DEV, WORKLOADS as BATCH_WORKLOADS, _Pipe, _setup, gpu_info  # noqa: E402

WORKLOADS = {n: BATCH_WORKLOADS[n] for n in ("lego-800", "lego-400", "hook", "trex", "dynerf", "dynerf-sky")}


def _step_fn(pc, pipe, bg):
    from gaussian_renderer import render_batch
    from fdgs.loss import l1_ssim_loss

    def step(views, gt):
        pkg = render_batch(views, pc, pipe, bg)
        loss = sum(l1_ssim_loss(pkg["render"][k], gt[k]) for k in range(gt.shape[0]))
        loss.backward()
        return loss, pkg
    return step


def bench(name, w, steps, warmup):
    from fdgs.graph import GraphedStep, _leaves
    pc, cams, gts = _setup(w)
    pipe, bg = _Pipe(w.get("sky")), torch.zeros(3, device=DEV)
    gt = torch.stack(gts)
    fn = _step_fn(pc, pipe, bg)
    out = {"workload": name, "P": w["P"], "W": w["W"], "H": w["H"], "B": w["B"]}

    def zero():
        for p in pc.leaves():
            p.grad = None

    # eager arm: warm-up and peak memory
    for _ in range(warmup):
        zero()
        fn(cams, gt)
    zero()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn(cams, gt)
    torch.cuda.synchronize()
    out["eager_peak_extra_MB"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
    zero()
    torch.cuda.synchronize()

    # graph arm: the first call warms up, sizes the capacity and captures
    if w.get("sky"):
        # the graph steps a learned map only as the "env_map" group of the model's FusedAdam (its gradient must be
        # one of the step's leaves)
        from bench_graph_iteration import _model
        params = _model(pc)
    else:
        params = pc.leaves
    leaves = lambda: _leaves(params)     # noqa: E731  (the order GraphedStep's calls use)
    step = GraphedStep(fn, params)
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    step(cams, gt)
    torch.cuda.synchronize()
    out["first_call_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
    out["graph_peak_extra_MB"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
    t0 = time.perf_counter()
    step._capture(leaves())     # a capture alone (the graph is rebuilt in place; the next call replays it)
    torch.cuda.synchronize()
    out["capture_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
    step._replay(leaves())
    for _ in range(warmup):
        step(cams, gt)

    times = {"eager": [], "graph": []}
    enqueue = {"eager": [], "graph": []}
    for _ in range(steps):
        # eager
        zero()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        h0 = time.perf_counter()
        fn(cams, gt)
        enqueue["eager"].append(1e3 * (time.perf_counter() - h0))
        e1.record()
        e1.synchronize()
        times["eager"].append(e0.elapsed_time(e1))
        # graph: load + replay, timed without the closing status read for the enqueue time
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        h0 = time.perf_counter()
        step.views.load(cams)
        step.gt.copy_(gt)
        step._graph.replay()
        enqueue["graph"].append(1e3 * (time.perf_counter() - h0))
        e1.record()
        e1.synchronize()
        times["graph"].append(e0.elapsed_time(e1))
        step(cams, gt)     # the full call (status read, re-capture on overflow) between timed replays
    for arm in times:
        out[arm + "_ms"] = round(statistics.median(times[arm]), 3)
        q = sorted(times[arm])
        out[arm + "_ms_iqr"] = [round(q[len(q) // 4], 3), round(q[(3 * len(q)) // 4], 3)]
        out[arm + "_enqueue_ms"] = round(statistics.median(enqueue[arm]), 3)
    out["speedup"] = round(out["eager_ms"] / out["graph_ms"], 3)
    out.update(captures=step.info["captures"], overflows=step.info["overflows"], capacity=step.info["capacity"],
               R=int(step._out[1]["status"][0]))
    return out


def sort_stage(name, reps=20):
    """tile_sort_pack stage time of eager calls of the exact entry and of the capacity entry (capacity = 1.25 R)."""
    import helpers
    import fdgs
    from fdgs.graph import StaticViews
    from gaussian_renderer import render_batch
    if name in WORKLOADS:
        pc, cams, _ = _setup(WORKLOADS[name])
    else:
        from bench_batch import _RawModel
        cfg, cam, sc, _ = helpers.build(name, device=DEV)
        pc, cams = _RawModel(sc), [cam.to(DEV)]
    pipe, bg = _Pipe(False), torch.zeros(3, device=DEV)
    views = StaticViews(len(cams), int(cams[0].image_height), int(cams[0].image_width), DEV)
    views.load(cams)
    R = int(render_batch(views, pc, pipe, bg)["status"][0])
    views.capacity = int(1.25 * R) + 1
    out = {"workload": name, "stage": "tile_sort_pack", "R": R, "B": len(cams)}
    for arm, src in (("exact", cams), ("capacity", views)):   # forwards only; each call's autograd graph is dropped
        for _ in range(3):
            render_batch(src, pc, pipe, bg)
        torch.cuda.synchronize()
        fdgs.profile_read()
        fdgs.profile_enable(True)
        for _ in range(reps):
            render_batch(src, pc, pipe, bg)
        torch.cuda.synchronize()
        fdgs.profile_enable(False)
        ms, calls = fdgs.profile_read()["tile_sort_pack"]
        out[arm + "_ms"] = round(ms / max(1, calls), 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", default="")
    ap.add_argument("--no-sort", action="store_true", help="skip the tile_sort_pack stage comparison")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_graph: no CUDA device")
    names = [n for n in WORKLOADS if not args.only or n in args.only.split(",")]
    info = gpu_info()
    for n in names:
        r = bench(n, WORKLOADS[n], args.steps, args.warmup)
        r.update(info)
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()
    if not args.no_sort:
        for n in ("trex", "cfg3"):
            r = sort_stage(n)
            r.update(info)
            print(json.dumps(r), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
