"""The whole training iteration as one CUDA graph against the graphed step with an eager tail, at tools/bench_batch.py's
workloads.

    python tools/bench_graph_iteration.py [--iters 20] [--rounds 15] [--warmup 5] [--only lego-400,trex]

For each workload (lego-800, lego-400, hook, trex, dynerf, lego-400-rigid: lego-400 with the rigidity loss, k = 20,
its neighbour list rebuilt inside the step, and dynerf-sky: dynerf with a learned 500^2 environment map) two copies of
the same seeded scene, each with a FusedAdam over nine named groups (with a map, a tenth, "env_map", at the features'
learning rate) and the densification accumulators, run two arms in alternating blocks of iterations:
  eager-tail  GraphedStep(fn) -> ViewBatchStats + B add_view + add_densification_stats -> FusedAdam.step() -> zero_grad
              (the INTEGRATION loop before the optimiser joined the graph)
  eager       (dynerf-sky, in place of eager-tail: before this graph took a map) fn(cams, gt) eagerly, render_batch
              over the camera list with the per-view sky sampler, then the same tail; the one FusedAdam step is both
              the Gaussians' and the map's Adam step
  graph       GraphedStep(fn, optimizer=FusedAdam)(cams, gt, densify_stats=True): statistics and Adam in the capture
Both set the xyz learning rate every iteration.  fn = render_batch + B fused L1/SSIM losses (+ the rigidity loss) +
backward.  Reported per workload: the median iteration time of each arm (host clock over a block of iterations ending in
a device synchronise, divided by the block length) with its inter-quartile range over the blocks, the median host time
to enqueue one iteration (inputs, staging and replay, plus for eager-tail the statistics and optimiser launches; the
status read is excluded; not given for the eager arm, which synchronises inside its forward), captures and overflows, and the peak memory of the first iteration above the resident scene.
Then, in a separate profiled run, the fused Adam kernel's time per step, eager (adam_kernel) against staged
(adam_staged_kernel), from torch.profiler.  One JSON line each, with the GPU's name, power limit and max SM clock read in
the same process.  Writes nothing into the tree.
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

WORKLOADS = {n: BATCH_WORKLOADS[n] for n in ("lego-800", "lego-400", "hook", "trex", "dynerf")}
WORKLOADS["lego-400-rigid"] = dict(BATCH_WORKLOADS["lego-400"], rigid=20)
WORKLOADS["dynerf-sky"] = BATCH_WORKLOADS["dynerf-sky"]
GROUPS = [("xyz", "_xyz", 1.6e-4), ("t", "_t", 1.6e-4), ("f_dc", "_features_dc", 2.5e-3),
          ("f_rest", "_features_rest", 2.5e-3 / 20), ("opacity", "_opacity", 5e-2), ("scaling", "_scaling", 5e-3),
          ("scaling_t", "_scaling_t", 5e-3), ("rotation", "_rotation", 1e-3), ("rotation_r", "_rotation_r", 1e-3)]


def _model(m):
    """bench_batch's raw-parameter model, given the reference's optimiser groups (configs/dnerf/lego.yaml:36-44) and
    densification accumulators."""
    from fdgs.optim import FusedAdam
    m.optimizer = FusedAdam([{"params": [getattr(m, a)], "lr": lr, "name": n} for n, a, lr in GROUPS], lr=0.0, eps=1e-15)
    if m.env_map is not None:      # the reference's Adam([env_map], lr=feature_lr, eps=1e-15)
        m.optimizer.add_param_group({"params": [m.env_map], "lr": 2.5e-3, "name": "env_map"})
    P = m._xyz.shape[0]
    m.xyz_gradient_accum, m.t_gradient_accum = torch.zeros(P, 1, device=DEV), torch.zeros(P, 1, device=DEV)
    m.denom, m.max_radii2D = torch.zeros(P, 1, device=DEV), torch.zeros(P, device=DEV)
    return m


def _fn(m, pipe, bg, rigid_k):
    from gaussian_renderer import render_batch
    from fdgs import regularize as fr
    from fdgs.loss import l1_ssim_loss

    def fn(views, gt):
        pkg = render_batch(views, m, pipe, bg)
        loss = sum(l1_ssim_loss(pkg["render"][k], gt[k]) for k in range(gt.shape[0])) / gt.shape[0]
        if rigid_k:
            loss = loss + fr.rigidity_loss(m, k=rigid_k, neighbours=fr.neighbours(m.get_xyz, rigid_k))
        loss.backward()
        return loss, pkg
    return fn


def _set_lr(m, it):
    m.optimizer.param_groups[0]["lr"] = 1.6e-4 * 0.01 ** (min(it, 30000) / 30000)   # expon_lr_func's log-linear decay


def _tail(m, pkg, B):
    """The eager statistics and optimiser step after a graphed step (INTEGRATION's loop without optimizer=)."""
    import fdgs.densify as D
    from fdgs.dist import ViewBatchStats
    st = ViewBatchStats(m._xyz.shape[0], DEV)
    for b in range(B):
        st.add_view(pkg["viewspace_points"].grad[b], pkg["radii"][b])
    D.add_densification_stats(m, t_grad=m._t.grad, batch_stats=st, batch_size=B)
    m.optimizer.step()
    m.optimizer.zero_grad(set_to_none=True)


def bench(name, w, iters, rounds, warmup):
    from fdgs.graph import GraphedStep
    pipe, bg = _Pipe(w.get("sky")), torch.zeros(3, device=DEV)
    out = {"workload": name, "P": w["P"], "W": w["W"], "H": w["H"], "B": w["B"], "rigid_k": w.get("rigid", 0)}
    arms = {}
    for arm in ("eager" if w.get("sky") else "eager_tail", "graph"):
        pc, cams, gts = _setup(w)
        m = _model(pc)
        gt = torch.stack(gts)
        fn = _fn(m, pipe, bg, w.get("rigid", 0))
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        if arm == "graph":
            step = GraphedStep(fn, m, optimizer=m.optimizer)
            call = lambda it, s=step, m=m: (_set_lr(m, it), s(cams, gt, densify_stats=True))   # noqa: E731
        elif arm == "eager":
            step = None
            call = lambda it, fn=fn, m=m: (_set_lr(m, it), _tail(m, fn(cams, gt)[1], w["B"]))  # noqa: E731
        else:
            step = GraphedStep(fn, m)
            call = lambda it, s=step, m=m: (_set_lr(m, it), _tail(m, s(cams, gt)[1], w["B"]))  # noqa: E731
        call(0)
        torch.cuda.synchronize()
        out[arm + "_peak_extra_MB"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
        for it in range(1, warmup + 1):
            call(it)
        arms[arm] = dict(m=m, step=step, call=call, cams=cams, gt=gt, it=warmup + 1, times=[])

    for _ in range(rounds):
        for arm, a in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(iters):
                a["call"](a["it"])
                a["it"] += 1
            torch.cuda.synchronize()
            a["times"].append(1e3 * (time.perf_counter() - t0) / iters)
    for arm, a in arms.items():
        q = sorted(a["times"])
        out[arm + "_ms"] = round(statistics.median(q), 3)
        out[arm + "_ms_iqr"] = [round(q[len(q) // 4], 3), round(q[(3 * len(q)) // 4], 3)]
        if a["step"] is None:
            out[arm + "_enqueue_ms"] = None
            continue
        out[arm + "_enqueue_ms"] = round(_enqueue(arm, a), 3)
        out[arm + "_captures"], out[arm + "_overflows"] = a["step"].info["captures"], a["step"].info["overflows"]
    out["speedup"] = round(out[("eager" if w.get("sky") else "eager_tail") + "_ms"] / out["graph_ms"], 3)
    out.update(_adam_kernels(arms["graph"]["m"]))
    return out


def _enqueue(arm, a, reps=15):
    """Median host time to enqueue one iteration without the status read: load the inputs, stage the optimiser's
    scalars (graph arm), replay; for the eager-tail arm, after the replay has finished, the statistics and optimiser
    launches."""
    step, m = a["step"], a["m"]
    leaves = [p for g in m.optimizer.param_groups for p in g["params"]]
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        h0 = time.perf_counter()
        step.views.load(a["cams"])
        step.gt.copy_(a["gt"])
        if arm == "graph":
            m.optimizer.stage(step._stepped)
        step._graph.replay()
        t = time.perf_counter() - h0
        torch.cuda.synchronize()
        if arm == "graph":
            m.optimizer.commit(step._stepped)
        else:
            for p, g in zip(leaves, step._grads):
                p.grad = g
            h0 = time.perf_counter()
            _tail(m, step._out[1], step.views.B)
            t += time.perf_counter() - h0
        times.append(1e3 * t)
    return statistics.median(times)


def _adam_kernels(m, reps=20):
    """Kernel time per step of the eager and the staged fused Adam over the nine groups (torch.profiler, own run)."""
    from torch.profiler import ProfilerActivity, profile
    leaves = [p for g in m.optimizer.param_groups for p in g["params"]]
    for p in leaves:
        p.grad = torch.zeros_like(p)
    opt = m.optimizer
    opt.init_state()
    for p in leaves:                     # one step count for all: the eager step is then one launch, like the staged one
        opt.state[p]["step"].fill_(100.0)
    res = {}
    for arm, run in (("eager", lambda: opt.step()),
                     ("staged", lambda: (opt.stage(leaves), opt.step_staged(leaves), opt.commit(leaves)))):
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                run()
            torch.cuda.synchronize()
        us = 0.0
        for e in prof.key_averages():
            if "adam" in e.key and "kernel" in e.key:
                us += getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
        res["adam_kernel_%s_ms" % arm] = round(us / reps / 1e3, 4)
    for p in leaves:
        p.grad = None
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20, help="iterations per timed block")
    ap.add_argument("--rounds", type=int, default=15, help="alternating blocks per arm")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_graph_iteration: no CUDA device")
    names = [n for n in WORKLOADS if not args.only or n in args.only.split(",")]
    info = gpu_info()
    for n in names:
        r = bench(n, WORKLOADS[n], args.iters, args.rounds, args.warmup)
        r.update(info)
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
