"""The training step as one CUDA graph.

At the image sizes the dnerf scenes train at (400x400, 1 to 24 views per step) a step of render_batch + loss + backward
waits on the host -- kernel launches, Python and autograd -- more than on the GPU.  A CUDA graph replays the whole step
with one launch, but a captured step must not synchronise and must not bake host values into the graph:

  StaticViews   device tensors that hold a step's cameras; render_batch(views, ...) reads the cameras from them and
                calls the rasterizer entry sized by an instance capacity (include/fdgs.h:
                fdgs_forward_batch_capacity), which never synchronises.  Its "status" output reports the true instance
                count R and whether it overflowed the capacity (the views then render as if no Gaussian were listed).
  GraphedStep   captures a user step fn(views, gt) -> (loss, pkg) once and replays it with new cameras and ground truth;
                it reads the status once per step, after all of the step's work is queued, and on overflow re-captures
                with a larger capacity and replays the same inputs.  Optionally the capture also runs the densification
                statistics and a fused Adam step (fdgs.optim.FusedAdam) whose learning rates and step counts are staged
                in device memory before each replay; both are predicated on the status, so an overflowed replay changes
                nothing and the replay after the re-capture applies them once.

Scenes with an environment map capture too: the views then also hold each camera's camera-to-world matrix and
intrinsics (StaticViews(..., sky=True)), render_batch samples every view's sky in one batched call, and the step's
miss flag (a ray that misses the sky sphere, which the reference asserts on) travels with the status in the one host
read; a miss also keeps the captured statistics and optimiser step from writing.

Densification itself (and the opacity reset) runs eagerly after the call.
"""
import math
from typing import Callable, Iterable, List, Optional

import torch


class StaticViews:
    """B cameras of one image size in device tensors: viewmatrix / projmatrix [B,4,4], campos [B,3], timestamp /
    tanfovx / tanfovy [B] (float32), and `capacity`, the instances the rasterizer's binning buffer holds summed over the
    views.  render_batch(views, ...) reads whatever load() last copied in.

    sky=True also holds what the environment-map sky sampler needs (fdgs.sky.sample_sky_batch): c2w [B,4,4], each
    camera's camera-to-world matrix, and intrinsics [B,4] = (fl_x, fl_y, cx, cy); the cameras must then carry the
    pinhole intrinsics of the reference's Camera."""

    def __init__(self, B: int, H: int, W: int, device, sky: bool = False):
        if B < 1 or H < 1 or W < 1:
            raise ValueError("StaticViews needs B, H, W >= 1, got %d, %d, %d" % (B, H, W))
        self.B, self.H, self.W = int(B), int(H), int(W)
        self.sky = bool(sky)
        self.device = torch.device(device)
        f = dict(dtype=torch.float32, device=self.device)
        self.viewmatrix = torch.zeros(self.B, 4, 4, **f)
        self.projmatrix = torch.zeros(self.B, 4, 4, **f)
        self.campos = torch.zeros(self.B, 3, **f)
        # the per-camera scalars (timestamp, tan(FoVx / 2), tan(FoVy / 2), then with sky the intrinsics) in one buffer,
        # so that one copy from one pinned host buffer fills them
        n = 3 * self.B + (4 * self.B if self.sky else 0)
        self._scalars = torch.zeros(n, **f)
        self.timestamp, self.tanfovx, self.tanfovy = self._scalars[:3 * self.B].view(3, self.B).unbind(0)
        self.c2w = torch.zeros(self.B, 4, 4, **f) if self.sky else None
        self.intrinsics = self._scalars[3 * self.B:].view(self.B, 4) if self.sky else None
        self._host = torch.zeros(n, dtype=torch.float32, pin_memory=True)
        self._copied: Optional[torch.cuda.Event] = None
        self.capacity = 0

    def load(self, cams) -> None:
        """Copy the reference Cameras `cams` (B of them, this image size) into the tensors, in place, on the current
        stream.  The scalars go through one pinned host buffer; it is rewritten only after the previous load's copy out
        of it has completed.  With sky, each c2w is torch.linalg.inv_ex of the camera's world_view_transform.T on the
        camera's device: fdgs.sky's single-view sampler inverts the same matrix with torch.linalg.inv, the same
        arithmetic, but inv_ex leaves its singularity check on the device."""
        cams = list(cams)
        if len(cams) != self.B:
            raise ValueError("StaticViews holds %d views, got %d cameras" % (self.B, len(cams)))
        for c in cams:
            if (int(c.image_height), int(c.image_width)) != (self.H, self.W):
                raise ValueError("StaticViews holds %dx%d views, got a %dx%d camera"
                                 % (self.W, self.H, int(c.image_width), int(c.image_height)))
        if self.sky:
            for c in cams:
                if not float(getattr(c, "fl_x", 0.0)) > 0.0:
                    raise ValueError("the environment-map sky needs cameras with pinhole intrinsics (fl_x > 0, fl_y, "
                                     "cx, cy), got fl_x = %r" % (getattr(c, "fl_x", None),))
        rows = [[float(c.timestamp) for c in cams], [math.tan(c.FoVx * 0.5) for c in cams],
                [math.tan(c.FoVy * 0.5) for c in cams]]
        if self.sky:
            rows.append([float(getattr(c, k)) for c in cams for k in ("fl_x", "fl_y", "cx", "cy")])
        if self._copied is not None:
            self._copied.synchronize()
        # the host values render_batch and the sky sampler compute for a camera list, rounded to float32 the same way
        self._host.copy_(torch.tensor([x for r in rows for x in r], dtype=torch.float32))
        self._scalars.copy_(self._host, non_blocking=True)
        self._copied = torch.cuda.Event()
        self._copied.record()
        for dst, name in ((self.viewmatrix, "world_view_transform"), (self.projmatrix, "full_proj_transform"),
                          (self.campos, "camera_center")):
            dst.copy_(torch.stack([getattr(c, name).to(self.device) for c in cams]))
        if self.sky:
            self.c2w.copy_(torch.stack([torch.linalg.inv_ex(c.world_view_transform.transpose(0, 1))[0].to(self.device)
                                        for c in cams]))


def _leaves(params) -> List[torch.Tensor]:
    src = params() if callable(params) else params
    opt = getattr(src, "optimizer", src)
    if hasattr(opt, "param_groups"):
        return [p for g in opt.param_groups for p in g["params"]]
    return list(src)


_STATS = ("xyz_gradient_accum", "denom", "max_radii2D", "t_gradient_accum")


class GraphedStep:
    """One training step, captured once and replayed: `step(cams, gt)` runs `fn(views, gt)` -- which calls
    render_batch(views, ...), computes its loss and calls backward() -- and returns fn's (loss, pkg), static tensors that
    every replay overwrites.  After the call each leaf's .grad holds the step's gradient.

    params: the Gaussian model (an object with an `optimizer` whose param groups hold the leaves, and
    `active_sh_degree` / `active_sh_degree_t`, like the reference's GaussianModel), an optimiser, a list of leaves, or a
    callable returning one of those.  The leaves are read on every call: a new leaf (densification, pruning), a new SH
    degree, or a new B, H or W re-captures.  margin: the capacity is margin x the instance count it is sized from.

    The first call warms up eagerly on a side stream, first at capacity 0 (a background-only render whose status reports
    the true R), then at ceil(margin R); each capture starts with every leaf's .grad set to None, so replays assign
    the gradients rather than accumulate them.  The step's one host synchronisation reads the status after the replay;
    on overflow the step re-captures at ceil(margin R) and replays the same inputs (the statistics and the optimiser
    step below are skipped by an overflowed replay, so nothing has moved).  `info` counts captures and overflows and
    holds the capacity.

    `step(cams, gt, densify_stats=True)` also captures the densification statistics after fn, from the replay's own
    pkg: one view, `add_densification_stats(model, viewspace_grad, radii)`; B >= 2 views, a ViewBatchStats over the views
    and the batch form; `params` must then be the Gaussian model (xyz_gradient_accum, denom, max_radii2D and, for 4D
    Gaussians, t_gradient_accum and _t).  optimizer: a fdgs.optim.FusedAdam over exactly the step's leaves; the capture
    ends with its dense step over every leaf that has a gradient, and the leaves' step counts advance after each call.
    `hold` keeps tensors from stepping in this call without re-capturing: True (none steps: densification iterations,
    whose new leaves the reference's Adam skips, and the last iteration) or a collection of group names (e.g.
    {"opacity"} on an opacity-reset iteration).  Do not call optimizer.step() as well.  The warm-up runs fn only.

    A model with a non-empty `env_map` gets views with sky tables (StaticViews(..., sky=True)); a learned map
    (requires_grad) must be a parameter group named "env_map" of the model's FusedAdam `optimizer`, so that its gradient
    is one of the step's leaves and the captured step moves it (hold={"env_map"} keeps it, e.g. past the reference's
    env_optimize_until).  When a ray misses the sky sphere the call raises AssertionError, as the reference's render
    does, and nothing -- parameters, moments, step counts, statistics -- has moved."""

    def __init__(self, fn: Callable, params, margin: float = 1.25, optimizer=None):
        from fdgs.optim import FusedAdam
        if not margin >= 1.0:
            raise ValueError("margin must be >= 1, got %r" % (margin,))
        if optimizer is not None and not isinstance(optimizer, FusedAdam):
            raise ValueError("GraphedStep captures the step of a fdgs.optim.FusedAdam only, got %s" % type(optimizer).__name__)
        self.fn, self.params, self.margin, self.optimizer = fn, params, float(margin), optimizer
        self.views: Optional[StaticViews] = None
        self.gt: Optional[torch.Tensor] = None
        self.info = {"captures": 0, "overflows": 0, "capacity": None}
        self._graph = None
        self._key = None
        self._out = None
        self._read = None         # the int32 [4] status, or [5] with the sky's miss flag, that the host reads
        self._grads: List[Optional[torch.Tensor]] = []
        self._stepped: List[torch.Tensor] = []    # the leaves the captured optimiser step updates

    def _sized(self, R: int) -> int:
        return int(math.ceil(self.margin * R))

    def _drop(self):
        """Free the graph and its static outputs before another capture."""
        self._graph, self._out, self._read, self._grads, self._stepped = None, None, None, [], []

    def _warm_up(self, leaves):
        side = torch.cuda.Stream(device=self.views.device)
        side.wait_stream(torch.cuda.current_stream(self.views.device))
        missed = False
        with torch.cuda.stream(side):
            self.views.capacity = 0
            _, pkg = self.fn(self.views, self.gt)
            R = int(pkg["status"][0])
            missed = "sky_miss" in pkg and int(pkg["sky_miss"][0]) != 0
            if not missed:
                self.views.capacity = self._sized(R)
                self.fn(self.views, self.gt)
        torch.cuda.current_stream(self.views.device).wait_stream(side)
        for p in leaves:
            p.grad = None
        if missed:
            from fdgs.sky import MISS_MESSAGE
            raise AssertionError(MISS_MESSAGE)
        self.info["capacity"] = self.views.capacity

    def _model(self):
        return self.params() if callable(self.params) else self.params

    def _stats(self, pkg, status):
        """The densification statistics of the step in pkg, skipped when status reports overflow or wrap (captured after
        fn)."""
        from fdgs import densify as D
        from fdgs.dist import ViewBatchStats
        model = self._model()
        vs = pkg["viewspace_points"].grad
        if vs is None:
            raise ValueError("densify_stats needs pkg['viewspace_points'].grad: fn must call backward()")
        t_grad = model._t.grad if int(getattr(model, "gaussian_dim", 3)) == 4 else None
        B = self.views.B
        if B == 1:
            D.add_densification_stats(model, vs[0], pkg["radii"][0], t_grad=t_grad, status=status)
        else:
            stats = ViewBatchStats(vs.shape[1], vs.device)
            for k in range(B):
                stats.add_view(vs[k], pkg["radii"][k])
            D.add_densification_stats(model, t_grad=t_grad, batch_stats=stats, batch_size=B, status=status)

    def _capture(self, leaves, densify_stats=False):
        self._drop()
        for p in leaves:
            p.grad = None
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = self.fn(self.views, self.gt)
            status = guard = read = out[1]["status"]
            miss = out[1].get("sky_miss")
            if miss is not None:
                # a miss reads as a wrap to the statistics and Adam kernels, which then write nothing; the host reads
                # the true status and the miss together, int32 [5]
                guard = torch.cat([status[:3], status[3:] | miss])
                read = torch.cat([status, miss])
            if densify_stats:
                self._stats(out[1], guard)
            if self.optimizer is not None:
                self._stepped = [p for p in leaves if p.grad is not None]
                self.optimizer.step_staged(self._stepped, guard)
        self._graph, self._out, self._read = graph, out, read
        self._grads = [p.grad for p in leaves]
        self.info["captures"] += 1
        self.info["capacity"] = self.views.capacity

    def _replay(self, leaves, hold=()):
        if self.optimizer is not None:
            self.optimizer.stage(self._stepped, hold)
        self._graph.replay()
        for p, g in zip(leaves, self._grads):
            p.grad = g
        status = self._read.tolist()
        if len(status) == 5 and status[4]:
            from fdgs.sky import MISS_MESSAGE
            raise AssertionError(MISS_MESSAGE)
        status = status[:4]
        if status[3]:
            raise RuntimeError("GraphedStep: more than 2^31 - 1 tile instances in one step")
        return status

    def _check(self, leaves, densify_stats, hold):
        """The new arguments' rejections, before any GPU work."""
        opt = self.optimizer
        if opt is None:
            if hold:
                raise ValueError("hold needs GraphedStep(..., optimizer=)")
        else:
            mine = opt._leaves()
            if len(mine) != len(leaves) or {id(p) for p in mine} != {id(p) for p in leaves}:
                raise ValueError("optimizer must be a FusedAdam over exactly the step's leaves")
            opt.held(hold)
        if densify_stats:
            model = self._model()
            dim = int(getattr(model, "gaussian_dim", 3))
            need = _STATS[:3] + ((_STATS[3], "_t") if dim == 4 else ())
            missing = [n for n in need if getattr(model, n, None) is None]
            if missing:
                raise ValueError("densify_stats needs the Gaussian model as params (missing: %s)" % ", ".join(missing))
        env = self._env_map()
        if env is not None and env.requires_grad:
            from fdgs.optim import FusedAdam
            model_opt = getattr(self._model(), "optimizer", None)
            groups = getattr(model_opt, "param_groups", []) if isinstance(model_opt, FusedAdam) else []
            if not any(g.get("name") == "env_map" and any(p is env for p in g["params"]) for g in groups):
                raise ValueError("a learned env_map must be a parameter group named 'env_map' of the model's FusedAdam "
                                 "optimizer: the captured step would otherwise write a gradient it does not own")

    def _env_map(self):
        """The model's environment map if it has a non-empty one, else None."""
        env = getattr(self._model(), "env_map", None)
        return env if isinstance(env, torch.Tensor) and env.numel() > 0 else None

    def __call__(self, cams, gt: torch.Tensor, densify_stats: bool = False, hold=()):
        cams = list(cams)
        if not cams:
            raise ValueError("GraphedStep needs at least one camera")
        leaves = _leaves(self.params)
        self._check(leaves, densify_stats, hold)
        B, H, W = len(cams), int(cams[0].image_height), int(cams[0].image_width)
        sky = self._env_map() is not None
        if (self.views is None or (self.views.B, self.views.H, self.views.W, self.views.sky) != (B, H, W, sky)
                or self.gt.shape != gt.shape):
            capacity = self.views.capacity if self.views is not None else None
            self._drop()
            self.views = StaticViews(B, H, W, gt.device, sky=sky)
            self.gt = torch.empty_like(gt)
            if capacity is not None:
                self.views.capacity = capacity
        self.views.load(cams)
        self.gt.copy_(gt)
        model = self._model()
        key = (B, H, W, tuple(p.shape[0] for p in leaves[:1]), tuple(p.data_ptr() for p in leaves),
               getattr(model, "active_sh_degree", None), getattr(model, "active_sh_degree_t", None), bool(densify_stats),
               sky)
        if densify_stats:
            key += tuple(getattr(model, n).data_ptr() if getattr(model, n, None) is not None else None for n in _STATS)
        if self.optimizer is not None:
            self.optimizer.init_state()
            st = self.optimizer.state
            key += (self.optimizer._table.data_ptr(),) + tuple(
                (st[p]["exp_avg"].data_ptr(), st[p]["exp_avg_sq"].data_ptr()) for p in leaves)
        if self._graph is None or key != self._key:
            if self.info["capacity"] is None:
                self._warm_up(leaves)
            self._capture(leaves, densify_stats)
            self._key = key
        status = self._replay(leaves, hold)
        if status[2]:
            self.info["overflows"] += 1
            self.views.capacity = self._sized(status[0])
            self._capture(leaves, densify_stats)
            status = self._replay(leaves, hold)
        if self.optimizer is not None and not status[2]:
            self.optimizer.commit(self._stepped, hold)
        return self._out
