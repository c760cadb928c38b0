"""Fused multi-tensor Adam over per-Gaussian parameter groups (csrc/optim.cu over the C-ABI).

Stands in for `torch.optim.Adam(l, lr=0.0, eps=1e-15)` as the reference sets it up
(scene/gaussian_model.py:331-357) and steps it (train.py:248-249): same `param_groups` list-of-dicts interface
(`params`, `lr`, optional `name`), same update, but every group is updated by ONE kernel launch per step, which
can also clear the gradients it consumed.  `step(rows=idx)` restricts the update to the listed Gaussians (the step's
rendered set, e.g. ViewBatchStats.max_radii > 0): the rasterizer's gradient rows of all others are exactly zero.
That sparse mode deliberately differs from torch's dense semantics (unrendered Gaussians keep their parameters and
moments instead of coasting on decaying momentum) and is opt-in.  CUDA only.

Step counts are per parameter, as in torch: `state[p]["step"]` (a CPU float32 scalar tensor, torch's format, so
`fdgs.densify` and state copied from `torch.optim.Adam` carry it) counts the steps in which `p` had a gradient, and
that count sets `p`'s bias correction.  A parameter whose `.grad` is None is skipped without advancing its count; a
parameter group added later starts at step 1.  Tensors of equal step share a launch.
"""
from typing import Iterable, Optional

import torch

import fdgs


class FusedAdam:
    def __init__(self, params: Iterable, lr: float = 0.0, betas=(0.9, 0.999), eps: float = 1e-15):
        params = list(params)
        if params and not isinstance(params[0], dict):
            params = [{"params": params}]
        self.param_groups = []
        for g in params:
            g = dict(g)
            g.setdefault("lr", lr)
            g["params"] = list(g["params"])
            self.param_groups.append(g)
        self.betas, self.eps = betas, eps
        self.state = {}

    def add_param_group(self, group):
        """torch.optim.Optimizer.add_param_group: a new group (default lr: the constructor's), its steps counted from 1."""
        group = dict(group)
        ps = group["params"]
        group["params"] = [ps] if isinstance(ps, torch.Tensor) else list(ps)
        group.setdefault("lr", self.param_groups[0]["lr"] if self.param_groups else 0.0)
        self.param_groups.append(group)

    def _state(self, p):
        st = self.state.get(p)
        if st is None:
            st = {"step": torch.tensor(0.0, dtype=torch.float32),
                  "exp_avg": torch.zeros_like(p, memory_format=torch.contiguous_format),
                  "exp_avg_sq": torch.zeros_like(p, memory_format=torch.contiguous_format)}
            self.state[p] = st
        return st

    @torch.no_grad()
    def step(self, rows: Optional[torch.Tensor] = None, zero_grad: bool = False):
        """One Adam step over every parameter that has a gradient.  rows: int64 CUDA index tensor or None (dense)."""
        by_step = {}   # step count -> (params, grads, exp_avg, exp_avg_sq, lrs): one bias correction per launch
        for g in self.param_groups:
            for p in g["params"]:
                if p.grad is None:
                    continue
                st = self._state(p)
                st["step"] += 1
                if not p.grad.is_contiguous():
                    p.grad = p.grad.contiguous()
                t = by_step.setdefault(int(st["step"]), ([], [], [], [], []))
                for lst, x in zip(t, (p.data, p.grad, st["exp_avg"], st["exp_avg_sq"], float(g["lr"]))):
                    lst.append(x)
        C = fdgs.ext()
        sparse = rows is not None
        rows_t = rows if sparse else torch.empty(0, dtype=torch.int64)
        for step, (ps, gs, ms, vs, lrs) in by_step.items():
            for i in range(0, len(ps), 16):
                C.adam_step(ps[i:i + 16], gs[i:i + 16], ms[i:i + 16], vs[i:i + 16], lrs[i:i + 16], rows_t, sparse,
                            step, self.betas[0], self.betas[1], self.eps, zero_grad)

    def zero_grad(self, set_to_none: bool = True):
        for g in self.param_groups:
            for p in g["params"]:
                if set_to_none:
                    p.grad = None
                elif p.grad is not None:
                    p.grad.zero_()
