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
parameter group added later starts at step 1.  Tensors of equal step and row count share a launch (a tensor of another
row count, such as an environment map [3,Hm,Wm] beside the per-Gaussian rows, gets its own).

For a step captured in a CUDA graph (fdgs.graph.GraphedStep(..., optimizer=)), the learning rates and step counts
cannot be kernel arguments: the graph would freeze them.  `init_state()` allocates every leaf's state outside the
capture, `step_staged(params, status)` launches (and so can be captured) a dense step that reads each tensor's
lr / bias_correction1, sqrt(bias_correction2) and enable flag from a persistent device table, `stage(params, hold)`
fills that table before each replay for "count + 1" from the groups' current `lr`, and `commit(params, hold)` advances
the counts once the replay is known to have stepped (its rasterizer status shows no overflow).  The scalars are
computed by the same host function as the eager step's (include/fdgs.h: fdgs_adam_scalars), so both give the same bits.
"""
from typing import Iterable, Optional

import torch

import fdgs


def _launches(params):
    """[i, j) runs of consecutive tensors that one launch can take: at most 16 (FDGS_MAX_PACK), all of one row count."""
    out, i = [], 0
    while i < len(params):
        j = i + 1
        while j < len(params) and j - i < 16 and params[j].shape[0] == params[i].shape[0]:
            j += 1
        out.append((i, j))
        i = j
    return out


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
        self._table = None        # device float32 [n, 3] of the staged step: lr / bc1, sqrt(bc2), enable
        self._table_host = None   # its pinned staging buffer
        self._staged = None       # event after the last copy out of the staging buffer

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
        by_step = {}   # (step count, rows) -> (params, grads, exp_avg, exp_avg_sq, lrs): one bias correction per launch
        for g in self.param_groups:
            for p in g["params"]:
                if p.grad is None:
                    continue
                st = self._state(p)
                st["step"] += 1
                if not p.grad.is_contiguous():
                    p.grad = p.grad.contiguous()
                t = by_step.setdefault((int(st["step"]), p.shape[0]), ([], [], [], [], []))
                for lst, x in zip(t, (p.data, p.grad, st["exp_avg"], st["exp_avg_sq"], float(g["lr"]))):
                    lst.append(x)
        C = fdgs.ext()
        sparse = rows is not None
        rows_t = rows if sparse else torch.empty(0, dtype=torch.int64)
        for (step, _), (ps, gs, ms, vs, lrs) in by_step.items():
            for i in range(0, len(ps), 16):
                C.adam_step(ps[i:i + 16], gs[i:i + 16], ms[i:i + 16], vs[i:i + 16], lrs[i:i + 16], rows_t, sparse,
                            step, self.betas[0], self.betas[1], self.eps, zero_grad)

    # ---- the staged step of a captured training step ------------------------------------------------------------------
    def _leaves(self):
        return [p for g in self.param_groups for p in g["params"]]

    def held(self, hold):
        """The ids of the leaves `hold` keeps from stepping: True = all of them, else a collection of group names
        (a single name may be given as a string)."""
        if hold is True:
            return {id(p) for p in self._leaves()}
        if not hold:
            return set()
        names = {hold} if isinstance(hold, str) else set(hold)
        known = {g.get("name") for g in self.param_groups}
        unknown = sorted(str(n) for n in names - known)
        if unknown:
            raise ValueError("hold names no parameter group of the optimiser: %s" % ", ".join(unknown))
        return {id(p) for g in self.param_groups if g.get("name") in names for p in g["params"]}

    def init_state(self):
        """Every leaf's step count and moments, and the device scalar table, allocated now: state first created while a
        CUDA graph captures would live in the graph's private memory pool and be freed with it."""
        leaves = self._leaves()
        for p in leaves:
            self._state(p)
        n = max(1, len(leaves))
        if self._table is None or self._table.shape[0] < n or (leaves and self._table.device != leaves[0].device):
            dev = leaves[0].device if leaves else "cuda"
            if self._staged is not None:
                self._staged.synchronize()
            self._table = torch.zeros(n, 3, dtype=torch.float32, device=dev)
            self._table_host = torch.zeros(n, 3, dtype=torch.float32, pin_memory=True)
            self._staged = None

    @torch.no_grad()
    def step_staged(self, params, status: Optional[torch.Tensor] = None):
        """Launch a dense step of `params` (leaves with a gradient) with the scalars `stage` last wrote for them, row i of
        the table for params[i]; status: the rasterizer's int32 [4] (nothing is written on overflow) or None.
        Synchronises nothing, so a CUDA graph can capture it; call init_state() before the capture."""
        params = list(params)
        if self._table is None or self._table.shape[0] < len(params) or any(p not in self.state for p in params):
            raise RuntimeError("FusedAdam.step_staged: call init_state() first (outside any graph capture)")
        C = fdgs.ext()
        st = status if status is not None else torch.empty(0, dtype=torch.int32)
        for i, j in _launches(params):
            ps = params[i:j]
            sts = [self.state[p] for p in ps]
            C.adam_step_staged([p.data for p in ps], [p.grad.contiguous() for p in ps], [s["exp_avg"] for s in sts],
                               [s["exp_avg_sq"] for s in sts], self._table[i:i + len(ps)].view(-1), st,
                               self.betas[0], self.betas[1], self.eps)

    def stage(self, params, hold=()):
        """Write the scalar table of the next staged step of `params` on the current stream: each tensor's group lr and
        its step count + 1, or a hold entry for the tensors of `hold` (see held()).  The pinned buffer is rewritten
        only after the previous copy out of it has completed."""
        params = list(params)
        held = self.held(hold)
        lr_of = {id(p): float(g["lr"]) for g in self.param_groups for p in g["params"]}
        lrs = [lr_of[id(p)] for p in params]
        enable = [0 if id(p) in held else 1 for p in params]
        steps = [int(self.state[p]["step"]) + e for p, e in zip(params, enable)]
        if self._staged is not None:
            self._staged.synchronize()
        C = fdgs.ext()
        for i in range(0, len(params), 16):
            C.adam_scalars(lrs[i:i + 16], steps[i:i + 16], enable[i:i + 16], self.betas[0], self.betas[1],
                           self._table_host[i:i + len(lrs[i:i + 16])].view(-1))
        n = len(params)
        self._table[:n].copy_(self._table_host[:n], non_blocking=True)
        self._staged = torch.cuda.Event()
        self._staged.record()

    def commit(self, params, hold=()):
        """Advance the step count of every tensor of `params` that the staged step updated (not held)."""
        held = self.held(hold)
        for p in params:
            if id(p) not in held:
                self.state[p]["step"] += 1

    def zero_grad(self, set_to_none: bool = True):
        for g in self.param_groups:
            for p in g["params"]:
                if set_to_none:
                    p.grad = None
                elif p.grad is not None:
                    p.grad.zero_()
