"""Data-parallel rendering over views (frames) -- the only way this path shards.

The reference renders the `batch_size` views of one optimisation step sequentially on one GPU and
lets autograd sum the per-Gaussian gradients (reference: train.py:104-166, loss scaled by
1/batch_size at :162), then merges the densification statistics of the views (train.py:168-183).
Here the views of a step are spread over the ranks (one process per GPU, replicated Gaussians):
every rank renders its own views, then `ViewParallelStep.finish()` leaves in every parameter's
`.grad` exactly what the sequential loop leaves there.  What travels:

  radii            MAX all-reduce (int32 [P]); it is the reference's `radii = max over views` statistic
                   (train.py:171) AND the union of the Gaussians any view rendered -- rows outside it are zero in
                   every rasterizer gradient on every rank and never move;
  geometry bucket  the 17 parameter-gradient floats of a Gaussian (xyz 3, t 1, scale 3, scale_t 1, rotation 4,
                   rotation_r 4, opacity 1) + the two SUM statistics (per-view screen-gradient norm, train.py:164,173;
                   visibility count, :169) as two more columns: the union's rows packed into ONE flat buffer
                   (csrc/exchange.cu), ONE SUM all-reduce, scattered back;
  SH colour        the 144 SH-gradient floats of a Gaussian (89 % of a gradient row) do NOT travel.  One view's
  factors          dL_dsh row is the outer product (SH basis weights of the view direction and time) x (colour
                   gradient), so the backward emits only the 3-float colour factor (fdgs_backward_args.sh_factors);
                   the factors of all views are all-gathered for the union's rows (12 B per Gaussian and view
                   instead of 576 B in an all-reduce) and every rank rebuilds and sums the rows itself from the
                   replicated parameters (csrc/preprocess_bwd.cu: sh_outer_sum_kernel), in global view order with
                   explicit round-to-nearest multiply-then-add -- bit-identical to accumulating the views'
                   dL_dsh tensors one after the other, and identical on every rank.  The dense 1.15 GB dL_dsh
                   tensor of a view is never materialised.
  dense params     parameters that are not per-Gaussian rows (an environment map): their .grad are concatenated into
                   one flat buffer and summed with ONE SUM all-reduce, launched beside the geometry all-reduce.

A single-view render never communicates.  `.grad` of the parameters must be None or zero when a step starts
(the sparse exchange and the reference's semantics both assume it); gradients that are NOT produced by the
rasterizer (e.g. a rigidity loss over all Gaussians, train.py:132-152) are detected on the device (a non-zero row
outside the union) and switch the geometry bucket to the dense all-reduce for that step.
"""
from typing import Callable, Dict, Iterable, List, Optional, Sequence

import torch
import torch.distributed as dist


def shard_views(num_views: int, rank: int, world: int) -> List[int]:
    """Indices of the views rank `rank` renders: contiguous blocks, sizes differing by at most one."""
    base, rem = divmod(num_views, world)
    start = rank * base + min(rank, rem)
    return list(range(start, start + base + (1 if rank < rem else 0)))


_SIDE_STREAMS: Dict[str, "torch.cuda.Stream"] = {}


def _side_stream(device):
    key = str(device)
    if key not in _SIDE_STREAMS:
        _SIDE_STREAMS[key] = torch.cuda.Stream(device=device)
    return _SIDE_STREAMS[key]


def _world(group=None) -> int:
    return dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1


def _rows_zero_outside(tensors: Sequence[torch.Tensor], radii: torch.Tensor) -> torch.Tensor:
    """1-element int32 tensor: non-zero if any row outside `radii > 0` holds a non-zero element."""
    if tensors and tensors[0].is_cuda:
        import fdgs
        return fdgs.ext().check_rows_zero(list(tensors), radii)
    out = radii <= 0
    bad = torch.zeros(1, dtype=torch.int32, device=radii.device)
    for t in tensors:
        bad |= (t.reshape(t.shape[0], -1)[out] != 0).any().to(torch.int32)
    return bad


def _pack(tensors: Sequence[torch.Tensor], idx: torch.Tensor):
    """rows `idx` of every tensor -> one flat buffer, one block per tensor (16-byte aligned block starts)."""
    if tensors[0].is_cuda:
        import fdgs
        return fdgs.ext().pack_rows(list(tensors), idx)
    K = idx.numel()
    blocks = []
    for t in tensors:
        w = t.numel() // t.shape[0]
        b = t.reshape(t.shape[0], w).index_select(0, idx).reshape(-1)
        pad = (-b.numel()) % 4
        blocks.append(torch.cat([b, b.new_zeros(pad)]) if pad else b)
    return torch.cat(blocks) if blocks else torch.empty(0)


def _unpack(flat: torch.Tensor, tensors: Sequence[torch.Tensor], idx: torch.Tensor):
    if tensors[0].is_cuda:
        import fdgs
        fdgs.ext().unpack_rows(flat, list(tensors), idx)
        return
    K, off = idx.numel(), 0
    for t in tensors:
        w = t.numel() // t.shape[0]
        t.view(t.shape[0], w).index_copy_(0, idx, flat[off:off + K * w].view(K, w))
        off += (K * w + 3) // 4 * 4


def allreduce_gradients(grads: Sequence[Optional[torch.Tensor]], group=None, average_over: Optional[int] = None,
                        union_radii: Optional[torch.Tensor] = None, dense_above: float = 0.6,
                        union_visible: Optional[torch.Tensor] = None):
    """In-place SUM all-reduce of per-Gaussian gradient tensors (None entries are skipped).

    `union_radii` (int32 [P], IDENTICAL on every rank: the MAX-reduced radii of the step; `union_visible`, a bool
    mask, is accepted as well) enables the sparse exchange: only the rows of Gaussians some view rendered are packed
    into one flat buffer, all-reduced with ONE collective and scattered back.  It is only valid when every row
    outside the union is zero on every rank; that is CHECKED on the device (one pass over the tensors, the flag is
    read with the union size, then MAX-reduced so that all ranks take the same path) and the call falls back to the
    dense all-reduce when it does not hold, or when the union covers more than `dense_above` of the Gaussians."""
    live = [g for g in grads if g is not None]
    if _world(group) == 1 or not live:
        if average_over:
            for g in live:
                g.div_(average_over)
        return
    if union_radii is None and union_visible is not None:
        union_radii = union_visible.reshape(-1).to(torch.int32)
    P = live[0].shape[0]
    idx = None
    if union_radii is not None and all(g.shape[0] == P and g.is_contiguous() for g in live):
        union_radii = union_radii.reshape(-1).to(torch.int32).contiguous()
        bad = _rows_zero_outside(live, union_radii)
        dist.all_reduce(bad, op=dist.ReduceOp.MAX, group=group)       # every rank must take the same path
        idx = torch.nonzero(union_radii > 0).squeeze(1)               # host sync: K sizes the collective
        if int(bad.item()) != 0 or idx.numel() > dense_above * P:
            idx = None
    if idx is None:
        works = [dist.all_reduce(g, op=dist.ReduceOp.SUM, group=group, async_op=True) for g in live]
        for w in works:
            w.wait()
    elif idx.numel() > 0:
        flat = _pack(live, idx)
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
        _unpack(flat, live, idx)
    if average_over:
        for g in live:
            g.div_(average_over)


class ViewBatchStats:
    """Accumulates the reference's per-step densification statistics over the local views and
    reduces them across ranks (reference: train.py:168-183, scene/gaussian_model.py:579-589)."""

    def __init__(self, P: int, device):
        self.grad_norm_sum = torch.zeros(P, 1, device=device)      # sum_views ||viewspace grad[:, :2]||
        self.visibility_count = torch.zeros(P, 1, device=device)   # sum_views (radii > 0)
        self.max_radii = torch.zeros(P, dtype=torch.int32, device=device)
        self.radii_reduced = False

    def add_view(self, viewspace_grad: torch.Tensor, radii: torch.Tensor):
        if (viewspace_grad.is_cuda and viewspace_grad.dtype == torch.float32 and viewspace_grad.is_contiguous()
                and radii.dtype == torch.int32 and radii.is_contiguous()):
            import fdgs
            fdgs.ext().view_stats(viewspace_grad, radii, self.grad_norm_sum, self.visibility_count, self.max_radii)
            return
        self.grad_norm_sum += torch.norm(viewspace_grad[:, :2], dim=-1, keepdim=True)
        self.visibility_count += (radii > 0).to(self.visibility_count.dtype).view(-1, 1)
        self.max_radii = torch.max(self.max_radii, radii.to(torch.int32))

    def reduce_radii(self, group=None):
        if _world(group) > 1 and not self.radii_reduced:
            dist.all_reduce(self.max_radii, op=dist.ReduceOp.MAX, group=group)
        self.radii_reduced = True
        return self

    def reduce(self, group=None):
        """Stand-alone reduction of all three statistics (ViewParallelStep.finish() folds the two SUM statistics
        into the geometry bucket instead)."""
        self.reduce_radii(group)
        if _world(group) > 1:
            both = torch.cat([self.grad_norm_sum, self.visibility_count], 1)
            dist.all_reduce(both, op=dist.ReduceOp.SUM, group=group)
            self.grad_norm_sum, self.visibility_count = both[:, :1].contiguous(), both[:, 1:].contiguous()
        return self


class _ViewRecord:
    """What the rasterizer's backward leaves behind for one view in SH-factor mode."""
    __slots__ = ("factors", "timestamp", "campos", "settings", "inputs")

    def __init__(self, factors, settings, inputs):
        self.factors = factors              # [P,3] clamp-masked colour gradient of the view
        self.timestamp = float(settings.timestamp)
        self.campos = settings.campos
        self.settings = settings
        self.inputs = inputs                # dict of the (replicated) rasterizer inputs of the view


class ViewParallelStep:
    """The gradient exchange of ONE optimisation step whose views are spread over the ranks.

        step = ViewParallelStep(P, device)
        with step:                                   # rasterizer backward switches to SH-factor mode
            for view in my_views:
                pkg = render(view, gaussians, pipe, bg)
                (loss_fn(pkg, view) / global_batch).backward()
                step.add_view_stats(pkg["viewspace_points"].grad, pkg["radii"])
        step.finish(geometry_params, sh_params)      # .grad == what the sequential loop leaves, on every rank

    `sh_params`: the leaf tensor(s) whose concatenation along dim 1 is the `shs` input of the rasterizer -- one
    [P,M,3] tensor, or the reference model's (features_dc [P,1,3], features_rest [P,M-1,3])
    (scene/gaussian_model.py:210-214); their `.grad` is written directly (no torch.cat backward, no dense per-view
    dL_dsh).  With `sh_factors=False` (or for rasterizer calls the factor mode does not cover: precomputed
    covariances / colours) dL_dsh is produced densely by autograd and exchanged as rows of the union like any
    other gradient -- list those tensors in `geometry_params` then.
    """

    _active: Optional["ViewParallelStep"] = None

    def __init__(self, P: int, device, group=None, sh_factors: bool = True, dense_above: float = 0.6,
                 outer_sum_fn: Optional[Callable] = None, expected_views: Optional[int] = None):
        """expected_views: how many views THIS rank renders in the step.  When given (and on CUDA), the union of the
        rendered Gaussians is built as soon as the last local FORWARD has run -- MAX all-reduce of the radii, prefix
        sum and its total to pinned host memory on a side stream -- so that this collective, the scan and the host's
        wait for the row count K all hide behind the backward pass instead of following it."""
        self.P, self.device, self.group = P, device, group
        self.sh_factors = sh_factors
        self.dense_above = dense_above
        self.stats = ViewBatchStats(P, device)
        self.views: List[_ViewRecord] = []
        self._outer_sum_fn = outer_sum_fn
        self.info: Dict[str, object] = {}
        self.profile = False            # True: CUDA events around the phases of finish() -> info["phase_ms"] (one sync)
        self.profile_serial = False     # with profile: wait for every collective where it is launched (no overlap), so
                                        # that the phases are the collectives' own durations (bus-bandwidth figures)
        self._marks = []
        self.expected_views = expected_views
        self._fwd_radii = None
        self._fwd_count = 0
        self._early = None              # (radii_max, prefix_sum, event, pinned K) once the early union was launched

    def _mark(self, name):
        if self.profile and torch.cuda.is_available() and str(self.device).startswith("cuda"):
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self._marks.append((name, ev))

    # ---- installation of the autograd hook (gaussian_renderer/diff_gaussian_rasterization.py) ----
    def __enter__(self):
        assert ViewParallelStep._active is None, "view-parallel steps do not nest"
        ViewParallelStep._active = self
        return self

    def __exit__(self, *exc):
        ViewParallelStep._active = None
        return False

    @classmethod
    def current(cls) -> Optional["ViewParallelStep"]:
        return cls._active

    def wants_factors(self, sh, cov3D_precomp) -> bool:
        """Asked by the rasterizer's backward: emit colour factors instead of the dense dL_dsh?"""
        return self.sh_factors and sh.numel() > 0 and cov3D_precomp.numel() == 0

    def record_view(self, factors, settings, inputs):
        self.views.append(_ViewRecord(factors, settings, inputs))

    def on_forward(self, radii: torch.Tensor):
        """Called by the rasterizer's forward (autograd hook): accumulate MAX radii; after the last expected view start
        the union build on a side stream (see __init__)."""
        if self.expected_views is None or not radii.is_cuda:
            return
        r = radii.to(torch.int32)
        self._fwd_radii = r.clone() if self._fwd_radii is None else torch.max(self._fwd_radii, r)
        self._fwd_count += 1
        if self._fwd_count == self.expected_views:
            cur = torch.cuda.current_stream()
            side = _side_stream(radii.device)
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                rmax = self._fwd_radii
                rmax.record_stream(side)
                if _world(self.group) > 1:
                    dist.all_reduce(rmax, op=dist.ReduceOp.MAX, group=self.group)
                cs = torch.cumsum(rmax > 0, 0, dtype=torch.int32)
                k_host = torch.empty(1, dtype=torch.int32).pin_memory()
                k_host.copy_(cs[-1:] if self.P > 0 else cs.new_zeros(1), non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(side)
            self._early = (rmax, cs, ev, k_host)

    def add_view_stats(self, viewspace_grad: torch.Tensor, radii: torch.Tensor):
        self.stats.add_view(viewspace_grad, radii)

    # ---- the exchange -----------------------------------------------------------------------------
    def finish(self, geometry_params: Sequence[torch.Tensor], sh_params: Sequence[torch.Tensor] = (),
               views_per_rank: Optional[int] = None, dense_params: Sequence[torch.Tensor] = ()) -> ViewBatchStats:
        """`dense_params`: parameters with no per-Gaussian rows (e.g. the environment map); their gradients are summed
        over the ranks whole, outside the union / row-guard logic of the geometry bucket."""
        group, world, P = self.group, _world(self.group), self.P
        st = self.stats
        self._marks = []
        self._mark("start")
        grads = []
        for p in geometry_params:
            if p.grad is None:
                p.grad = torch.zeros_like(p)
            grads.append(p.grad)
        have_factors = len(self.views) > 0
        cs = None
        if self._early is not None:
            # the union was built behind the backward pass: wait for ITS event only (not for the whole stream)
            rmax, cs, ev, k_host = self._early
            ev.synchronize()
            torch.cuda.current_stream().wait_event(ev)
            st.max_radii, st.radii_reduced = rmax, True
            K = int(k_host[0])
        else:
            st.reduce_radii(group)                                      # union of rendered Gaussians + MAX statistic
        self._mark("radii_max_allreduce")
        if world == 1 and not have_factors:
            return st

        union = st.max_radii
        # guard of the sparse exchange (rows outside the union must be zero): checked on the device, MAX-reduced, read
        # at the END of finish() -- the optimistic sparse path is repaired there in the (rare) case it was wrong
        bad = _rows_zero_outside(grads, union) if (grads and world > 1) else torch.zeros(1, dtype=torch.int32, device=union.device)
        bad_work = dist.all_reduce(bad, op=dist.ReduceOp.MAX, group=group, async_op=True) if world > 1 else None
        bad_host = bad_ready = None
        if bad_work is not None and bad.is_cuda:
            # the reduced flag travels to pinned host memory on the side stream as soon as ITS collective is done, so
            # that reading it at the end of finish() waits for that early event only -- not for the whole step's GPU
            # work (a full synchronisation there would leave the GPU idle while the host launches the next step)
            side = _side_stream(bad.device)
            with torch.cuda.stream(side):
                bad_work.wait()
                bad.record_stream(side)
                bad_host = torch.empty(1, dtype=torch.int32).pin_memory()
                bad_host.copy_(bad, non_blocking=True)
                bad_ready = torch.cuda.Event()
                bad_ready.record(side)
        mask = union > 0
        if union.is_cuda:
            import fdgs
            if cs is None:
                cs = torch.cumsum(mask, 0, dtype=torch.int32)
                K = int(cs[-1].item()) if P > 0 else 0                  # host sync: K sizes the buffers
            slot_of, idx = fdgs.ext().union_maps(union.contiguous(), cs, K)   # one pass (csrc/exchange.cu)
        else:
            idx = torch.nonzero(mask).squeeze(1)
            K = int(idx.numel())
            slot_of = torch.where(mask, torch.cumsum(mask.to(torch.int32), 0, dtype=torch.int32) - 1,
                                  torch.full_like(union, -1)).to(torch.int32).contiguous()
        sparse_ok = K <= self.dense_above * P
        self._mark("union_index_build")
        self.info = {"K": K, "union_fraction": K / max(P, 1), "geometry_path": "rows" if sparse_ok else "dense",
                     "views_local": len(self.views), "early_union": self._early is not None}

        # -- both payloads are packed first, both collectives are launched asynchronously (NCCL runs them in issue
        #    order on its own stream: the small factor all-gather, then the geometry all-reduce), and the SH
        #    reconstruction -- the longest phase, needing only the factors -- runs on the compute stream WHILE the
        #    geometry bucket is being reduced; the bucket is scattered back afterwards
        want_sh = have_factors or (self.sh_factors and len(sh_params) > 0 and world > 1)
        local = table = None
        if want_sh:
            assert len(sh_params) in (1, 2), "sh_params: the [P,M,3] SH tensor or (features_dc, features_rest)"
            v_local = len(self.views)
            if views_per_rank is None:
                vmax = torch.tensor([v_local], dtype=torch.int32, device=union.device)
                if world > 1:
                    dist.all_reduce(vmax, op=dist.ReduceOp.MAX, group=group)
                views_per_rank = int(vmax.item())
            assert v_local <= views_per_rank
            meta_off = (3 * K + 3) // 4 * 4
            stride = meta_off + 8
            local = torch.zeros(views_per_rank, stride, dtype=torch.float32, device=union.device)
            if 2 < v_local <= 16 and union.is_cuda:
                # several local views: ONE row gather for all of them (the pack kernel of the geometry bucket: block v
                # = view v's K rows, padded to a multiple of 4 floats = meta_off) and three small copies for the
                # metadata, instead of four launches per view
                if K > 0:
                    flat_f = _pack([rec.factors for rec in self.views], idx)
                    local[:v_local, :meta_off] = flat_f.view(v_local, meta_off)
                ts_host = torch.tensor([rec.timestamp for rec in self.views], dtype=torch.float32).pin_memory()
                local[:v_local, meta_off] = ts_host.to(union.device, non_blocking=True)
                local[:v_local, meta_off + 1:meta_off + 4] = torch.stack([rec.campos.reshape(3) for rec in self.views]).to(local.dtype)
            else:
                for v, rec in enumerate(self.views):
                    if K > 0:
                        torch.index_select(rec.factors, 0, idx, out=local[v, :3 * K].view(K, 3))
                    local[v, meta_off] = rec.timestamp
                    local[v, meta_off + 1:meta_off + 4] = rec.campos.reshape(3).to(local.dtype)
            self._mark("factor_pack")
        bucket = grads + [st.grad_norm_sum, st.visibility_count]
        flat, geo_works = None, []
        if world > 1 and sparse_ok and K > 0:
            flat = _pack(bucket, idx)
            self._mark("geometry_pack")
            self.info["geometry_allreduce_bytes"] = int(flat.numel() * 4)
        gather_work = None
        if want_sh and world > 1:
            table = torch.empty(world * views_per_rank, stride, dtype=torch.float32, device=union.device)
            gather_work = dist.all_gather_into_tensor(table, local, group=group, async_op=True)
            if self.profile_serial:
                gather_work.wait()
                self._mark("factor_allgather")
                gather_work = None
        elif want_sh:
            table = local
        dense_flat = dense_work = None
        if world > 1 and len(dense_params) > 0:
            for p in dense_params:
                if p.grad is None:
                    p.grad = torch.zeros_like(p)
            dense_flat = torch.cat([p.grad.reshape(-1) for p in dense_params])
            dense_work = dist.all_reduce(dense_flat, op=dist.ReduceOp.SUM, group=group, async_op=True)
        if world > 1:
            if flat is not None:
                geo_works = [dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group, async_op=True)]
            elif not sparse_ok:
                geo_works = [dist.all_reduce(g, op=dist.ReduceOp.SUM, group=group, async_op=True) for g in bucket]
            if self.profile_serial and geo_works:
                for w in geo_works:
                    w.wait()
                self._mark("geometry_allreduce")
                geo_works = []
        if want_sh:
            if gather_work is not None:
                gather_work.wait()
                self._mark("factor_allgather")
            outs = []
            for p in sh_params:
                if p.grad is None:
                    p.grad = torch.empty_like(p)
                outs.append(p.grad)
            self._outer_sum(table, stride, meta_off, table.shape[0], K, slot_of, outs, idx)
            self._mark("sh_outer_sum")
            self.info.update(views_total=int(table.shape[0]), factor_bytes_per_rank=int(local.numel() * 4))
        for w in geo_works:
            w.wait()
        if geo_works:
            self._mark("geometry_allreduce_exposed")   # what is left of it after the SH reconstruction
        if flat is not None:
            _unpack(flat, bucket, idx)
            self._mark("geometry_unpack")
        if dense_work is not None:
            dense_work.wait()
            off = 0
            for p in dense_params:
                n = p.grad.numel()
                p.grad.copy_(dense_flat[off:off + n].view_as(p.grad))
                off += n
            self._mark("dense_allreduce")
        self.views = []
        self._early, self._fwd_radii, self._fwd_count = None, None, 0
        if world > 1:
            if bad_ready is not None:
                bad_ready.synchronize()
                is_bad = int(bad_host[0]) != 0
            else:
                bad_work.wait()
                is_bad = int(bad.item()) != 0
            if is_bad and sparse_ok:
                # some rank holds gradients outside the union (a loss over ALL Gaussians): the union's rows are summed
                # already, sum the remaining rows densely
                self.info["geometry_path"] = "rows + dense repair"
                outside = (~mask)
                for g in grads + [st.grad_norm_sum, st.visibility_count]:
                    m = outside.view(-1, *([1] * (g.dim() - 1)))
                    tmp = g * m
                    dist.all_reduce(tmp, op=dist.ReduceOp.SUM, group=group)
                    g.mul_(~m).add_(tmp)
            self._mark("guard_check")
        if self._marks:
            torch.cuda.synchronize()
            self.info["phase_ms"] = {b[0]: a[1].elapsed_time(b[1]) for a, b in zip(self._marks[:-1], self._marks[1:])}
        return st

    def _outer_sum(self, table, stride, meta_off, V, K, slot_of, outs, idx):
        # the replicated inputs and the per-step constants come from any recorded view; a rank without views (more
        # ranks than views) has none and must be handed them by the caller through `outer_sum_fn`
        if self._outer_sum_fn is not None:
            return self._outer_sum_fn(table, stride, meta_off, V, K, slot_of, outs, self.views)
        assert self.views, "finish(): this rank rendered no view -- pass outer_sum_fn, or give every rank a view"
        rec = self.views[0]
        s, i = rec.settings, rec.inputs
        if i.get("raw"):
            # recorded by the raw-parameter entry: the reconstruction kernel takes the activated values (three small
            # elementwise kernels once per STEP, not per view)
            act = lambda t, f: f(t) if (t is not None and t.numel()) else t
            i = dict(i, scales=act(i["scales"], torch.exp), scales_t=act(i["scales_t"], torch.exp),
                     rotations=act(i["rotations"], torch.nn.functional.normalize),
                     rotations_r=act(i["rotations_r"], torch.nn.functional.normalize))
        import fdgs
        fdgs.ext().sh_outer_sum(table, stride, meta_off, V, K, slot_of, idx, i["means3D"], i["ts"], i["scales"], i["scales_t"],
                                i["rotations"], i["rotations_r"], float(s.scale_modifier), float(s.time_duration),
                                bool(s.rot_4d), int(s.gaussian_dim), bool(s.force_sh_3d), int(s.sh_degree),
                                int(s.sh_degree_t), outs, False)


def render_view_batch(render_fn, views: Iterable, params: Dict[str, torch.Tensor], loss_fn, global_batch: int,
                      group=None, sh_keys: Sequence[str] = (), dense_keys: Sequence[str] = ()) -> Dict[str, object]:
    """One optimisation step's worth of rendering, data-parallel over views.

    render_fn(view) -> the dict render() returns; loss_fn(pkg, view) -> scalar loss of that view.
    `views` are the views THIS rank owns (see shard_views).  After the call every tensor in `params`
    holds, in .grad, the batch gradient (sum over all ranks' views of d(loss/global_batch)), exactly
    what the reference's sequential loop leaves there, and the returned stats are the merged
    densification statistics.  `sh_keys` names the entries of `params` that form the rasterizer's SH input
    (exchanged as colour factors, see ViewParallelStep); `dense_keys` the entries that are not per-Gaussian (e.g.
    "env_map"), summed whole; everything else goes through the geometry bucket."""
    first = next(p for k, p in params.items() if k not in dense_keys)
    step = ViewParallelStep(first.shape[0], first.device, group=group, sh_factors=len(sh_keys) > 0)
    total = torch.zeros((), device=first.device)
    with step:
        for view in views:
            pkg = render_fn(view)
            loss = loss_fn(pkg, view) / global_batch
            loss.backward()
            total += loss.detach()
            step.add_view_stats(pkg["viewspace_points"].grad, pkg["radii"])
    geometry = [p for k, p in params.items() if k not in sh_keys and k not in dense_keys]
    stats = step.finish(geometry, [params[k] for k in sh_keys], dense_params=[params[k] for k in dense_keys])
    if _world(group) > 1:
        dist.all_reduce(total, op=dist.ReduceOp.SUM, group=group)
    return {"loss": total, "stats": stats, "exchange": step.info}
