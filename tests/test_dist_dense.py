"""CPU, world_size 2 over gloo: parameters that are not per-Gaussian rows (an environment map) are summed over the ranks
by ViewParallelStep.finish(dense_params=...) / render_view_batch(dense_keys=...) -- the same .grad the sequential loop
leaves, on every rank."""
import os

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from fdgs import dist as fdist
from test_dist_gloo import _fake_render, _free_port

P, ENV = 257, (3, 8, 16)


def _render_with_env(params, view):
    pkg = _fake_render(params, view)
    w = torch.rand(*ENV, generator=torch.Generator().manual_seed(500 + view))
    pkg["render"] = pkg["render"].sum() + (params["env_map"] * w).sum() * (view + 1)
    return pkg


def _params():
    torch.manual_seed(0)
    return {"xyz": torch.randn(P, 3, requires_grad=True), "opacity": torch.rand(P, 1, requires_grad=True),
            "env_map": torch.rand(*ENV, requires_grad=True)}


def _worker(rank, world, port, num_views, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        params = _params()
        views = fdist.shard_views(num_views, rank, world)
        fdist.render_view_batch(lambda v: _render_with_env(params, v), views, params, lambda pkg, v: pkg["render"],
                                global_batch=num_views, dense_keys=("env_map",))
        out[rank] = (params["env_map"].grad.clone(), params["xyz"].grad.clone())
    finally:
        dist.destroy_process_group()


def test_dense_parameters_are_summed_over_ranks():
    num_views, world = 5, 2
    ref = _params()
    for v in range(num_views):
        (_render_with_env(ref, v)["render"] / num_views).backward()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), num_views, out), nprocs=world, join=True)
    for r in range(world):
        genv, gxyz = out[r]
        assert torch.allclose(genv, ref["env_map"].grad, rtol=1e-5, atol=1e-7)
        assert torch.allclose(gxyz, ref["xyz"].grad, rtol=1e-5, atol=1e-6)
    assert torch.equal(out[0][0], out[1][0])
