"""The environment-map sky as the reference's PyTorch code computes it (Camera.get_rays + the sphere / grid_sample
composition of its render()), restated for the tests and tools/bench_sky.py, plus a float64 CPU restatement of the same
mathematics and a camera stand-in exposing what both need.  TEST / BENCH INFRASTRUCTURE."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from fdgs import synth

R_SKY = 60.0


class SkyCamera:
    """A synth camera with the pinhole intrinsics and get_rays() of the reference's Camera (scene/cameras.py)."""

    def __init__(self, W, H, R=None, T=None, timestamp=0.5, focal_scale=0.54, device="cpu"):
        cam = synth.make_camera(W, H, timestamp=timestamp, focal_scale=focal_scale, R=R, T=T).to(device)
        self.image_width, self.image_height = W, H
        self.FoVx, self.FoVy = cam.FoVx, cam.FoVy
        self.world_view_transform, self.full_proj_transform = cam.world_view_transform, cam.full_proj_transform
        self.camera_center, self.timestamp = cam.camera_center, cam.timestamp
        self.fl_x = self.fl_y = focal_scale * W
        self.cx, self.cy = W / 2.0, H / 2.0
        self.device = device

    def get_rays(self):
        ys, xs = torch.meshgrid(torch.arange(self.image_height, dtype=torch.float32),
                                torch.arange(self.image_width, dtype=torch.float32), indexing="ij")
        i, j = xs + 0.5, ys + 0.5
        pts_view = torch.stack([(i - self.cx) / self.fl_x, (j - self.cy) / self.fl_y, torch.ones_like(i),
                                torch.ones_like(i)], -1).to(self.device)
        c2w = torch.linalg.inv(self.world_view_transform.transpose(0, 1))
        pts_world = pts_view @ c2w.T
        directions = pts_world[..., :3] - self.camera_center[None, None, :]
        return self.camera_center[None, None], directions / torch.norm(directions, dim=-1, keepdim=True)


def torch_sky(env_map, cam, R=R_SKY):
    """The reference's sky in PyTorch (fp32 on env_map's device); asserts like the reference when a ray misses."""
    rays_o, rays_d = cam.get_rays()
    od = (rays_o * rays_d).sum(-1)
    dd = (rays_d ** 2).sum(-1)
    delta = od ** 2 - dd * ((rays_o ** 2).sum(-1) - R ** 2)
    assert (delta > 0).all()
    t_inter = -od + torch.sqrt(delta) / dd
    hit = rays_o + rays_d * t_inter.unsqueeze(-1)
    tu = torch.atan2(hit[..., 1:2], hit[..., 0:1]) / (2 * torch.pi) + 0.5
    tv = torch.acos(hit[..., 2:3] / R) / torch.pi
    texcoord = torch.cat([tu, tv], dim=-1) * 2 - 1
    return F.grid_sample(env_map[None], texcoord[None])[0]


def torch_composition(rendered, alpha, sky):
    """rendered + (1 - alpha) * sky: the reference's composition of the sky behind the Gaussians."""
    return rendered + (1 - alpha) * sky


def f64_grid(cam, R=R_SKY):
    """float64 CPU texture coordinates [1,H,W,2] of every pixel (the same mathematics, no fp32 rounding)."""
    W, H = cam.image_width, cam.image_height
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    pv = np.stack([(xs + 0.5 - cam.cx) / cam.fl_x, (ys + 0.5 - cam.cy) / cam.fl_y, np.ones_like(xs), np.ones_like(xs)], -1)
    c2w = np.linalg.inv(cam.world_view_transform.detach().cpu().double().numpy().T)
    o = np.linalg.inv(cam.world_view_transform.detach().cpu().double().numpy())[3, :3]
    d = (pv @ c2w.T)[..., :3] - o
    d = d / np.linalg.norm(d, axis=-1, keepdims=True)
    od = (d * o).sum(-1)
    dd = (d * d).sum(-1)
    delta = od ** 2 - dd * ((o * o).sum() - R * R)
    t = -od + np.sqrt(delta) / dd
    hit = o + d * t[..., None]
    tu = np.arctan2(hit[..., 1], hit[..., 0]) / (2 * math.pi) + 0.5
    tv = np.arccos(np.clip(hit[..., 2] / R, -1.0, 1.0)) / math.pi
    return torch.from_numpy(np.stack([tu, tv], -1) * 2 - 1)[None]


def f64_sky(env_map, cam, R=R_SKY):
    return F.grid_sample(env_map.detach().cpu().double()[None], f64_grid(cam, R))[0]


def f64_sky_grad(env_map, cam, g, R=R_SKY):
    """float64 dL/d env_map of the sky for the image gradient g [3,H,W] (grid_sample's backward)."""
    env = env_map.detach().cpu().double().requires_grad_(True)
    (F.grid_sample(env[None], f64_grid(cam, R))[0] * g.detach().cpu().double()).sum().backward()
    return env.grad
