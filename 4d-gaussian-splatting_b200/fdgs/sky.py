"""Environment-map sky behind the Gaussians (csrc/sky.cu; include/fdgs.h: fdgs_sky_forward / fdgs_sky_backward).

Scenes configured with an environment map (`env_map_res`) see, through every pixel the Gaussians leave transparent,
a sphere of radius 60 about the origin textured with a learned [3,Hm,Wm] map in longitude / colatitude layout.  The
reference samples it in PyTorch (Camera.get_rays + F.grid_sample) and composes `rendered + (1 - alpha) * sky`; here
the sampling is one CUDA kernel each way and the composition happens inside the rasterizer (its `bg_image` input).

    sky = sky_background(pc.env_map, camera)                  # [3,H,W], differentiable w.r.t. env_map
    color, radii, depth, alpha, flow, covs = rasterizer(..., bg_image=sky)

sample_sky_batch(env_map, views) samples the B cameras of an fdgs.graph.StaticViews(..., sky=True) in one launch each
way from the views' device tables: it neither synchronises nor reads the miss flag on the host, so a CUDA graph can
capture it.
"""
import torch

RADIUS = 60.0


def _camera_inputs(camera):
    # camera-to-world as the reference's Camera.get_rays builds it: one 4x4 inverse of the world-to-view matrix
    c2w = torch.linalg.inv(camera.world_view_transform.transpose(0, 1)).contiguous()
    campos = camera.camera_center.reshape(3).to(torch.float32).contiguous()
    return c2w, campos, float(camera.fl_x), float(camera.fl_y), float(camera.cx), float(camera.cy)


class _SkyBackground(torch.autograd.Function):
    @staticmethod
    def forward(ctx, env_map, c2w, campos, fl_x, fl_y, cx, cy, radius, H, W):
        import fdgs
        env = env_map.detach().contiguous()
        sky, miss = fdgs.ext().sky_forward(env, c2w, campos, fl_x, fl_y, cx, cy, radius, H, W)
        ctx.save_for_backward(env, c2w, campos)
        ctx.consts = (fl_x, fl_y, cx, cy, radius)
        ctx.mark_non_differentiable(miss)
        return sky, miss

    @staticmethod
    def backward(ctx, grad_sky, _grad_miss):
        import fdgs
        env, c2w, campos = ctx.saved_tensors
        denv = fdgs.ext().sky_backward(env, c2w, campos, *ctx.consts, grad_sky.contiguous())
        return (denv,) + (None,) * 9


MISS_MESSAGE = "a camera ray does not intersect the sky sphere (camera outside the radius-%g sphere)" % RADIUS


class _SkyBatch(torch.autograd.Function):
    @staticmethod
    def forward(ctx, env_map, c2w, campos, intrinsics, radius, H, W):
        import fdgs
        env = env_map.detach().contiguous()
        sky, miss = fdgs.ext().sky_forward_batch(env, c2w, campos, intrinsics, radius, H, W)
        ctx.save_for_backward(env, c2w, campos, intrinsics)
        ctx.radius = radius
        ctx.mark_non_differentiable(miss)
        return sky, miss

    @staticmethod
    def backward(ctx, grad_sky, _grad_miss):
        import fdgs
        env, c2w, campos, intrinsics = ctx.saved_tensors
        denv = fdgs.ext().sky_backward_batch(env, c2w, campos, intrinsics, ctx.radius, grad_sky.contiguous())
        return (denv,) + (None,) * 6


class MissFlag:
    """Whether any ray of a sky_background() call missed the sphere (a camera outside it looking away).  The device flag
    travels to pinned host memory right behind the sky kernel; check() waits only for that copy, so called after the
    rasterizer's forward -- which synchronises on the stream anyway to learn its instance count -- it costs nothing."""

    def __init__(self, flag):
        self.host = torch.empty(1, dtype=torch.int32, pin_memory=True)
        self.host.copy_(flag, non_blocking=True)
        self.ready = torch.cuda.Event()
        self.ready.record()

    def check(self):
        self.ready.synchronize()
        # the reference asserts the same condition on its ray / sphere discriminant
        assert int(self.host[0]) == 0, MISS_MESSAGE


def sample_sky(env_map, camera, radius=RADIUS):
    """(sky [3,H,W], MissFlag) -- the sky of `camera`; call MissFlag.check() once the flag is wanted."""
    if env_map.dim() != 3 or env_map.shape[0] != 3 or env_map.dtype != torch.float32 or not env_map.is_cuda:
        raise ValueError("env_map must be a float32 CUDA tensor [3,Hm,Wm], got %s %s on %s"
                         % (tuple(env_map.shape), env_map.dtype, env_map.device))
    c2w, campos, fl_x, fl_y, cx, cy = _camera_inputs(camera)
    H, W = int(camera.image_height), int(camera.image_width)
    sky, miss = _SkyBackground.apply(env_map, c2w.to(env_map.device), campos.to(env_map.device), fl_x, fl_y, cx, cy,
                                     float(radius), H, W)
    return sky, MissFlag(miss)


def sky_background(env_map, camera, radius=RADIUS):
    """[3,H,W] colour of the environment map `env_map` [3,Hm,Wm] seen through every pixel of `camera` on the sky
    sphere of radius `radius`; gradients flow to env_map.  `camera` provides world_view_transform, camera_center,
    fl_x, fl_y, cx, cy, image_height and image_width, like the reference's Camera.  Raises AssertionError when a ray
    misses the sphere (the check waits for the sky kernel; render() defers it to avoid that wait)."""
    sky, miss = sample_sky(env_map, camera, radius)
    miss.check()
    return sky


def sample_sky_batch(env_map, views, radius=RADIUS):
    """(sky [B,3,H,W], miss int32 [1] on the device) -- the sky of every camera of `views`, an fdgs.graph.StaticViews
    built with sky=True; gradients flow to env_map, summed over the views.  View b's sky equals sample_sky(env_map,
    camera b) bit for bit.  miss is 1 if a ray of any view missed the sphere; nothing here reads it (the reference
    asserts on it: raise AssertionError(MISS_MESSAGE) once it is read)."""
    if env_map.dim() != 3 or env_map.shape[0] != 3 or env_map.dtype != torch.float32 or not env_map.is_cuda:
        raise ValueError("env_map must be a float32 CUDA tensor [3,Hm,Wm], got %s %s on %s"
                         % (tuple(env_map.shape), env_map.dtype, env_map.device))
    if getattr(views, "c2w", None) is None:
        raise ValueError("sample_sky_batch needs StaticViews(..., sky=True) (camera-to-world and intrinsics tables)")
    return _SkyBatch.apply(env_map, views.c2w, views.campos, views.intrinsics, float(radius), views.H, views.W)
