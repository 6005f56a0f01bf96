"""Differentiable restatements behind the camera-gradient tests: the camera set-up chain (k_camera_setup:
extrinsics, intrinsics -> viewmatrix, projmatrix, campos, tanfov) and one view of the rasterizer with its depth
channel, both plain torch, so that autograd in float64 is the yardstick of ps_raster_camera_grads and
ps_camera_setup_backward."""
from __future__ import annotations

import torch

from oracle import raster_torch as rt


def camera_chain(ext: torch.Tensor, K: torch.Tensor, near, far, scale_invariant: bool = True):
    """One view: ext [4,4] camera-to-world, K [3,3] normalised -> (vm [16], pm [16], campos [3], tanfov [2],
    scene_scale), the column-major arrays k_camera_setup writes.  near / far are plain numbers (not differentiated)."""
    near, far = float(near), float(far)
    scale = 1.0 / near if scale_invariant else 1.0
    sv = torch.tensor([1.0, 1.0, 1.0, scale], dtype=ext.dtype, device=ext.device)
    e = torch.cat([ext[:3] * sv, ext[3:]], 0)             # the translation column scaled
    nr, fr = near * scale, far * scale
    kinv = torch.linalg.inv(K)

    def unit(x, y):
        v = kinv @ torch.tensor([x, y, 1.0], dtype=K.dtype, device=K.device)
        return v / v.norm()

    tx = (0.5 * (unit(0.0, 0.5) * unit(1.0, 0.5)).sum().acos()).tan()
    ty = (0.5 * (unit(0.5, 0.0) * unit(0.5, 1.0)).sum().acos()).tan()
    z = torch.zeros((), dtype=ext.dtype, device=ext.device)
    one = torch.ones((), dtype=ext.dtype, device=ext.device)
    proj = torch.stack([torch.stack([2 * nr / (2 * tx * nr), z, z, z]),
                        torch.stack([z, 2 * nr / (2 * ty * nr), z, z]),
                        torch.stack([z, z, fr / (fr - nr) * one, -(fr * nr) / (fr - nr) * one]),
                        torch.stack([z, z, one, z])])
    w2c = torch.linalg.inv(e)
    view_t = w2c.T
    return (view_t.reshape(16), (view_t @ proj.T).reshape(16), e[:3, 3], torch.stack([tx, ty]), scale)


def depth_value(mode: str, z, near, far):
    if mode == "disparity":
        return 1 / z
    if mode == "relative_disparity":
        eps = 1e-10
        dn, df = 1 / (near + eps), 1 / (far + eps)
        return 1 - (1 / (z + eps) - df) / (dn - df + eps)
    if mode == "log":
        return z.minimum(torch.as_tensor(near, dtype=z.dtype)).maximum(torch.as_tensor(far, dtype=z.dtype)).log()
    return z


def render_view(means, cov6, opac, sh, colors, vm, pm, campos, tanfov, bg, W, H, degree, scale=1.0,
                depth_mode=None, near=None, far=None):
    """One view as the CUDA rasterizer computes it: means and covariances in world units with the view's
    scene_scale applied inside (means * s, cov * s^2), optional depth channel z = view z / s composited with the
    colour's alphas over 0.  -> (color [3,H,W], depth [H,W] | None)."""
    m, c = means * scale, cov6 * (scale * scale)
    color, _ = rt.rasterize(m, c, opac, sh, colors, vm, pm, campos, tanfov[0], tanfov[1], bg, W, H, degree)
    if depth_mode is None:
        return color, None
    z = (vm[2] * m[:, 0] + vm[6] * m[:, 1] + vm[10] * m[:, 2] + vm[14]) / scale
    d = depth_value(depth_mode, z, near, far)
    dcol, _ = rt.rasterize(m, c, opac, None, d[:, None].expand(-1, 3), vm, pm, campos, tanfov[0], tanfov[1],
                           torch.zeros(3, dtype=m.dtype), W, H, degree)
    return color, dcol[0]
