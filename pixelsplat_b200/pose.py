"""Test-time pose alignment: refine the target views' extrinsics against their images with the Gaussians frozen.

Pose-free evaluation of novel views renders each target view from Gaussians an encoder predicted, optimises only the
view's camera pose against the ground-truth image for a few hundred steps, and then measures PSNR / SSIM.  Here every
(scene, view) gets one 6-vector twist xi = (omega, t), applied in the camera frame, E' = E @ T(xi), with
T(xi) = [[exp(omega^), t], [0, 1]].  The loss is the rasterizer's fused squared-error epilogue (no image is
materialised), and Adam updates the [s, v, 6] twists: Adam is element-wise and each view's loss depends on its own
twist only, so the s x v alignments are independent problems solved together, one rasterizer call per step.  With the
Gaussians not requiring grad, the rasterizer's backward is the camera-only one (no Gaussian gradient is formed).
"""
from __future__ import annotations

from typing import NamedTuple, Optional

import torch
from torch import Tensor

from .decoder.cuda_splatting import render_views_mse

_SMALL_ANGLE2 = 1e-8    # |omega|^2 below which exp(omega^) uses its Taylor series


def twist_to_transform(xi: Tensor) -> Tensor:
    """[..., 6] twists (omega, t) -> [..., 4, 4] rigid transforms [[exp(omega^), t], [0, 1]].  The rotation is
    Rodrigues' formula, with its Taylor series near omega = 0 so that the derivative there is exact and finite; plain
    torch operations, differentiable, no host synchronisation."""
    w, t = xi[..., :3], xi[..., 3:]
    th2 = (w * w).sum(-1, keepdim=True)[..., None]                       # [..., 1, 1]
    small = th2 < _SMALL_ANGLE2
    th2_safe = torch.where(small, torch.ones_like(th2), th2)
    th = th2_safe.sqrt()
    a = torch.where(small, 1.0 - th2 / 6.0, th.sin() / th)               # sin(th) / th
    b = torch.where(small, 0.5 - th2 / 24.0, (1.0 - th.cos()) / th2_safe)  # (1 - cos(th)) / th^2
    z = torch.zeros_like(w[..., 0])
    W = torch.stack([torch.stack([z, -w[..., 2], w[..., 1]], -1),
                     torch.stack([w[..., 2], z, -w[..., 0]], -1),
                     torch.stack([-w[..., 1], w[..., 0], z], -1)], -2)
    eye = torch.eye(3, dtype=xi.dtype, device=xi.device).expand(W.shape)
    R = eye + a * W + b * (W @ W)
    top = torch.cat([R, t[..., :, None]], -1)
    bottom = torch.zeros_like(top[..., :1, :])
    bottom[..., 0, 3] = 1.0
    return torch.cat([top, bottom], -2)


def apply_twists(extrinsics: Tensor, twists: Tensor) -> Tensor:
    """Camera-to-world extrinsics [..., 4, 4] moved by twists [..., 6] in the camera frame: E @ T(xi)."""
    return extrinsics @ twist_to_transform(twists)


def alignment_loss(twists: Tensor, extrinsics: Tensor, intrinsics: Tensor, near: Tensor, far: Tensor,
                   background_color: Tensor, gaussian_means: Tensor, gaussian_covariances: Tensor,
                   gaussian_sh_coefficients: Tensor, gaussian_opacities: Tensor, target: Tensor,
                   scale_invariant: bool = True) -> Tensor:
    """Per-view sum of squared errors [s, v] of the views rendered from E @ T(twists) against `target`
    [s, v, 3, h, w], through the fused loss epilogue (no colour image).  Differentiable with respect to `twists`
    [s, v, 6] (and whatever else requires grad)."""
    h, w = target.shape[-2:]
    sse, _, _ = render_views_mse(apply_twists(extrinsics, twists), intrinsics, near, far, (h, w), background_color,
                                 gaussian_means, gaussian_covariances, gaussian_sh_coefficients, gaussian_opacities,
                                 target, scale_invariant=scale_invariant, want_color=False)
    return sse


class AlignedPoses(NamedTuple):
    extrinsics: Tensor   # [s, v, 4, 4] refined camera-to-world extrinsics
    loss: Tensor         # [s, v] mean squared error per pixel and channel at the refined pose
    twists: Tensor       # [s, v, 6] the twists that were optimised: extrinsics = initial @ T(twists)


def align_poses(extrinsics: Tensor, intrinsics: Tensor, near: Tensor, far: Tensor, background_color: Tensor,
                gaussian_means: Tensor, gaussian_covariances: Tensor, gaussian_sh_coefficients: Tensor,
                gaussian_opacities: Tensor, target: Tensor, *, steps: int = 150, lr: float = 2e-3,
                scale_invariant: bool = True, initial_twists: Optional[Tensor] = None) -> AlignedPoses:
    """Refines the extrinsics [s, v, 4, 4] (camera-to-world) of s x v target views against their images `target`
    [s, v, 3, h, w], the Gaussians [s, g, ...] (render_views layouts) held fixed: `steps` Adam steps (learning rate
    `lr`) on one twist per view, starting from `initial_twists` [s, v, 6] (default 0).  Only the extrinsics are
    refined; intrinsics, near, far and the background are used as given.  The Gaussians are read, never written,
    and receive no gradient.  Each step is one rasterizer forward + camera-only backward and one Adam update, all
    on the device: the only host wait per step is the rasterizer's instance-count check."""
    s, v = extrinsics.shape[:2]
    if tuple(target.shape[:3]) != (s, v, 3):
        raise ValueError(f"target must be [s, v, 3, h, w] for extrinsics of shape {tuple(extrinsics.shape)}, "
                         f"got {tuple(target.shape)}")
    frozen = [t.detach() for t in (gaussian_means, gaussian_covariances, gaussian_sh_coefficients,
                                   gaussian_opacities)]
    ext = extrinsics.detach().to(torch.float32)
    cams = (intrinsics.detach(), near.detach(), far.detach(), background_color.detach())
    tgt = target.detach()
    xi = torch.zeros((s, v, 6), dtype=torch.float32, device=ext.device)
    if initial_twists is not None:
        xi.copy_(initial_twists.detach())
    xi.requires_grad_(True)
    opt = torch.optim.Adam([xi], lr=lr)
    for _ in range(int(steps)):
        opt.zero_grad(set_to_none=True)
        alignment_loss(xi, ext, *cams, *frozen, tgt, scale_invariant).sum().backward()
        opt.step()
    with torch.no_grad():
        sse = alignment_loss(xi, ext, *cams, *frozen, tgt, scale_invariant)
        h, w = target.shape[-2:]
        return AlignedPoses(apply_twists(ext, xi), sse / (3 * h * w), xi.detach().clone())
