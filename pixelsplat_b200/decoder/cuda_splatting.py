"""Drop-in for /root/reference/src/model/decoder/cuda_splatting.py: same public functions,
argument meaning and return values (`render_cuda` :47-127, `render_cuda_orthographic` :130-220,
`render_depth_cuda` :226-269, `get_projection_matrix` :17-44), re-designed so that a whole batch
of views is ONE forward call into the CUDA library:
  * no per-view Python loop, no `.item()` host syncs, no per-view workspace allocations;
  * the SH tensor is consumed in pixelSplat's native [g, 3, d_sh] layout and the covariance as
    [g, 3, 3] (no permute / triu-gather copies); the scale-invariant rescale is fused into the
    kernels;
  * `render_views` additionally lets V cameras share one Gaussian set, which removes
    DecoderSplattingCUDA's `repeat` of every Gaussian tensor (decoder_splatting_cuda.py:53-56).
"""
from __future__ import annotations

import ctypes
from math import isqrt
from typing import Literal, Optional

import torch
from torch import Tensor

from .. import _lib
from ..rasterizer import _rasterize, rasterize_gaussians

DepthRenderingMode = Literal["depth", "disparity", "relative_disparity", "log"]


def get_projection_matrix(near: Tensor, far: Tensor, fov_x: Tensor, fov_y: Tensor) -> Tensor:
    """Maps the frustum to (-1, 1) in X/Y and (0, 1) in Z, +Z forward (row-major [b, 4, 4])."""
    tan_x, tan_y = (0.5 * fov_x).tan(), (0.5 * fov_y).tan()
    top, right = tan_y * near, tan_x * near
    bottom, left = -top, -right
    (b,) = near.shape
    out = torch.zeros((b, 4, 4), dtype=torch.float32, device=near.device)
    out[:, 0, 0] = 2 * near / (right - left)
    out[:, 1, 1] = 2 * near / (top - bottom)
    out[:, 0, 2] = (right + left) / (right - left)
    out[:, 1, 2] = (top + bottom) / (top - bottom)
    out[:, 3, 2] = 1
    out[:, 2, 2] = far / (far - near)
    out[:, 2, 3] = -(far * near) / (far - near)
    return out


class _CameraSetup(torch.autograd.Function):
    """ps_camera_setup forward, ps_camera_setup_backward backward: (extrinsics, intrinsics) -> (viewmatrix,
    projmatrix, campos, tanfov, scene_scale).  near, far and scene_scale are not differentiated."""

    @staticmethod
    def forward(ctx, extrinsics, intrinsics, near, far, scale_invariant: bool):
        n = extrinsics.shape[0]
        dev = extrinsics.device
        f = lambda t: t.to(torch.float32).contiguous()
        e, k, nr, fr = f(extrinsics), f(intrinsics), f(near), f(far)
        view = torch.empty((n, 16), dtype=torch.float32, device=dev)
        proj = torch.empty((n, 16), dtype=torch.float32, device=dev)
        campos = torch.empty((n, 3), dtype=torch.float32, device=dev)
        tanfov = torch.empty((n, 2), dtype=torch.float32, device=dev)
        scale = torch.empty((n,), dtype=torch.float32, device=dev)
        p = lambda t: ctypes.c_void_p(t.data_ptr())
        stream = torch.cuda.current_stream(dev)
        rc = _lib.on_device(dev, _lib.lib.ps_camera_setup, n, p(e), p(k), p(nr), p(fr), 1 if scale_invariant else 0,
                            p(view), p(proj), p(campos), p(tanfov), p(scale), ctypes.c_void_p(stream.cuda_stream))
        _lib.check(rc, "ps_camera_setup")
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(scale)
        ctx.save_for_backward(e, k, nr, fr)
        ctx.scale_invariant = scale_invariant
        ctx.dtypes = (extrinsics.dtype, intrinsics.dtype)
        return view, proj, campos, tanfov, scale

    @staticmethod
    def backward(ctx, d_view, d_proj, d_campos, d_tanfov, _d_scale):
        e, k, nr, fr = ctx.saved_tensors
        n, dev = e.shape[0], e.device
        d_e = torch.empty((n, 4, 4), dtype=torch.float32, device=dev)
        d_k = torch.empty((n, 3, 3), dtype=torch.float32, device=dev)
        p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
        keep = [None if t is None else t.to(torch.float32).contiguous() for t in (d_view, d_proj, d_campos, d_tanfov)]
        stream = torch.cuda.current_stream(dev)
        rc = _lib.on_device(dev, _lib.lib.ps_camera_setup_backward, n, p(e), p(k), p(nr), p(fr),
                            1 if ctx.scale_invariant else 0, *[p(t) for t in keep], p(d_e), p(d_k),
                            ctypes.c_void_p(stream.cuda_stream))
        _lib.check(rc, "ps_camera_setup_backward")
        return (d_e.to(ctx.dtypes[0]) if ctx.needs_input_grad[0] else None,
                d_k.to(ctx.dtypes[1]) if ctx.needs_input_grad[1] else None, None, None, None)


def camera_setup(extrinsics: Tensor, intrinsics: Tensor, near: Tensor, far: Tensor,
                 scale_invariant: bool) -> dict[str, Tensor]:
    """[n,4,4], [n,3,3], [n], [n] -> rasterizer camera arrays, one kernel launch.  Differentiable with respect to
    extrinsics and intrinsics (one more launch in the backward); not with respect to near and far."""
    if not extrinsics.is_cuda:
        raise ValueError("extrinsics must be a CUDA tensor (pixelsplat_b200 has no CPU path)")
    view, proj, campos, tanfov, scale = _CameraSetup.apply(extrinsics, intrinsics, near, far, bool(scale_invariant))
    return dict(viewmatrix=view, projmatrix=proj, campos=campos, tanfov=tanfov, scene_scale=scale)


def _render(extrinsics: Tensor, intrinsics: Tensor, near: Tensor, far: Tensor, image_shape: tuple[int, int],
            background_color: Tensor, gaussian_means: Tensor, gaussian_covariances: Tensor,
            gaussian_sh_coefficients: Tensor, gaussian_opacities: Tensor, scale_invariant: bool, use_sh: bool = True,
            state_out: Optional[list] = None, target: Optional[Tensor] = None,
            mode: Optional[DepthRenderingMode] = None, want_color: bool = True, means2d: Optional[Tensor] = None):
    """One rasterizer call for [s, v] cameras over [s, g] Gaussians, with the loss epilogue when `target`
    [s, v, 3, h, w] is given, the depth channel when `mode` is, and the projected means' gradient into `means2d`
    [s v, g, 3] when it is given.  -> (color [s, v, 3, h, w] or None when want_color=False, depth [s, v, h, w] | None,
    sse [s, v] | None, sse_clipped [s, v] | None, radii [s v, g] int32)."""
    s, v = extrinsics.shape[:2]
    n = s * v
    h, w = image_shape
    cams = camera_setup(extrinsics.reshape(n, 4, 4), intrinsics.reshape(n, 3, 3), near.reshape(n), far.reshape(n),
                        scale_invariant)
    if use_sh:
        colors, layout = gaussian_sh_coefficients, _lib.PS_SH_3M
    else:
        colors, layout = gaussian_sh_coefficients[..., 0], _lib.PS_SH_M3
    color, depth, radii, sse, sse_clipped = _rasterize(
        gaussian_means, gaussian_covariances, gaussian_opacities, colors,
        viewmatrix=cams["viewmatrix"], projmatrix=cams["projmatrix"], campos=cams["campos"],
        tanfov=cams["tanfov"], background=background_color.reshape(n, 3).to(torch.float32),
        image_shape=(h, w), views_per_scene=v, sh_degree=isqrt(gaussian_sh_coefficients.shape[-1]) - 1,
        use_sh=use_sh, sh_layout=layout, scene_scale=cams["scene_scale"] if scale_invariant else None,
        state_out=state_out, target=None if target is None else target.reshape(n, 3, h, w).to(torch.float32),
        depth_mode=mode,
        near_far=None if mode is None else torch.stack([near.reshape(n), far.reshape(n)], -1).to(torch.float32),
        want_color=want_color, means2d=means2d)
    return (color.reshape(s, v, 3, h, w) if want_color else None,
            None if depth is None else depth.reshape(s, v, h, w),
            None if sse is None else sse.reshape(s, v),
            None if sse_clipped is None else sse_clipped.reshape(s, v), radii)


def render_views(
    extrinsics: Tensor,            # [s, v, 4, 4]
    intrinsics: Tensor,            # [s, v, 3, 3]
    near: Tensor,                  # [s, v]
    far: Tensor,                   # [s, v]
    image_shape: tuple[int, int],
    background_color: Tensor,      # [s, v, 3]
    gaussian_means: Tensor,        # [s, g, 3]
    gaussian_covariances: Tensor,  # [s, g, 3, 3]
    gaussian_sh_coefficients: Tensor,  # [s, g, 3, d_sh]
    gaussian_opacities: Tensor,    # [s, g]
    scale_invariant: bool = True,
    use_sh: bool = True,
    state_out: Optional[list] = None,
) -> Tensor:                       # [s, v, 3, h, w]
    """V cameras per scene share the scene's Gaussians (no `repeat`)."""
    assert use_sh or gaussian_sh_coefficients.shape[-1] == 1
    color, _, _, _, _ = _render(extrinsics, intrinsics, near, far, image_shape, background_color, gaussian_means,
                             gaussian_covariances, gaussian_sh_coefficients, gaussian_opacities, scale_invariant,
                             use_sh=use_sh, state_out=state_out)
    return color


def render_views_mse(extrinsics: Tensor, intrinsics: Tensor, near: Tensor, far: Tensor, image_shape: tuple[int, int],
                     background_color: Tensor, gaussian_means: Tensor, gaussian_covariances: Tensor,
                     gaussian_sh_coefficients: Tensor, gaussian_opacities: Tensor, target: Tensor,
                     scale_invariant: bool = True, want_color: bool = True):
    """render_views with the loss epilogue fused into the compositor (SURVEY.md 8 row f-4): `target`
    [s, v, 3, h, w] -> (sse [s, v] differentiable sum of squared errors, sse_clipped [s, v] the same on images
    clipped to [0, 1] (what compute_psnr needs), color [s, v, 3, h, w] detached or None).  See
    pixelsplat_b200/loss.py for the LossMse / PSNR built on top."""
    color, _, sse, sse_clipped, _ = _render(extrinsics, intrinsics, near, far, image_shape, background_color,
                                         gaussian_means, gaussian_covariances, gaussian_sh_coefficients,
                                         gaussian_opacities, scale_invariant, target=target, want_color=want_color)
    return sse, sse_clipped, color


def render_views_mse_means2d(extrinsics: Tensor, intrinsics: Tensor, near: Tensor, far: Tensor,
                             image_shape: tuple[int, int], background_color: Tensor, gaussian_means: Tensor,
                             gaussian_covariances: Tensor, gaussian_sh_coefficients: Tensor,
                             gaussian_opacities: Tensor, target: Tensor, means2d: Tensor, scale_invariant: bool = True,
                             want_color: bool = True):
    """render_views_mse with upstream's screen-space gradient holder: `means2d` [s v, g, 3], a tensor that requires
    grad, receives the gradient of the loss with respect to each view's projected means (3DGS's densification
    statistic).  -> (sse [s, v], sse_clipped [s, v], color or None, radii [s v, g] int32)."""
    color, _, sse, sse_clipped, radii = _render(extrinsics, intrinsics, near, far, image_shape, background_color,
                                                gaussian_means, gaussian_covariances, gaussian_sh_coefficients,
                                                gaussian_opacities, scale_invariant, target=target,
                                                want_color=want_color, means2d=means2d)
    return sse, sse_clipped, color, radii


def render_views_means2d(extrinsics: Tensor, intrinsics: Tensor, near: Tensor, far: Tensor,
                         image_shape: tuple[int, int], background_color: Tensor, gaussian_means: Tensor,
                         gaussian_covariances: Tensor, gaussian_sh_coefficients: Tensor, gaussian_opacities: Tensor,
                         means2d: Tensor, scale_invariant: bool = True):
    """render_views with the screen-space gradient holder of render_views_mse_means2d, for a loss computed on the
    colour render.  -> (color [s, v, 3, h, w] differentiable, radii [s v, g] int32)."""
    color, _, _, _, radii = _render(extrinsics, intrinsics, near, far, image_shape, background_color, gaussian_means,
                                    gaussian_covariances, gaussian_sh_coefficients, gaussian_opacities,
                                    scale_invariant, means2d=means2d)
    return color, radii


def _legacy_compositor() -> bool:
    """The legacy CTA-per-tile compositor (composite_impl = 1) has no depth channel."""
    return _lib.get_option("composite_impl") == 1


def render_views_with_depth(extrinsics: Tensor, intrinsics: Tensor, near: Tensor, far: Tensor,
                            image_shape: tuple[int, int], background_color: Tensor, gaussian_means: Tensor,
                            gaussian_covariances: Tensor, gaussian_sh_coefficients: Tensor, gaussian_opacities: Tensor,
                            scale_invariant: bool = True, mode: DepthRenderingMode = "depth",
                            state_out: Optional[list] = None) -> tuple[Tensor, Tensor]:
    """render_views and render_depth_views in one pass: the depth map is a fourth channel of the colour
    compositor (same visibility, sort order and alphas), not a second rasterization over per-view copies of the
    Gaussians.  -> (color [s, v, 3, h, w], depth [s, v, h, w]), both differentiable.  Under the legacy compositor
    the two are rendered separately, as render_views + render_depth_views."""
    if _legacy_compositor():
        color = render_views(extrinsics, intrinsics, near, far, image_shape, background_color, gaussian_means,
                             gaussian_covariances, gaussian_sh_coefficients, gaussian_opacities, scale_invariant,
                             state_out=state_out)
        return color, render_depth_views(extrinsics, intrinsics, near, far, image_shape, gaussian_means,
                                         gaussian_covariances, gaussian_opacities, scale_invariant, mode)
    color, depth, _, _, _ = _render(extrinsics, intrinsics, near, far, image_shape, background_color, gaussian_means,
                                 gaussian_covariances, gaussian_sh_coefficients, gaussian_opacities, scale_invariant,
                                 state_out=state_out, mode=mode)
    return color, depth


def render_views_mse_with_depth(extrinsics: Tensor, intrinsics: Tensor, near: Tensor, far: Tensor,
                                image_shape: tuple[int, int], background_color: Tensor, gaussian_means: Tensor,
                                gaussian_covariances: Tensor, gaussian_sh_coefficients: Tensor,
                                gaussian_opacities: Tensor, target: Tensor, scale_invariant: bool = True,
                                mode: DepthRenderingMode = "depth", want_color: bool = True):
    """render_views_mse with the depth channel of render_views_with_depth: -> (sse [s, v], sse_clipped [s, v],
    color [s, v, 3, h, w] detached or None, depth [s, v, h, w] differentiable)."""
    color, depth, sse, sse_clipped, _ = _render(extrinsics, intrinsics, near, far, image_shape, background_color,
                                             gaussian_means, gaussian_covariances, gaussian_sh_coefficients,
                                             gaussian_opacities, scale_invariant, target=target, mode=mode,
                                             want_color=want_color)
    return sse, sse_clipped, color, depth


def render_cuda(
    extrinsics: Tensor,            # [batch, 4, 4] camera-to-world
    intrinsics: Tensor,            # [batch, 3, 3] normalised
    near: Tensor,                  # [batch]
    far: Tensor,                   # [batch]
    image_shape: tuple[int, int],
    background_color: Tensor,      # [batch, 3]
    gaussian_means: Tensor,        # [batch, gaussian, 3]
    gaussian_covariances: Tensor,  # [batch, gaussian, 3, 3]
    gaussian_sh_coefficients: Tensor,  # [batch, gaussian, 3, d_sh]
    gaussian_opacities: Tensor,    # [batch, gaussian]
    scale_invariant: bool = True,
    use_sh: bool = True,
) -> Tensor:                       # [batch, 3, height, width]
    """Reference signature (cuda_splatting.py:47-60): every batch element brings its own Gaussians."""
    out = render_views(extrinsics[:, None], intrinsics[:, None], near[:, None], far[:, None],
                       image_shape, background_color[:, None], gaussian_means, gaussian_covariances,
                       gaussian_sh_coefficients, gaussian_opacities, scale_invariant, use_sh)
    return out[:, 0]


def render_cuda_orthographic(
    extrinsics: Tensor, width: Tensor, height: Tensor, near: Tensor, far: Tensor,
    image_shape: tuple[int, int], background_color: Tensor, gaussian_means: Tensor,
    gaussian_covariances: Tensor, gaussian_sh_coefficients: Tensor, gaussian_opacities: Tensor,
    fov_degrees: float = 0.1, use_sh: bool = True, dump: dict | None = None,
) -> Tensor:
    """Fake orthographic projection: camera moved far back with a tiny field of view
    (cuda_splatting.py:130-220).  Visualisation path: camera math stays in torch."""
    b = extrinsics.shape[0]
    h, w = image_shape
    assert use_sh or gaussian_sh_coefficients.shape[-1] == 1
    n = gaussian_sh_coefficients.shape[-1]
    degree = isqrt(n) - 1
    dev = extrinsics.device
    fov_x = torch.tensor(fov_degrees, device=dev).deg2rad()
    tan_fov_x = (0.5 * fov_x).tan()
    distance_to_near = (0.5 * width) / tan_fov_x
    tan_fov_y = 0.5 * height / distance_to_near
    fov_y = (2 * tan_fov_y).atan()
    near = near + distance_to_near
    far = far + distance_to_near
    move_back = torch.eye(4, dtype=torch.float32, device=dev).repeat(b, 1, 1)
    move_back[:, 2, 3] = -distance_to_near
    extrinsics = extrinsics @ move_back
    if dump is not None:
        dump["extrinsics"], dump["fov_x"], dump["fov_y"] = extrinsics, fov_x, fov_y
        dump["near"], dump["far"] = near, far
    proj = get_projection_matrix(near, far, fov_x.expand(b), fov_y).transpose(1, 2)
    view = extrinsics.inverse().transpose(1, 2)
    full = view @ proj
    tanfov = torch.stack([tan_fov_x.expand(b), tan_fov_y.expand(b)], -1).to(torch.float32)
    if use_sh:
        colors, layout = gaussian_sh_coefficients, _lib.PS_SH_3M
    else:
        colors, layout = gaussian_sh_coefficients[..., 0], _lib.PS_SH_M3
    color, _ = rasterize_gaussians(
        gaussian_means, gaussian_covariances, gaussian_opacities, colors,
        viewmatrix=view.reshape(b, 16), projmatrix=full.reshape(b, 16),
        campos=extrinsics[:, :3, 3], tanfov=tanfov, background=background_color.to(torch.float32),
        image_shape=(h, w), views_per_scene=1, sh_degree=degree, use_sh=use_sh, sh_layout=layout)
    return color


def _relative_disparity(depth: Tensor, near: Tensor, far: Tensor, eps: float = 1e-10) -> Tensor:
    disp_near, disp_far, disp = 1 / (near + eps), 1 / (far + eps), 1 / (depth + eps)
    return 1 - (disp - disp_far) / (disp_near - disp_far + eps)


def depth_colors(extrinsics: Tensor, gaussian_means: Tensor, near: Tensor, far: Tensor,
                 mode: DepthRenderingMode = "depth") -> Tensor:
    """The per-Gaussian "colour" render_depth_cuda composites (cuda_splatting.py:238-251): camera-space z
    of every Gaussian, optionally as disparity / relative disparity / log.  [s, v] cameras over [s, g]
    Gaussians -> [s, v, g].  Pure torch (any device)."""
    w2c = extrinsics.inverse()                                      # [s, v, 4, 4]
    fake = torch.einsum("svj,sgj->svg", w2c[:, :, 2, :3], gaussian_means) + w2c[:, :, 2, 3:4]
    if mode == "disparity":
        fake = 1 / fake
    elif mode == "relative_disparity":
        fake = _relative_disparity(fake, near[..., None], far[..., None])
    elif mode == "log":
        fake = fake.minimum(near[..., None]).maximum(far[..., None]).log()
    return fake


def render_depth_views(extrinsics, intrinsics, near, far, image_shape, gaussian_means,
                       gaussian_covariances, gaussian_opacities, scale_invariant=True,
                       mode: DepthRenderingMode = "depth") -> Tensor:
    """[s, v] cameras over [s, g] Gaussians -> [s, v, h, w].  Depth is rendered as a colour
    (cuda_splatting.py:238-269); because the colour depends on the camera, each view needs its
    own colour set, so the views are flattened into scenes here."""
    s, v = extrinsics.shape[:2]
    fake = depth_colors(extrinsics, gaussian_means, near, far, mode)
    g = gaussian_means.shape[1]
    rep = lambda t: t[:, None].expand(s, v, *t.shape[1:]).reshape(s * v, *t.shape[1:])
    colors = fake.reshape(s * v, g, 1, 1).expand(s * v, g, 3, 1)
    out = render_cuda(extrinsics.reshape(s * v, 4, 4), intrinsics.reshape(s * v, 3, 3),
                      near.reshape(s * v), far.reshape(s * v), image_shape,
                      torch.zeros((s * v, 3), dtype=fake.dtype, device=fake.device),
                      rep(gaussian_means), rep(gaussian_covariances), colors, rep(gaussian_opacities),
                      scale_invariant=scale_invariant, use_sh=False)
    return out.mean(dim=1).reshape(s, v, *image_shape)


def render_depth_cuda(extrinsics, intrinsics, near, far, image_shape, gaussian_means,
                      gaussian_covariances, gaussian_opacities, scale_invariant: bool = True,
                      mode: DepthRenderingMode = "depth") -> Tensor:
    """Reference signature (cuda_splatting.py:226-237): [batch] cameras, [batch, g] Gaussians."""
    out = render_depth_views(extrinsics[:, None], intrinsics[:, None], near[:, None], far[:, None],
                             image_shape, gaussian_means, gaussian_covariances, gaussian_opacities,
                             scale_invariant, mode)
    return out[:, 0]
