"""Videos of a scene: the reference's camera trajectories (src/visualization/camera_trajectory/{interpolation,
wobble}.py) and its three validation videos (ModelWrapper.render_video_interpolation, render_video_wobble and
render_video_interpolation_exaggerated), each frame the reference's layout of colour and depth, probabilistic on
the left and deterministic on the right.

- `interpolate_extrinsics`, `interpolate_intrinsics`, `generate_wobble_transformation` and `generate_wobble` are
  drop-ins with the reference's signatures, broadcasting and arithmetic (float64 inside, scipy's YXZ Euler angles).
- `video_trajectory(context, target, name)` is the cameras of one video; `render_video` renders it from one scene's
  encoder trunk and writes nothing; `write_mp4` encodes frames with OpenCV.

The GPU work is the encoder and the multi-view render with the fused depth channel; quantiles, the colour table
lookup and the layout are torch ops on the device, and the colour panels go through the frame pass of
csrc/eval_images.cu.
"""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass
from pathlib import Path
from typing import Callable, Optional

import numpy as np
import torch
from scipy.spatial.transform import Rotation
from torch import Tensor

from .encoder.encoder_tail import EncoderEpipolarTail
from .evaluation.frames import frame_pass
from .evaluation.image_io import comparison_layout
from .evaluation.metrics import CHUNK

QUANTILE_LIMIT = 16_000_000   # the reference's slice before each quantile (torch.quantile takes at most 2^24 values)
FPS = 30


# ---- trajectories: src/visualization/camera_trajectory/interpolation.py, wobble.py ---------------------------------

def interpolate_intrinsics(initial: Tensor, final: Tensor, t: Tensor) -> Tensor:
    """[*batch, 3, 3] x2, t [T] -> [*batch, T, 3, 3]: the linear blend initial + (final - initial) t."""
    a, b = initial[..., None, :, :], final[..., None, :, :]
    return a + (b - a) * t[:, None, None]


def _intersect_rays(a_origins: Tensor, a_directions: Tensor, b_origins: Tensor, b_directions: Tensor) -> Tensor:
    """The least-squares point nearest to two rays: sum_i (n_i n_i^T - I) p = sum_i (n_i n_i^T - I) o_i."""
    a_origins, a_directions, b_origins, b_directions = torch.broadcast_tensors(a_origins, a_directions, b_origins,
                                                                              b_directions)
    origins = torch.stack((a_origins, b_origins), dim=-2)
    directions = torch.stack((a_directions, b_directions), dim=-2)
    n = torch.einsum("...ni,...nj->...nij", directions, directions) - torch.eye(3, dtype=origins.dtype,
                                                                                 device=origins.device)
    lhs = n.sum(dim=-3)
    rhs = torch.einsum("...nij,...nj->...ni", n, origins).sum(dim=-2)
    return torch.linalg.lstsq(lhs, rhs).solution


def _normalize(a: Tensor) -> Tensor:
    return a / a.norm(dim=-1, keepdim=True)


def _coordinate_frame(y: Tensor, z: Tensor) -> Tensor:
    """The matrix with columns (y x z, y, z)."""
    y, z = torch.broadcast_tensors(y, z)
    return torch.stack([torch.linalg.cross(y, z), y, z], dim=-1)


def _rotation_coordinate_frame(a: Tensor, b: Tensor, eps: float) -> Tensor:
    """A frame whose Y axis is normal to the plane of unit vectors a and b and whose Z axis is a.  A b (anti)parallel
    to a is replaced by +z, and where that is parallel too, by +y."""
    b = b.detach().clone()
    for replacement in ((0, 0, 1), (0, 1, 0)):
        parallel = (torch.einsum("...i,...i->...", a, b).abs() - 1).abs() < eps
        b[parallel] = torch.tensor(replacement, dtype=b.dtype, device=b.device)
    return _coordinate_frame(_normalize(torch.linalg.cross(a, b)), a)


def _matrix_to_euler(rotations: Tensor, pattern: str) -> Tensor:
    shape = rotations.shape[:-2]
    angles = Rotation.from_matrix(rotations.detach().reshape(-1, 3, 3).cpu().numpy()).as_euler(pattern)
    return torch.tensor(angles, dtype=rotations.dtype, device=rotations.device).reshape(*shape, 3)


def _euler_to_matrix(angles: Tensor, pattern: str) -> Tensor:
    shape = angles.shape[:-1]
    matrices = Rotation.from_euler(pattern, angles.detach().reshape(-1, 3).cpu().numpy()).as_matrix()
    return torch.tensor(matrices, dtype=angles.dtype, device=angles.device).reshape(*shape, 3, 3)


def _to_pivot_parameters(extrinsics: Tensor, pivot_frame: Tensor, pivot_point: Tensor) -> Tensor:
    """Camera-to-world [*batch, 4, 4] -> [*batch, 5]: the pivot point's offset from the camera in the frame
    (look x pivot axis, pivot axis, look), then the YXZ Euler angles Y and Z of the rotation in the pivot frame."""
    translation_frame = _coordinate_frame(pivot_frame[..., :, 1], extrinsics[..., :3, 2])
    delta = pivot_point - extrinsics[..., :3, 3]
    translation = torch.einsum("...ij,...i->...j", translation_frame, delta)
    y, _, z = _matrix_to_euler(pivot_frame.inverse() @ extrinsics[..., :3, :3], "YXZ").unbind(dim=-1)
    return torch.cat([translation, y[..., None], z[..., None]], dim=-1)


def _from_pivot_parameters(parameters: Tensor, pivot_frame: Tensor, pivot_point: Tensor) -> Tensor:
    translation, y, z = parameters.split((3, 1, 1), dim=-1)
    rotation = pivot_frame @ _euler_to_matrix(torch.cat((y, torch.zeros_like(y), z), dim=-1), "YXZ")
    translation_frame = _coordinate_frame(pivot_frame[..., :, 1], rotation[..., :3, 2])
    origin = pivot_point - torch.einsum("...ij,...j->...i", translation_frame, translation)
    extrinsics = torch.eye(4, dtype=parameters.dtype, device=parameters.device)
    extrinsics = extrinsics.broadcast_to((*origin.shape[:-1], 4, 4)).clone()
    extrinsics[..., :3, :3] = rotation
    extrinsics[..., :3, 3] = origin
    return extrinsics


def _interpolate_circular(a: Tensor, b: Tensor, t: Tensor) -> Tensor:
    """Angles a -> b along the shorter way round: the direct blend, or the one from a - 2 pi, or from a + 2 pi."""
    a, b, t = torch.broadcast_tensors(a, b, t)
    tau = 2 * math.pi
    a, b = a % tau, b % tau
    a_left, a_right = a - tau, a + tau
    d, d_left, d_right = (b - a).abs(), (b - a_left).abs(), (b - a_right).abs()
    use_d = (d < d_left) & (d < d_right)
    use_left = (d_left < d_right) & ~use_d
    use_right = ~use_d & ~use_left
    result = a + (b - a) * t
    result[use_left] = (a_left + (b - a_left) * t)[use_left]
    result[use_right] = (a_right + (b - a_right) * t)[use_right]
    return result


@torch.no_grad()
def interpolate_extrinsics(initial: Tensor, final: Tensor, t: Tensor, eps: float = 1e-4) -> Tensor:
    """Camera-to-world [*batch, 4, 4] x2, t [T] -> float32 [*batch, T, 4, 4]: both cameras in pivot parameters about
    their focus point (the least-squares meeting point of the look rays; their origins' midpoint when the looks are
    parallel within `eps`), the translations blended linearly and the two angles circularly, in float64."""
    initial, final, t = initial.double(), final.double(), t.double()
    initial_look, final_look = initial[..., :3, 2], final[..., :3, 2]
    parallel = (torch.einsum("...i,...i->...", initial_look, final_look).abs() - 1).abs() < eps
    initial_origin, final_origin = initial[..., :3, 3], final[..., :3, 3]
    pivot_point = 0.5 * (initial_origin + final_origin)
    pivot_point[~parallel] = _intersect_rays(initial_origin[~parallel], initial_look[~parallel],
                                             final_origin[~parallel], final_look[~parallel])
    pivot_frame = _rotation_coordinate_frame(initial_look, final_look, eps)
    p0 = _to_pivot_parameters(initial, pivot_frame, pivot_point)[..., None, :]
    p1 = _to_pivot_parameters(final, pivot_frame, pivot_point)[..., None, :]
    tt = t[:, None]
    blended = torch.cat((p0[..., :3] + (p1[..., :3] - p0[..., :3]) * tt,
                         _interpolate_circular(p0[..., 3:], p1[..., 3:], tt)), dim=-1)
    return _from_pivot_parameters(blended.float(), pivot_frame[..., None, :, :].float(),
                                  pivot_point[..., None, :].float())


@torch.no_grad()
def generate_wobble_transformation(radius: Tensor, t: Tensor, num_rotations: int = 1,
                                   scale_radius_with_t: bool = True) -> Tensor:
    """radius [*batch], t [T] -> float32 [*batch, T, 4, 4]: translations in the image plane round a circle,
    (sin, -cos)(2 pi num_rotations t) times the radius (times t when `scale_radius_with_t`)."""
    tf = torch.eye(4, dtype=torch.float32, device=t.device).broadcast_to((*radius.shape, t.shape[0], 4, 4)).clone()
    radius = radius[..., None]
    if scale_radius_with_t:
        radius = radius * t
    angle = 2 * math.pi * num_rotations * t
    tf[..., 0, 3] = torch.sin(angle) * radius
    tf[..., 1, 3] = -torch.cos(angle) * radius
    return tf


@torch.no_grad()
def generate_wobble(extrinsics: Tensor, radius: Tensor, t: Tensor) -> Tensor:
    """[*batch, 4, 4], radius [*batch], t [T] -> [*batch, T, 4, 4]: each camera moved by its wobble."""
    return extrinsics[..., None, :, :] @ generate_wobble_transformation(radius, t)


# ---- spin: src/visualization/camera_trajectory/spin.py --------------------------------------------------------------

def generate_spin(num_frames: int, device, elevation: float, radius: float) -> Tensor:
    """The reference's generate_spin: float32 camera-to-world [num_frames, 4, 4] orbiting the origin about +y at
    `radius`, raised by `elevation` degrees, each camera looking at the origin with its up vector (-Y) along +y at
    zero elevation."""
    tf_translation = torch.eye(4, dtype=torch.float32, device=device)
    tf_translation[:2] *= -1
    tf_translation[2, 3] = -radius
    phi = 2 * np.pi * (np.arange(num_frames) / num_frames)
    rotation_vectors = np.stack([np.zeros_like(phi), phi, np.zeros_like(phi)], axis=-1)
    azimuth = torch.tensor(Rotation.from_rotvec(rotation_vectors).as_matrix(), dtype=torch.float32, device=device)
    tf_azimuth = torch.eye(4, dtype=torch.float32, device=device).repeat(num_frames, 1, 1)
    tf_azimuth[:, :3, :3] = azimuth
    tilt = Rotation.from_rotvec(np.array([np.deg2rad(elevation), 0, 0], dtype=np.float32))
    tf_elevation = torch.eye(4, dtype=torch.float32, device=device)
    tf_elevation[:3, :3] = torch.tensor(tilt.as_matrix())
    return tf_azimuth @ tf_elevation @ tf_translation


# +y -> +z, +z -> -y: the reference's spin turned to orbit the up axis of the PLY export frame (+z)
_Y_UP_TO_Z_UP = ((1.0, 0.0, 0.0, 0.0), (0.0, 0.0, -1.0, 0.0), (0.0, 1.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0))


def spin_trajectory(num_frames: int, radius: float, elevation: float) -> tuple[Tensor, Tensor, Tensor, Tensor]:
    """Cameras orbiting the origin of a PLY export frame about its +z up axis: float32 extrinsics [T, 4, 4],
    the intrinsics the reference's test_splatter script renders its spin with (fx = fy = 0.5, centred) [T, 3, 3],
    near = radius / 100 and far = 2 radius [T], on the host."""
    extrinsics = torch.tensor(_Y_UP_TO_Z_UP, dtype=torch.float32) @ generate_spin(num_frames, "cpu", elevation, radius)
    k = torch.tensor([[0.5, 0.0, 0.5], [0.0, 0.5, 0.5], [0.0, 0.0, 1.0]], dtype=torch.float32)
    near = torch.full((num_frames,), radius / 100, dtype=torch.float32)
    far = torch.full((num_frames,), 2 * radius, dtype=torch.float32)
    return extrinsics, k.expand(num_frames, 3, 3).contiguous(), near, far


@torch.no_grad()
def render_spin(decoder, gaussians, num_frames: int, radius: float, elevation: float, shape: tuple[int, int],
                log: Optional[Callable[[str], None]] = print) -> Tensor:
    """The spin of one scene's `gaussians` (batch 1, on the device): uint8 [T, h, 2 w, 3] on the host, colour on
    the left and turbo depth on the right."""
    device = gaussians.means.device
    extrinsics, intrinsics, near, far = (t.to(device)[None] for t in spin_trajectory(num_frames, radius, elevation))
    color, depth = _render_panels(decoder, gaussians, extrinsics, intrinsics, near, far, shape, log)
    return torch.cat([color, depth], dim=-1).permute(0, 2, 3, 1).cpu()


# ---- the three videos: ModelWrapper.render_video_* -----------------------------------------------------------------

@dataclass(frozen=True)
class VideoSpec:
    num_frames: int
    smooth: bool
    loop_reverse: bool
    needs_two_views: bool   # the wobble radius is the distance between context views 0 and 1


VIDEOS = {
    "rgb": VideoSpec(30, True, True, False),
    "wobble": VideoSpec(60, True, True, True),
    "interpolation_exagerrated": VideoSpec(300, False, False, True),   # the reference's spelling
}
VALIDATION_VIDEOS = ("rgb", "wobble")


def time_steps(num_frames: int, smooth: bool) -> Tensor:
    """render_video_generic's float32 time base on the host: linspace(0, 1), eased by (cos(pi (t + 1)) + 1) / 2."""
    t = torch.linspace(0, 1, num_frames, dtype=torch.float32)
    return (torch.cos(torch.pi * (t + 1)) + 1) / 2 if smooth else t


def num_video_frames(name: str) -> int:
    """Frames of the written video: loop-reversed videos play forward and back, 2 n - 2 frames."""
    spec = VIDEOS[name]
    return 2 * spec.num_frames - 2 if spec.loop_reverse else spec.num_frames


def video_trajectory(context: dict, target: dict, name: str) -> Optional[tuple[Tensor, Tensor]]:
    """The cameras of video `name` for scene 0 of a (shimmed) batch: float32 extrinsics [T, 4, 4] and intrinsics
    [T, 3, 3] on the host, or None when the video needs two context views and the batch has another number (the
    reference skips it).  The interpolation ends at context view 1, or at target 0 without two context views.
    Computed on the host, where the trajectory functions are pinned against the reference."""
    spec = VIDEOS[name]
    ext = context["extrinsics"][0].detach().float().cpu()
    intr = context["intrinsics"][0].detach().float().cpu()
    v = ext.shape[0]
    if spec.needs_two_views and v != 2:
        return None
    end_ext = ext[1] if v == 2 else target["extrinsics"][0, 0].detach().float().cpu()
    end_intr = intr[1] if v == 2 else target["intrinsics"][0, 0].detach().float().cpu()
    t = time_steps(spec.num_frames, spec.smooth)
    if name == "rgb":
        return interpolate_extrinsics(ext[0], end_ext, t), interpolate_intrinsics(intr[0], end_intr, t)
    delta = (ext[0, :3, 3] - ext[1, :3, 3]).norm(dim=-1)
    if name == "wobble":
        return generate_wobble(ext[0], delta * 0.25, t), intr[0].expand(spec.num_frames, 3, 3)
    tf = generate_wobble_transformation(delta * 0.5, t, 5, scale_radius_with_t=False)
    return interpolate_extrinsics(ext[0], end_ext, t * 5 - 2) @ tf, interpolate_intrinsics(intr[0], end_intr, t * 5 - 2)


@functools.cache
def turbo_table() -> np.ndarray:
    """OpenCV's turbo colour map as uint8 RGB [256, 3]."""
    cv2 = _cv2()
    bgr = cv2.applyColorMap(np.arange(256, dtype=np.uint8)[:, None], cv2.COLORMAP_TURBO)[:, 0]
    return np.ascontiguousarray(bgr[:, ::-1])


def depth_color_index(depth: Tensor) -> Optional[Tensor]:
    """The colour-table entry of each depth value under the reference's depth_map, int64 in [0, 256] (256: NaN,
    drawn black), or None when no depth is positive.  In float32 as the reference:
        near = log quantile_0.01(d[d > 0][:16e6]),  far = log quantile_0.99(d.view(-1)[:16e6]),
        x = clip(1 - (log d - near) / (far - near), 0, 1),  entry = min(floor(256 x), 255)   (matplotlib's rule)."""
    positive = depth[depth > 0][:QUANTILE_LIMIT]
    if positive.numel() == 0:
        return None
    near = positive.quantile(0.01).log()
    far = depth.reshape(-1)[:QUANTILE_LIMIT].quantile(0.99).log()
    x = (1 - (depth.log() - near) / (far - near)).clip(0, 1)
    return torch.where(x.isnan(), 256, (x * 256).long().clamp_max(255))


def depth_panels(depth: Tensor, log: Optional[Callable[[str], None]] = print) -> Tensor:
    """depth [T, h, w] -> uint8 [T, h, w, 3]: the turbo entries of `depth_color_index` (black without positive
    depth, with one line to `log`)."""
    table = torch.zeros(257, 3, dtype=torch.uint8)
    table[:256] = torch.from_numpy(turbo_table())
    index = depth_color_index(depth)
    if index is None:
        if log is not None:
            log(f"video: no positive depth in {depth.shape[0]} frames; the depth panels are black")
        index = torch.full_like(depth, 256, dtype=torch.long)
    return table.to(depth.device)[index]


def _render_panels(decoder, gaussians, extrinsics: Tensor, intrinsics: Tensor, near: Tensor, far: Tensor,
                   shape: tuple[int, int], log) -> tuple[Tensor, Tensor]:
    """Colour and depth panels, uint8 [T, 3, h, w] each (channel-first views of [T, h, w, 3]): the render in chunks of
    CHUNK views with the fused depth channel, the colour quantised by the frame pass."""
    color, depth = [], []
    for i in range(0, extrinsics.shape[1], CHUNK):
        out = decoder.forward(gaussians, extrinsics[:, i:i + CHUNK], intrinsics[:, i:i + CHUNK],
                              near[:, i:i + CHUNK], far[:, i:i + CHUNK], shape, depth_mode="depth")
        color.append(frame_pass(out.color[0], frames=True, planes=False).frames)
        depth.append(out.depth[0])
    return (torch.cat(color).permute(0, 3, 1, 2), depth_panels(torch.cat(depth), log).permute(0, 3, 1, 2))


@torch.no_grad()
def render_video(encoder, decoder, context: dict, target: dict, name: str, global_step: int = 0,
                 features: Optional[Tensor] = None, log: Optional[Callable[[str], None]] = print) -> Optional[Tensor]:
    """Video `name` ("rgb", "wobble" or "interpolation_exagerrated") of scene 0 of a shimmed batch, as
    ModelWrapper.render_video_generic draws it without its text labels: uint8 [T, H, W, 3] on the host (536 x 536
    at 256 x 256), or None when the video needs two context views and the batch has another number.

    `features` is `encoder.trunk(context)[0]`, computed here when not given: one trunk can serve every video of a
    scene.  The tails run probabilistic then deterministic, so with two context views the draws are those of the
    reference's two full encoder calls."""
    cameras = video_trajectory(context, target, name)
    if cameras is None:
        return None
    if features is None:
        features, _ = encoder.trunk(context)
    device = context["extrinsics"].device
    extrinsics, intrinsics = (c.to(device).contiguous()[None] for c in cameras)
    frames = extrinsics.shape[1]
    near = context["near"][:1, :1].expand(-1, frames).contiguous()
    far = context["far"][:1, :1].expand(-1, frames).contiguous()
    shape = tuple(context["image"].shape[-2:])
    columns = []
    for deterministic in (False, True):
        gaussians = EncoderEpipolarTail.forward(encoder, features, context, global_step, deterministic)
        columns.append(_render_panels(decoder, gaussians, extrinsics, intrinsics, near, far, shape, log))
    video = comparison_layout(*columns).permute(0, 2, 3, 1).cpu()
    if VIDEOS[name].loop_reverse:
        video = torch.cat([video, video.flip(0)[1:-1]])
    return video


# ---- files ---------------------------------------------------------------------------------------------------------

def _cv2():
    try:
        import cv2
    except ImportError as e:
        raise ImportError("pixelsplat_b200.video needs OpenCV for the turbo colour table and the MP4 encoder: "
                          "install opencv-python-headless") from e
    return cv2


def write_mp4(frames, path: Path | str, fps: int = FPS) -> Path:
    """uint8 RGB frames [T, H, W, 3] (array or tensor) -> an MPEG-4 Part 2 ("mp4v") file, creating the parent
    directory."""
    cv2 = _cv2()
    frames = np.asarray(frames)
    if frames.dtype != np.uint8 or frames.ndim != 4 or frames.shape[-1] != 3 or len(frames) == 0:
        raise ValueError(f"write_mp4: expected uint8 frames [T > 0, H, W, 3], got {frames.dtype} {frames.shape}")
    path = Path(path)
    path.parent.mkdir(parents=True, exist_ok=True)
    _, h, w, _ = frames.shape
    writer = cv2.VideoWriter(str(path), cv2.VideoWriter_fourcc(*"mp4v"), fps, (w, h))
    if not writer.isOpened():
        raise RuntimeError(f"write_mp4: OpenCV cannot open an mp4v writer for {path}")
    try:
        for frame in frames:
            writer.write(np.ascontiguousarray(frame[..., ::-1]))
    finally:
        writer.release()
    return path
