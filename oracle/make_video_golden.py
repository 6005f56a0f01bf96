"""Generates tests/golden/video_trajectories_v1.npz by running the REFERENCE's camera trajectory functions
(src/visualization/camera_trajectory/{interpolation,wobble}.py) on the CPU.  Authoring container only:

    python oracle/make_video_golden.py

TEST INFRASTRUCTURE.  The trajectory modules need torch, einops, jaxtyping and scipy only; everything run here is
the reference's own code.  The time bases are render_video_generic's (linspace, cosine easing), computed here as it
computes them.  Stored per camera pair `<case>/...`:

    initial, final              float32 [4, 4] camera-to-world     k0, k1   float32 [3, 3]
    rgb_extrinsics              interpolate_extrinsics(initial, final, t_rgb)              [30, 4, 4]
    rgb_intrinsics              interpolate_intrinsics(k0, k1, t_rgb)                      [30, 3, 3]
    exaggerated_extrinsics      interpolate_extrinsics(initial, final, t_exaggerated * 5 - 2) @ the 5-turn wobble
    exaggerated_intrinsics      interpolate_intrinsics(k0, k1, t_exaggerated * 5 - 2)      [300, 3, 3]
    wobble_extrinsics           generate_wobble(initial, 0.25 |o0 - o1|, t_wobble)         [60, 4, 4]
    wobble_tf, exaggerated_tf   the wobble transformations of both videos

and once: t_rgb, t_wobble, t_exaggerated, t_exaggerated_5t_minus_2, the batched interpolation of every pair
(`batch/...`), and interpolate_circular on crafted angles (`circular/...`, every branch).
"""
from __future__ import annotations

import math
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
REFERENCE = Path("/root/reference")
OUT = ROOT / "tests" / "golden" / "video_trajectories_v1.npz"


def reference():
    if str(REFERENCE) not in sys.path:
        sys.path.insert(0, str(REFERENCE))
    from src.visualization.camera_trajectory import interpolation, wobble
    return interpolation, wobble


def camera(yaw: float, pitch: float, roll: float, origin) -> torch.Tensor:
    """Camera-to-world from OpenCV-style angles (degrees): yaw about world y, pitch about x, roll about the look."""
    from scipy.spatial.transform import Rotation
    e = torch.eye(4, dtype=torch.float32)
    e[:3, :3] = torch.tensor(Rotation.from_euler("YXZ", [yaw, pitch, roll], degrees=True).as_matrix())
    e[:3, 3] = torch.tensor(origin, dtype=torch.float32)
    return e


def intrinsics(fx, fy, cx, cy) -> torch.Tensor:
    return torch.tensor([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], dtype=torch.float32)


K = intrinsics(0.86, 0.86, 0.5, 0.5)
CASES = {
    # converging looks, the least-squares focus point
    "general": (camera(10, 5, 2, [0.0, 0.0, 0.0]), camera(-25, -8, -4, [1.0, 0.1, 0.2]), K, K),
    # identical looks off the z axis: the midpoint pivot, b replaced by +z
    "parallel": (camera(30, 10, 0, [0.0, 0.0, 0.0]), camera(30, 10, 0, [0.5, -0.2, 0.3]), K, K),
    # opposite looks: the midpoint pivot
    "anti_parallel": (camera(20, 0, 0, [0.0, 0.0, 0.0]), camera(200, 0, 0, [0.0, 0.0, 2.0]), K, K),
    # both looks along +z: b replaced by +z, which is parallel too, then by +y
    "replaced_b": (camera(0, 0, 0, [0.0, 0.0, 0.0]), camera(0, 0, 15, [0.3, 0.1, 0.0]), K, K),
    # world yaws either side of +-180 degrees, with rolls that put the pivot twists either side of 0: the left and
    # the right branch of interpolate_circular
    "yaw_wrap_left": (camera(175, 0, -14, [0.0, 0.0, 0.0]), camera(-170, 3, -8, [0.4, 0.0, -0.1]), K, K),
    "yaw_wrap_right": (camera(175, 0, -8, [0.0, 0.0, 0.0]), camera(-170, 3, -14, [0.4, 0.0, -0.1]), K, K),
    # looking almost straight down
    "near_gimbal_pitch": (camera(10, 89.9, 0, [0.0, 0.0, 0.0]), camera(40, 89.5, 5, [0.2, 0.0, 0.1]), K, K),
    # different fx / fy and principal points
    "anisotropic": (camera(5, -3, 1, [0.0, 0.0, 0.0]), camera(-12, 4, 0, [0.6, 0.0, 0.1]),
                    intrinsics(0.9, 1.3, 0.45, 0.55), intrinsics(1.1, 0.7, 0.52, 0.48)),
}


def time_steps(n: int, smooth: bool) -> torch.Tensor:
    t = torch.linspace(0, 1, n, dtype=torch.float32)
    return (torch.cos(torch.pi * (t + 1)) + 1) / 2 if smooth else t


def main() -> None:
    interpolation, wobble = reference()
    t_rgb, t_wobble, t_exaggerated = time_steps(30, True), time_steps(60, True), time_steps(300, False)
    t_5 = t_exaggerated * 5 - 2
    out = {"t_rgb": t_rgb, "t_wobble": t_wobble, "t_exaggerated": t_exaggerated, "t_exaggerated_5t_minus_2": t_5}
    for name, (e0, e1, k0, k1) in CASES.items():
        delta = (e0[:3, 3] - e1[:3, 3]).norm(dim=-1)
        tf = wobble.generate_wobble_transformation(delta * 0.5, t_exaggerated, 5, scale_radius_with_t=False)
        out.update({
            f"{name}/initial": e0, f"{name}/final": e1, f"{name}/k0": k0, f"{name}/k1": k1,
            f"{name}/rgb_extrinsics": interpolation.interpolate_extrinsics(e0, e1, t_rgb),
            f"{name}/rgb_intrinsics": interpolation.interpolate_intrinsics(k0, k1, t_rgb),
            f"{name}/exaggerated_extrinsics": interpolation.interpolate_extrinsics(e0, e1, t_5) @ tf,
            f"{name}/exaggerated_intrinsics": interpolation.interpolate_intrinsics(k0, k1, t_5),
            f"{name}/exaggerated_tf": tf,
            f"{name}/wobble_extrinsics": wobble.generate_wobble(e0, delta * 0.25, t_wobble),
            f"{name}/wobble_tf": wobble.generate_wobble_transformation(delta * 0.25, t_wobble),
        })
    e0 = torch.stack([c[0] for c in CASES.values()])
    e1 = torch.stack([c[1] for c in CASES.values()])
    radius = (e0[:, :3, 3] - e1[:, :3, 3]).norm(dim=-1)
    out.update({"batch/extrinsics": interpolation.interpolate_extrinsics(e0, e1, t_rgb),
                "batch/wobble": wobble.generate_wobble(e0, radius * 0.25, t_wobble)})
    # angle pairs whose shorter way round is direct, through 0 from below (left) and from above (right)
    a = torch.tensor([0.1, 3.0, 6.2, 0.1, -3.1, 3.1, 2.0, -0.5, 7.0, math.pi], dtype=torch.float64)
    b = torch.tensor([0.5, 3.2, 0.1, 6.2, 3.1, -3.1, -2.0, 0.5, -7.0, -math.pi], dtype=torch.float64)
    t = torch.linspace(-0.5, 1.5, 9, dtype=torch.float64)[:, None]
    out.update({"circular/a": a, "circular/b": b, "circular/t": t,
                "circular/result": interpolation.interpolate_circular(a, b, t)})
    OUT.parent.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(OUT, **{k: v.numpy() for k, v in out.items()})
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes, {len(CASES)} camera pairs)")


if __name__ == "__main__":
    main()
