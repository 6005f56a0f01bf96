"""Seeded synthetic camera trajectories for the evaluation-index generator (oracle/make_index_golden.py, its tests
and tools/bench_index.py): OpenCV-style camera-to-world matrices (x right, y down, z forward) and normalised
intrinsics, float32, each family chosen to reach one part of the reference's walk.

  dolly       forward motion with a slow yaw wobble: the overlap stays high, walks end on distance
  pan         sideways motion while the camera yaws 0.45 degrees a frame: walks end on overlap
  rotate      rotation in place about a tilted axis: every pair shares its centre (project_rays' at-camera branch)
  repeated    runs of 12 identical poses along a yawing path (at-camera pairs inside a run)
  nonsquare   anisotropic, off-centre intrinsics on a yawing, climbing path
  short       fewer frames than the default min_distance (45)
  none        a fast yaw in place: frames min_distance apart or more are 32 degrees or more apart, so no pair overlaps enough
"""
from __future__ import annotations

import numpy as np

FAMILIES = ("dolly", "pan", "rotate", "repeated", "nonsquare", "short", "none")
LENGTHS = {"dolly": 200, "pan": 250, "rotate": 300, "repeated": 180, "nonsquare": 220, "short": 30, "none": 150}
# (name, image h, w, generator config overrides)
CONFIGS = (("default", 256, 256, {}), ("small", 64, 64, {"min_distance": 2, "max_distance": 6}))


def _rot(axis, angle: float) -> np.ndarray:
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    k = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle) * k + (1 - np.cos(angle)) * k @ k


def trajectory(family: str, seed: int = 0, frames: int | None = None) -> tuple[np.ndarray, np.ndarray]:
    """(extrinsics [v, 4, 4] c2w, intrinsics [v, 3, 3]) float32 of one family."""
    rng = np.random.default_rng([FAMILIES.index(family), seed])
    v = LENGTHS[family] if frames is None else frames
    deg = np.pi / 180
    base = _rot(rng.normal(size=3), 0.3)                      # a random, fixed world orientation
    # rotations in place sit at the world origin, where the pose inverse returns an exact zero translation: the
    # reference's at-camera test (|origin| < 1e-6 in float32) is then far from its threshold
    origin = np.zeros(3) if family in ("rotate", "none") else rng.normal(size=3)
    R, t = [], []
    for i in range(v):
        if family == "dolly":
            r = _rot([0, 1, 0], 4 * deg * np.sin(i / 17))
            p = np.array([0.0, 0.0, 0.05 * i])
        elif family in ("pan", "short"):
            r = _rot([0, 1, 0], 0.45 * deg * i)
            p = np.array([0.03 * i, 0.0, 0.0])
        elif family == "rotate":
            r = _rot([0.2, 1, 0.1], 0.3 * deg * i)
            p = np.zeros(3)
        elif family == "repeated":
            j = i // 12
            r = _rot([0, 1, 0], 1.2 * deg * j)
            p = np.array([0.1 * j, 0.0, 0.05 * j])
        elif family == "nonsquare":
            r = _rot([0.1, 1, 0], 0.35 * deg * i)
            p = np.array([0.02 * i, -0.01 * i, 0.01 * i])
        else:                                                 # none: 2.2 degrees a frame, no full turn in 150
            r = _rot([0, 1, 0], 2.2 * deg * i)
            p = np.zeros(3)
        R.append(base @ r)
        t.append(origin + base @ p)
    E = np.tile(np.eye(4), (v, 1, 1))
    E[:, :3, :3] = np.stack(R)
    E[:, :3, 3] = np.stack(t)
    K = np.tile(np.eye(3), (v, 1, 1))
    if family == "nonsquare":
        K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2] = 1.1, 0.7, 0.47, 0.53
    else:
        K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2] = 0.86, 0.86, 0.5, 0.5
    return E.astype(np.float32), K.astype(np.float32)
