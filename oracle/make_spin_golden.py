"""Generates tests/golden/spin_trajectory_v1.npz by running the REFERENCE's generate_spin
(src/visualization/camera_trajectory/spin.py) on the CPU.  Authoring container only:

    python oracle/make_spin_golden.py

TEST INFRASTRUCTURE.  The module needs torch, einops, jaxtyping and scipy only; everything run here is the
reference's own code.  Stored per case `<case>/`: num_frames, elevation, radius and extrinsics (float32
[num_frames, 4, 4]).
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
REFERENCE = Path("/root/reference")
OUT = ROOT / "tests" / "golden" / "spin_trajectory_v1.npz"

# (num_frames, elevation in degrees, radius): the reference's test_splatter spin, one frame, odd counts, negative
# and steep elevations, small and fractional radii
CASES = {"test_splatter": (60, 0.0, 10.0), "one_frame": (1, 15.0, 2.0), "odd": (7, 30.0, 1.5),
         "below": (13, -25.0, 3.25), "steep": (90, 80.0, 0.75), "long": (300, 20.0, 2.0)}


def main() -> None:
    if str(REFERENCE) not in sys.path:
        sys.path.insert(0, str(REFERENCE))
    from src.visualization.camera_trajectory.spin import generate_spin
    out = {}
    for name, (n, elevation, radius) in CASES.items():
        out.update({f"{name}/num_frames": np.int64(n), f"{name}/elevation": np.float64(elevation),
                    f"{name}/radius": np.float64(radius),
                    f"{name}/extrinsics": generate_spin(n, torch.device("cpu"), elevation, radius).numpy()})
    OUT.parent.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes, {len(CASES)} cases)")


if __name__ == "__main__":
    main()
