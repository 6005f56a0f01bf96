"""Shared by oracle/make_ply_golden.py and the PLY export tests: the seeded inputs of the reference-format fixture
(regenerated on both sides from tests/golden_util.py; only the reference's outputs are stored) and a reader of the
binary PLY files the exporter writes."""
from __future__ import annotations

from pathlib import Path

import numpy as np
import torch

from tests import golden_util as gu

# (name, camera rotation, Gaussian count): an identity and a general view-0 rotation, odd and even counts, counts
# below, at and off a multiple of the kernel's 64-Gaussian CTA
PLY_CASES = (("identity", False, 1000), ("general", True, 777), ("general_one_cta", True, 64),
             ("identity_tail", False, 129))


def ply_case(name: str) -> dict:
    """Float32 CPU inputs of export_ply for PLY_CASES[name]: extrinsics [4, 4] (camera-to-world), means, scales,
    rotations (xyzw, not normalised), harmonics [n, 3, 25], opacities."""
    _, rotated, n = next(c for c in PLY_CASES if c[0] == name)
    ext = torch.eye(4, dtype=torch.float64)
    if rotated:
        ext[:3, :3] = gu.rotation(0.3, -0.5, 1.1)
        ext[:3, 3] = torch.tensor([0.4, -1.2, 2.5], dtype=torch.float64)
    p = f"ply.{name}."
    means = gu.seeded_like(p + "means", (n, 3), 2.0) + torch.tensor([0.3, -1.0, 4.0], dtype=torch.float64)
    return dict(extrinsics=ext.float(), means=means.float(),
                scales=(gu.seeded_like(p + "scales", (n, 3), 1.0) - 4.0).exp().float(),
                rotations=gu.seeded_like(p + "rotations", (n, 4), 1.0).float(),
                harmonics=gu.seeded_like(p + "harmonics", (n, 3, 25), 1.0).float(),
                opacities=gu.seeded_like(p + "opacities", (n,), 2.0).sigmoid().float())


def read_ply(path: Path) -> tuple[list[str], np.ndarray]:
    """(property names, float32 [count, len(names)]) of a binary little-endian PLY file holding one vertex element
    of float properties, checking the header line by line."""
    data = Path(path).read_bytes()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    lines = data[:end].decode("ascii").splitlines()
    assert lines[:2] == ["ply", "format binary_little_endian 1.0"], lines[:2]
    kind, element, count = lines[2].split()
    assert (kind, element) == ("element", "vertex"), lines[2]
    names = []
    for line in lines[3:-1]:
        prop, typ, name = line.split()
        assert (prop, typ) == ("property", "float"), line
        names.append(name)
    assert lines[-1] == "end_header"
    body = np.frombuffer(data[end:], dtype="<f4")
    assert body.size == int(count) * len(names), (body.size, count, len(names))
    return names, body.reshape(int(count), len(names))
