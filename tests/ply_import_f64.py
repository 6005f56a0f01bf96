"""A float64 restatement of ps_ply_unpack (csrc/ply_import.cu) in numpy, and a writer of 3D Gaussian splatting PLY
files for the import tests.

`unpack_f64` reads the records by property name, as a 3DGS loader does, and computes every output in float64 from
the float32 record values and the float32 SH blocks the kernel's descriptor holds.  With each output it returns the
entry's magnitude: the sum of the absolute values of the terms that form it, which bounds the float64 rounding of the
sum."""
from __future__ import annotations

from pathlib import Path

import numpy as np

BLOCK_OFFSETS = (0, 1, 10, 35)


def write_ply(path: Path, names: list[str], records: np.ndarray, fmt: str = "binary_little_endian",
              extra_header: str = "") -> Path:
    """A PLY file of one vertex element of float properties `names`, holding float32 `records` [n, len(names)]."""
    header = (f"ply\nformat {fmt} 1.0\n{extra_header}element vertex {records.shape[0]}\n"
              + "".join(f"property float {n}\n" for n in names) + "end_header\n")
    Path(path).write_bytes(header.encode("ascii") + np.ascontiguousarray(records, dtype="<f4").tobytes())
    return Path(path)


def gs_properties(degree: int, normals: bool = True) -> list[str]:
    """3DGS's own property order for an SH degree."""
    rest = 3 * ((degree + 1) ** 2 - 1)
    return (["x", "y", "z"] + (["nx", "ny", "nz"] if normals else []) + [f"f_dc_{i}" for i in range(3)]
            + [f"f_rest_{i}" for i in range(rest)] + ["opacity"] + [f"scale_{i}" for i in range(3)]
            + [f"rot_{i}" for i in range(4)])


def blocks_of(sh_transform84: np.ndarray, degree: int) -> list[np.ndarray]:
    """The descriptor's 84 floats as the degree 0..`degree` blocks."""
    t = np.asarray(sh_transform84, dtype=np.float32).astype(np.float64)
    return [t[BLOCK_OFFSETS[l]:BLOCK_OFFSETS[l] + (2 * l + 1) ** 2].reshape(2 * l + 1, 2 * l + 1)
            for l in range(degree + 1)]


def quat_to_matrix(q: np.ndarray) -> np.ndarray:
    """wxyz [n, 4] -> [n, 3, 3], normalised; a zero quaternion is the identity."""
    q = q.astype(np.float64)
    n2 = (q * q).sum(-1)
    q = np.where(n2[:, None] > 0, q / np.sqrt(np.where(n2 > 0, n2, 1.0))[:, None], np.array([1.0, 0, 0, 0]))
    w, x, y, z = q.T
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def unpack_f64(records: np.ndarray, names: list[str], degree: int, sh_coeffs: int, blocks: list[np.ndarray],
               rotation=None, center=None, scale: float = 1.0) -> dict[str, tuple[np.ndarray, np.ndarray]]:
    """name -> (float64 value, float64 magnitude) for means [n, 3], covariances [n, 3, 3], harmonics
    [n, 3, sh_coeffs] and opacities [n]; the frame (rotation M, center c, scale s) is the identity when omitted."""
    col = {n: i for i, n in enumerate(names)}
    r = records.astype(np.float64)
    f = lambda name: r[:, col[name]]
    m = np.eye(3) if rotation is None else np.asarray(rotation, dtype=np.float64)
    c = np.zeros(3) if center is None else np.asarray(center, dtype=np.float64)
    s = float(scale)
    p = np.stack([f("x"), f("y"), f("z")], -1)
    means = p @ m * s + c
    means_mag = np.abs(p) @ np.abs(m) * s + np.abs(c)

    rot = quat_to_matrix(np.stack([f(f"rot_{i}") for i in range(4)], -1))
    var = np.exp(2 * np.stack([f(f"scale_{i}") for i in range(3)], -1)) * s * s
    b = np.swapaxes(rot, -1, -2) @ m                              # R^T M
    cov = np.einsum("nk,nki,nkj->nij", var, b, b)
    cov_mag = np.einsum("nk,nki,nkj->nij", var, np.abs(b), np.abs(b))

    nc = (degree + 1) ** 2
    coef = np.zeros((r.shape[0], 3, nc))
    for ch in range(3):
        coef[:, ch, 0] = f(f"f_dc_{ch}")
        for k in range(1, nc):
            coef[:, ch, k] = f(f"f_rest_{ch * (nc - 1) + k - 1}")
    harm = np.zeros((r.shape[0], 3, sh_coeffs))
    harm_mag = np.zeros_like(harm)
    for l, blk in enumerate(blocks[:degree + 1]):
        sl = slice(l * l, (l + 1) ** 2)
        harm[..., sl] = coef[..., sl] @ blk.T
        harm_mag[..., sl] = np.abs(coef[..., sl]) @ np.abs(blk).T
    opac = 1 / (1 + np.exp(-f("opacity")))
    return {"means": (means, means_mag), "covariances": (cov, cov_mag), "harmonics": (harm, harm_mag),
            "opacities": (opac, opac)}


def error_ratio(got: np.ndarray, want: np.ndarray, mag: np.ndarray) -> np.ndarray:
    """|got - want| in units of the kernel's own rounding allowance: half a float32 ulp of the value plus 64 float64
    roundings of the entry's magnitude.  An entry whose value and magnitude are 0 must be exactly 0."""
    unit = 0.5 * np.finfo(np.float32).eps * np.abs(want) + 64 * np.finfo(np.float64).eps * mag
    err = np.abs(got.astype(np.float64) - want)
    return np.where(unit > 0, err / np.where(unit > 0, unit, 1.0), np.where(err == 0, 0.0, np.inf))
