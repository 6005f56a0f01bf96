"""PLY export of one scene's Gaussians, in the 3D Gaussian splatting layout that splat viewers read.

Two formats, one kernel (csrc/ply_export.cu, `ps_ply_pack`) that writes the vertex records on the device:

* `export_ply` is the reference's `src/model/ply_export.py` with the same signature and output: the camera-frame
  quaternions composed with the export frame, the DC band only and the raw opacity.
* `export_gaussians_ply` writes what the rasterizer renders.  Each Gaussian's scale and rotation come from its
  covariance in the export frame; the opacity is stored as a logit, as viewers apply a sigmoid; the harmonics up to
  degree 3 are rotated into the export frame in the 3DGS basis.  Degree 4 is dropped: the format has no slot for it.

Both centre the scene on the median of the means and divide by s, the largest per-axis 0.95 quantile of the centred
means' absolute values.  Both rotate into the reference's frame M = Rz(-45 deg) [[0,0,1],[-1,0,0],[0,-1,0]] R_c2w^-1,
with R_c2w the rotation of the context view 0 camera.  Median and s are computed on the device and the kernel reads
them there, so nothing is read back before the records.  The file is an ASCII header followed by the records,
written in one call from a pinned host buffer.
"""
from __future__ import annotations

import ctypes
import json
import math
from dataclasses import dataclass
from pathlib import Path
from typing import Union

import torch
from torch import Tensor

from . import _lib
from .sh import convention_id, sh_rotation_matrices, sh_signs

MAX_SH_DEGREE = 3   # f_rest_0..44: the most a 3D Gaussian splatting PLY holds
_BLOCK_OFFSETS = (0, 1, 10, 35)   # of the degree-0..3 blocks in ps_ply_desc.sh_transform
_OPENGL_UP = ((0.0, 0.0, 1.0), (-1.0, 0.0, 0.0), (0.0, -1.0, 0.0))   # makes +z the world up vector


def ply_properties(sh_degree: int | None) -> list[str]:
    """The vertex properties in file order: the reference's order, with f_rest_* after f_dc_* when `sh_degree` is
    given (viewer format; degree 0 has none).  `None` is the reference format."""
    rest = 0 if sh_degree is None else 3 * ((min(sh_degree, MAX_SH_DEGREE) + 1) ** 2 - 1)
    return (["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(rest)]
            + ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"])


def ply_header(properties: list[str], count: int) -> bytes:
    return ("ply\nformat binary_little_endian 1.0\n" + f"element vertex {count}\n"
            + "".join(f"property float {p}\n" for p in properties) + "end_header\n").encode("ascii")


def reference_frame(extrinsics: Tensor) -> Tensor:
    """M as the reference's export_ply forms it: float32 products on the host, R_c2w inverted in float32."""
    c = math.cos(math.pi / 4)
    adjustment = torch.tensor([[c, c, 0.0], [-c, c, 0.0], [0.0, 0.0, 1.0]], dtype=torch.float32)
    rotation = adjustment @ torch.tensor(_OPENGL_UP, dtype=torch.float32)
    return rotation @ extrinsics.detach().cpu().float()[:3, :3].inverse()


def viewer_frame(extrinsics: Tensor) -> Tensor:
    """M in float64 [3, 3]: what the viewer format rotates positions, covariances and harmonics with."""
    c = math.cos(math.pi / 4)
    adjustment = torch.tensor([[c, c, 0.0], [-c, c, 0.0], [0.0, 0.0, 1.0]], dtype=torch.float64)
    return adjustment @ torch.tensor(_OPENGL_UP, dtype=torch.float64) @ \
        extrinsics.detach().cpu().double()[:3, :3].inverse()


def sh_transform(frame: Tensor, degree: int, basis) -> Tensor:
    """float64 [n, n], n = (degree + 1)^2: coefficients c in the rasterizer basis `basis` ("3dgs" or "e3nn") to
    coefficients c' in the 3DGS basis of the frame `frame` maps world directions to:
        sum_i c'_i Y_3dgs,i(M d) = sum_i c_i Y_basis,i(d)   for every direction d.
    Block diagonal (a rotation never mixes degrees)."""
    rotate = sh_rotation_matrices(frame.double()[None], degree, "3dgs")[0]
    if convention_id(basis) == 0:
        return rotate
    # Y_e3nn(d) = S Y_3dgs(P d) with P d = (z, x, y), so e3nn coefficients c are 3DGS coefficients D(P)^T S c
    perm = torch.tensor([[0.0, 0.0, 1.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]], dtype=torch.float64)
    to_3dgs = sh_rotation_matrices(perm[None], degree, "3dgs")[0].T * sh_signs(degree)[None, :]
    return rotate @ to_3dgs


def normalisation(means: Tensor) -> tuple[Tensor, Tensor]:
    """(median of the means [3], s [1]) on the means' device, as the reference computes them.  The median is the
    lower-interpolated 0.5 quantile: the element torch.median(dim=0) returns, NaN propagation included, without
    its indices, which CUDA cannot compute under torch.use_deterministic_algorithms."""
    center = means.quantile(0.5, dim=0, interpolation="lower")
    scale = (means - center).abs().quantile(0.95, dim=0).max().reshape(1)
    return center.contiguous(), scale


@dataclass(frozen=True)
class ExportFrame:
    """The map from the world to a viewer-format file: x = M (p - c) / s.  `center` c (float32 [3]) and `scale` s
    (float32 [1], a zero 0.95 quantile replaced by 1) stay on the means' device; `rotation` M is float64 [3, 3] on
    the host."""
    center: Tensor
    scale: Tensor
    rotation: Tensor

    def to_json(self) -> dict:
        """c, s and M as JSON numbers: the float32 values of c and s are exact in a double, so a reader gets the bits
        the kernel used."""
        return {"center": [float(v) for v in self.center.cpu()], "scale": float(self.scale.cpu()[0]),
                "rotation": [[float(v) for v in row] for row in self.rotation]}


def export_frame(means: Tensor, extrinsics: Tensor) -> ExportFrame:
    """The frame `export_gaussians_ply` writes one scene's Gaussians in: the median of `means` [n, 3], s and
    M = viewer_frame(extrinsics)."""
    center, scale = normalisation(means)
    return ExportFrame(center, torch.where(scale > 0, scale, torch.ones_like(scale)), viewer_frame(extrinsics))


def write_frame_json(frame: ExportFrame, path: Union[Path, str]) -> None:
    path = Path(path)
    path.parent.mkdir(exist_ok=True, parents=True)
    path.write_text(json.dumps(frame.to_json(), indent=1) + "\n")


def _check(fn: str, name: str, t, shape: tuple, device=None) -> Tensor:
    """`t` a CUDA float32 tensor of `shape` (None = any size), on `device` when given."""
    if not isinstance(t, Tensor):
        raise ValueError(f"{fn}: `{name}` must be a torch.Tensor, got {type(t).__name__}")
    if not t.is_cuda:
        raise ValueError(f"{fn}: `{name}` must be a CUDA tensor (pixelsplat_b200 has no CPU path)")
    if t.dtype != torch.float32:
        raise ValueError(f"{fn}: `{name}` must be float32, got {t.dtype}")
    if t.dim() != len(shape) or any(w is not None and s != w for s, w in zip(t.shape, shape)):
        want = "[" + ", ".join("*" if w is None else str(w) for w in shape) + "]"
        raise ValueError(f"{fn}: `{name}` has shape {list(t.shape)}, expected {want}")
    if device is not None and t.device != device:
        raise ValueError(f"{fn}: `{name}` is on {t.device}, the means on {device}")
    return t.detach().contiguous()


def _check_harmonics(fn: str, harmonics: Tensor, n: int, device) -> tuple[Tensor, int]:
    h = _check(fn, "harmonics", harmonics, (n, 3, None), device)
    degree = math.isqrt(h.shape[-1]) - 1
    if h.shape[-1] < 1 or (degree + 1) ** 2 != h.shape[-1] or degree > 4:
        raise ValueError(f"{fn}: `harmonics` has {h.shape[-1]} coefficients per channel, expected (degree + 1)^2 "
                         "with a degree of 0 to 4")
    return h, degree


def _pack(desc: _lib.PlyDesc, device, count: int, floats: int, tensors: dict) -> Tensor:
    out = torch.empty((count, floats), dtype=torch.float32, device=device)
    for name, t in tensors.items():
        setattr(desc, name, t.data_ptr())
    desc.n_gaussians = count
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device)
        rc = _lib.lib.ps_ply_pack(ctypes.byref(desc), ctypes.c_void_p(out.data_ptr()),
                                  ctypes.c_void_p(stream.cuda_stream))
    _lib.check(rc, "ps_ply_pack")
    return out


def pack_reference(extrinsics: Tensor, means: Tensor, scales: Tensor, rotations: Tensor, harmonics: Tensor,
                   opacities: Tensor) -> tuple[Tensor, list[str]]:
    """The device half of `export_ply`: (records float32 [n, 17] on the means' device, property names)."""
    fn = "export_ply"
    means = _check(fn, "means", means, (None, 3))
    n, dev = means.shape[0], means.device
    if n < 1:
        raise ValueError(f"{fn}: `means` holds no Gaussian")
    _check(fn, "extrinsics", extrinsics, (4, 4), dev)
    t = dict(means=means, scales=_check(fn, "scales", scales, (n, 3), dev),
             rotations=_check(fn, "rotations", rotations, (n, 4), dev),
             harmonics=_check_harmonics(fn, harmonics, n, dev)[0],
             opacities=_check(fn, "opacities", opacities, (n,), dev))
    t["center"], t["scale"] = normalisation(means)
    desc = _lib.PlyDesc(mode=_lib.PS_PLY_REFERENCE, sh_degree=0, sh_coeffs=t["harmonics"].shape[-1])
    desc.frame[:] = [float(v) for v in reference_frame(extrinsics).double().reshape(-1)]
    names = ply_properties(None)
    return _pack(desc, dev, n, len(names), t), names


def pack_viewer(gaussians, extrinsics: Tensor, sh_degree: int = MAX_SH_DEGREE) -> tuple[Tensor, list[str]]:
    """The device half of `export_gaussians_ply`: (records float32 [n, 17 + 3 ((d + 1)^2 - 1)], property names),
    d = min(sh_degree, 3, the harmonics' degree)."""
    from .rasterizer import get_sh_basis
    fn = "export_gaussians_ply"
    fields = {k: getattr(gaussians, k, None) for k in ("means", "covariances", "harmonics", "opacities")}
    means = fields["means"]
    if isinstance(means, Tensor) and means.dim() == 3:
        if means.shape[0] != 1:
            raise ValueError(f"{fn}: `gaussians` holds a batch of {means.shape[0]} scenes; pass one scene "
                             "(batch 1, or one batch element)")
        fields = {k: v[0] if isinstance(v, Tensor) else v for k, v in fields.items()}
    means = _check(fn, "gaussians.means", fields["means"], (None, 3))
    n, dev = means.shape[0], means.device
    if n < 1:
        raise ValueError(f"{fn}: `gaussians` holds no Gaussian")
    _check(fn, "extrinsics", extrinsics, (4, 4), dev)
    if isinstance(sh_degree, bool) or not isinstance(sh_degree, int) or sh_degree < 0:
        raise ValueError(f"{fn}: `sh_degree` must be a non-negative int, got {sh_degree!r}")
    harmonics, have = _check_harmonics(fn, fields["harmonics"], n, dev)
    t = dict(means=means, covariances=_check(fn, "gaussians.covariances", fields["covariances"], (n, 3, 3), dev),
             harmonics=harmonics, opacities=_check(fn, "gaussians.opacities", fields["opacities"], (n,), dev))
    frame = export_frame(means, extrinsics)
    t["center"], t["scale"] = frame.center, frame.scale
    degree = min(sh_degree, MAX_SH_DEGREE, have)
    transform = sh_transform(frame.rotation, degree, get_sh_basis())
    desc = _lib.PlyDesc(mode=_lib.PS_PLY_VIEWER, sh_degree=degree, sh_coeffs=harmonics.shape[-1])
    desc.frame[:] = [float(v) for v in frame.rotation.reshape(-1)]
    for l in range(degree + 1):
        block = transform[l * l:(l + 1) ** 2, l * l:(l + 1) ** 2].reshape(-1)
        desc.sh_transform[_BLOCK_OFFSETS[l]:_BLOCK_OFFSETS[l] + block.numel()] = [float(v) for v in block]
    names = ply_properties(degree)
    return _pack(desc, dev, n, len(names), t), names


_pinned: list[Tensor] = []


def write_ply(path: Union[Path, str], properties: list[str], records: Tensor) -> None:
    """The header, then `records` (float32 [n, len(properties)] on a CUDA device) copied through a pinned host buffer
    and written in one call."""
    path = Path(path)
    count = records.numel()
    if not _pinned or _pinned[0].numel() < count:
        _pinned[:] = [torch.empty(max(count, 1), dtype=torch.float32, pin_memory=True)]
    host = _pinned[0][:count]
    with torch.cuda.device(records.device):
        host.copy_(records.reshape(-1), non_blocking=True)
        torch.cuda.current_stream(records.device).synchronize()
    path.parent.mkdir(exist_ok=True, parents=True)
    with open(path, "wb") as f:
        f.write(ply_header(properties, records.shape[0]))
        f.write(memoryview(host.numpy()))


def export_ply(extrinsics: Tensor, means: Tensor, scales: Tensor, rotations: Tensor, harmonics: Tensor,
               opacities: Tensor, path: Union[Path, str]) -> None:
    """The reference's export_ply: extrinsics [4, 4] (camera-to-world of context view 0), means [n, 3], scales
    [n, 3], rotations [n, 4] (xyzw, the adapter's camera-frame quaternions), harmonics [n, 3, d_sh], opacities [n],
    all CUDA float32.  Writes the reference's 17 properties: the DC band, the raw opacity and log(scale / s)."""
    records, properties = pack_reference(extrinsics, means, scales, rotations, harmonics, opacities)
    write_ply(path, properties, records)


def export_gaussians_ply(gaussians, extrinsics: Tensor, path: Union[Path, str], *,
                         sh_degree: int = MAX_SH_DEGREE) -> None:
    """What the rasterizer renders, as a splat viewer reads it.  `gaussians`: one scene's `Gaussians` (means [n, 3],
    covariances [n, 3, 3], harmonics [n, 3, d_sh], opacities [n], with or without a batch dimension of 1);
    `extrinsics` [4, 4]: context view 0's camera-to-world.  Writes f_dc and f_rest up to degree
    min(sh_degree, 3, the harmonics' degree), in the 3DGS basis whichever basis the rasterizer evaluates
    (`rasterizer.set_sh_basis`), the opacity as a logit and scale / rotation from each covariance."""
    records, properties = pack_viewer(gaussians, extrinsics, sh_degree)
    write_ply(path, properties, records)
