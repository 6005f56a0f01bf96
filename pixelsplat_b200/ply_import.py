"""PLY import: a 3D Gaussian splatting PLY file as one scene's Gaussians, ready for `DecoderSplattingCUDA.forward`
and `render_views`.  The inverse of `ply_export.export_gaussians_ply`.

The header is parsed here, on the host; the body goes unchanged through a pinned buffer to the device, where one
kernel (csrc/ply_import.cu, `ps_ply_unpack`) turns the records into means, full covariances, harmonics in the
rasterizer's SH basis and sigmoid opacities.

Accepted: a binary little-endian file with one `vertex` element of float properties holding x y z, f_dc_0..2,
f_rest_0..3((d+1)^2-1)-1 for a degree d of 0 to 3, opacity (a logit), scale_0..2 (log scales) and rot_0..3 (a wxyz
quaternion, normalised here; a zero quaternion is the identity rotation).  Properties may come in any order and any
other float property (normals, other pipelines' fields) is ignored.

Not accepted as render input: the reference format (`export_ply`, `export-ply --format reference`).  Its header
cannot be told apart from a degree-0 file of this format, but its opacity is raw rather than a logit and its
rotations are the reference's camera-frame quaternions, so it would load without an error and render wrongly.

`frame` (an `ply_export.ExportFrame`, or the path of the JSON file `export-ply --write-frame` writes) maps the file
back into the world it was exported from: p = M^T x s + c, Sigma = s^2 M^T Sigma_file M, and the harmonics through
the inverse of the exporter's SH matrix.  Without it, the file's frame is the world.
"""
from __future__ import annotations

import ctypes
import json
import os
from dataclasses import dataclass
from pathlib import Path
from typing import Optional, Union

import torch
from torch import Tensor

from . import _lib
from .ply_export import _BLOCK_OFFSETS, MAX_SH_DEGREE, ExportFrame, sh_transform

REQUIRED = ("x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2", "opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1",
            "rot_2", "rot_3")
_MAX_HEADER_BYTES = 1 << 20


class PlyFormatError(ValueError):
    """A file this importer cannot read, with what is wrong with it."""


@dataclass(frozen=True)
class PlyLayout:
    """What the header says: the vertex count, the property names in file order, the SH degree and where the body
    starts."""
    count: int
    properties: tuple[str, ...]
    sh_degree: int
    body_offset: int


def parse_header(header: bytes, path: str = "<ply>") -> PlyLayout:
    """The layout of a file whose bytes start with `header` (at least up to and including `end_header\\n`)."""
    end = header.find(b"end_header\n")
    if not header.startswith(b"ply\n") and not header.startswith(b"ply\r\n"):
        raise PlyFormatError(f"{path}: not a PLY file (it does not start with 'ply')")
    if end < 0:
        raise PlyFormatError(f"{path}: no 'end_header' line in the first {_MAX_HEADER_BYTES} bytes")
    try:
        lines = header[:end].decode("ascii").splitlines()[1:]
    except UnicodeDecodeError as e:
        raise PlyFormatError(f"{path}: the header is not ASCII") from e
    fmt, elements, names = None, [], []
    for line in lines:
        words = line.split()
        if not words or words[0] in ("comment", "obj_info"):
            continue
        if words[0] == "format":
            fmt = " ".join(words[1:])
            if words[1:2] != ["binary_little_endian"]:
                raise PlyFormatError(f"{path}: format {fmt!r} is not supported; only binary_little_endian files "
                                     "can be imported")
        elif words[0] == "element":
            if len(words) != 3 or not words[2].isdigit():
                raise PlyFormatError(f"{path}: malformed element line {line!r}")
            elements.append((words[1], int(words[2])))
        elif words[0] == "property":
            if not elements:
                raise PlyFormatError(f"{path}: property before any element: {line!r}")
            if len(words) != 3 or words[1] not in ("float", "float32"):
                raise PlyFormatError(f"{path}: property {words[-1]!r} of element {elements[-1][0]!r} is "
                                     f"'{' '.join(words[1:-1])}'; only float properties are supported")
            names.append(words[2])
        else:
            raise PlyFormatError(f"{path}: unknown header line {line!r}")
    if fmt is None:
        raise PlyFormatError(f"{path}: no format line")
    if [e for e, _ in elements] != ["vertex"]:
        raise PlyFormatError(f"{path}: elements {[e for e, _ in elements]}; expected exactly one 'vertex' element")
    count = elements[0][1]
    if count < 1:
        raise PlyFormatError(f"{path}: the vertex element has a count of 0")
    if len(set(names)) != len(names):
        raise PlyFormatError(f"{path}: a property appears twice")
    missing = [n for n in REQUIRED if n not in names]
    if missing:
        raise PlyFormatError(f"{path}: missing required properties {missing}")
    rest = sum(n.startswith("f_rest_") for n in names)
    degree = next((d for d in range(MAX_SH_DEGREE + 1) if 3 * ((d + 1) ** 2 - 1) == rest), None)
    if degree is None:
        raise PlyFormatError(f"{path}: {rest} f_rest properties; expected 3 ((d + 1)^2 - 1) = 0, 9, 24 or 45 "
                             "for an SH degree d of 0 to 3")
    absent = [f"f_rest_{i}" for i in range(rest) if f"f_rest_{i}" not in names]
    if absent:
        raise PlyFormatError(f"{path}: the f_rest properties are not f_rest_0..{rest - 1} (no {absent[0]})")
    if len(names) > _lib.PLY_IMPORT_MAX_PROPERTIES:
        raise PlyFormatError(f"{path}: {len(names)} properties; at most {_lib.PLY_IMPORT_MAX_PROPERTIES} "
                             "are supported")
    return PlyLayout(count, tuple(names), degree, end + len(b"end_header\n"))


def read_frame_json(path: Union[Path, str], device=None) -> ExportFrame:
    """The frame `export-ply --write-frame` wrote: c and s as float32 on `device`, M float64 on the host."""
    d = json.loads(Path(path).read_text())
    device = _device(device)
    return ExportFrame(torch.tensor(d["center"], dtype=torch.float32, device=device),
                       torch.tensor([d["scale"]], dtype=torch.float32, device=device),
                       torch.tensor(d["rotation"], dtype=torch.float64))


def import_sh_blocks(rotation: Optional[Tensor], degree: int, basis) -> list[Tensor]:
    """float64 blocks of degree 0..`degree`: file coefficients (3DGS basis, the frame `rotation` maps the world to;
    the world itself when None) to coefficients in the rasterizer basis `basis`.  Each is the inverse of the block
    of `ply_export.sh_transform`, the exporter's matrix."""
    m = torch.eye(3, dtype=torch.float64) if rotation is None else rotation.double().cpu()
    t = sh_transform(m, degree, basis)
    return [torch.linalg.inv(t[l * l:(l + 1) ** 2, l * l:(l + 1) ** 2]) for l in range(degree + 1)]


def _device(device) -> torch.device:
    return torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)


def unpack_records(records: Tensor, properties, sh_degree: int, *, frame: Optional[ExportFrame] = None,
                   sh_coeffs: Optional[int] = None, out=None):
    """The device half of `load_gaussians_ply`: `records` float32 [n, P] on a CUDA device, the file's vertex
    records with `properties` (P names) -> `Gaussians` of one scene, without a batch dimension.  `out`, a
    `Gaussians` of dense float32 tensors ([n, 3], [n, 3, 3], [n, 3, sh_coeffs], [n]), receives the result instead
    of new tensors."""
    from .decoder import Gaussians
    fn = "unpack_records"
    properties = list(properties)
    if not isinstance(records, Tensor) or not records.is_cuda or records.dtype != torch.float32 or \
            records.dim() != 2 or records.shape[1] != len(properties):
        raise ValueError(f"{fn}: `records` must be a CUDA float32 [n, {len(properties)}] tensor")
    n, dev = records.shape[0], records.device
    nc = (sh_degree + 1) ** 2
    coeffs = nc if sh_coeffs is None else sh_coeffs
    if isinstance(coeffs, bool) or not isinstance(coeffs, int) or not nc <= coeffs <= _lib.PLY_IMPORT_MAX_COEFFS:
        raise ValueError(f"{fn}: `sh_coeffs` must be an int in [{nc}, {_lib.PLY_IMPORT_MAX_COEFFS}] for a degree-"
                         f"{sh_degree} file, got {sh_coeffs!r}")
    if out is None:
        out = Gaussians(torch.empty((n, 3), device=dev), torch.empty((n, 3, 3), device=dev),
                        torch.empty((n, 3, coeffs), device=dev), torch.empty((n,), device=dev))
    shapes = dict(means=(n, 3), covariances=(n, 3, 3), harmonics=(n, 3, coeffs), opacities=(n,))
    for name, shape in shapes.items():
        t = getattr(out, name)
        if t.shape != shape or t.dtype != torch.float32 or t.device != dev or not t.is_contiguous():
            raise ValueError(f"{fn}: `out.{name}` must be a dense float32 {list(shape)} tensor on {dev}")
    records = records.contiguous()
    desc = import_desc(properties, sh_degree, coeffs, n, frame)
    desc.records = records.data_ptr()
    for name in shapes:
        setattr(desc, name, getattr(out, name).data_ptr())
    _launch(desc, dev)
    return out


def import_desc(properties, sh_degree: int, sh_coeffs: int, n: int,
                frame: Optional[ExportFrame] = None) -> _lib.PlyImportDesc:
    """The descriptor of `ps_ply_unpack` for records with `properties`, without its pointers: columns, frame and
    the import SH blocks of the rasterizer's basis."""
    from .rasterizer import get_sh_basis
    nc = (sh_degree + 1) ** 2
    col = {p: i for i, p in enumerate(properties)}
    desc = _lib.PlyImportDesc(sh_degree=sh_degree, sh_coeffs=sh_coeffs, n_props=len(properties), n_gaussians=n)
    desc.col_xyz[:] = [col[k] for k in ("x", "y", "z")]
    desc.col_dc[:] = [col[f"f_dc_{c}"] for c in range(3)]
    for i in range(3 * (nc - 1)):
        desc.col_rest[i] = col[f"f_rest_{i}"]
    desc.col_opacity = col["opacity"]
    desc.col_scale[:] = [col[f"scale_{k}"] for k in range(3)]
    desc.col_rot[:] = [col[f"rot_{k}"] for k in range(4)]
    if frame is None:
        desc.frame[:] = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]
        desc.center[:], desc.scale = [0.0, 0.0, 0.0], 1.0
    else:
        desc.frame[:] = [float(v) for v in frame.rotation.double().reshape(-1)]
        desc.center[:] = [float(v) for v in frame.center.cpu()]
        desc.scale = float(frame.scale.reshape(-1)[0])
    blocks = import_sh_blocks(None if frame is None else frame.rotation, sh_degree, get_sh_basis())
    for l, block in enumerate(blocks):
        desc.sh_transform[_BLOCK_OFFSETS[l]:_BLOCK_OFFSETS[l] + block.numel()] = [float(v) for v in block.reshape(-1)]
    return desc


def _launch(desc: _lib.PlyImportDesc, device) -> None:
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device)
        rc = _lib.lib.ps_ply_unpack(ctypes.byref(desc), ctypes.c_void_p(stream.cuda_stream))
    _lib.check(rc, "ps_ply_unpack")


_pinned: list[Tensor] = []       # the host buffer every body goes through, kept between calls
_pinned_free: list = []          # the event after which its last copy has left it


def read_ply_body(path: Union[Path, str], device=None) -> tuple[PlyLayout, Tensor]:
    """(layout, records float32 [count, P] on `device`): the header parsed, the body read into the pinned buffer
    and copied to the device without waiting for the copy."""
    path = Path(path)
    device = _device(device)
    with open(path, "rb") as f:
        layout = parse_header(f.read(_MAX_HEADER_BYTES), str(path))
        p = len(layout.properties)
        want = layout.count * p * 4
        have = os.fstat(f.fileno()).st_size - layout.body_offset
        if have != want:
            raise PlyFormatError(f"{path}: the body holds {have} bytes; {layout.count} vertices of {p} floats "
                                 f"need {want}")
        count = layout.count * p
        if _pinned_free:
            _pinned_free[0].synchronize()
        if not _pinned or _pinned[0].numel() < count:
            _pinned[:] = [torch.empty(count, dtype=torch.float32, pin_memory=True)]
        host = _pinned[0][:count]
        f.seek(layout.body_offset)
        view = memoryview(host.numpy()).cast("B")
        got = f.readinto(view)
        if got != want:
            raise PlyFormatError(f"{path}: read {got} of the body's {want} bytes")
    with torch.cuda.device(device):
        records = host.to(device, non_blocking=True).reshape(layout.count, p)
        event = torch.cuda.Event()
        event.record(torch.cuda.current_stream(device))
    _pinned_free[:] = [event]
    return layout, records


def load_gaussians_ply(path: Union[Path, str], device=None, *, frame: Union[ExportFrame, Path, str, None] = None,
                       sh_coeffs: Optional[int] = None):
    """A 3D Gaussian splatting PLY file as `Gaussians` of batch 1 on `device` (default: the current CUDA device):
    means [1, n, 3], covariances [1, n, 3, 3], harmonics [1, n, 3, sh_coeffs] in the rasterizer's SH basis
    (`rasterizer.set_sh_basis`), zero above the file's degree, and opacities [1, n].  `sh_coeffs` defaults to the
    file's (d + 1)^2; 16 or 25 pad the harmonics for a degree-3 or degree-4 rasterizer.

    `frame`: the export frame (an `ExportFrame`, or a `<scene>.frame.json` path) to map the file back into the
    world of the scene it was exported from; None keeps the file's frame.  Files in the reference's format are not
    supported (module docstring).  Raises `PlyFormatError` on a file it cannot read."""
    from .decoder import Gaussians
    device = _device(device)
    if isinstance(frame, (str, Path)):
        frame = read_frame_json(frame, device)
    layout, records = read_ply_body(path, device)
    g = unpack_records(records, layout.properties, layout.sh_degree, frame=frame, sh_coeffs=sh_coeffs)
    return Gaussians(*(t[None] for t in (g.means, g.covariances, g.harmonics, g.opacities)))
