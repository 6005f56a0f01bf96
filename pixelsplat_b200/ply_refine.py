"""Test-time refinement of a 3D Gaussian splatting scene: Adam on the vertex records of a PLY file (or of
`ply_export.pack_viewer`), against the fused-MSE loss of renders of the scene's own views, as 3DGS optimises a scene.

Each step renders the views with `render_views_mse` (the unpacked Gaussians are the autograd leaves), then one kernel
(csrc/ply_import.cu, `ps_ply_refine_step`) differentiates the unpack, applies Adam with one learning rate per
property group and unpacks the updated records into the Gaussians the next step renders.  Records stay in the file's
layout throughout, so a refined file has the input's header and property order.

Learning rates are 3DGS's per-group rates.  The position rate is in the file's units: a viewer-format export
normalises the scene so that the 0.95 quantile of its centred means is 1 (`ply_export.export_frame`), which plays the
part of 3DGS's scene extent.  The position rate is constant; there is no densification, pruning or opacity reset.
"""
from __future__ import annotations

import ctypes
import math
from dataclasses import dataclass
from pathlib import Path
from typing import Optional, Union

import torch
from torch import Tensor

from . import _lib
from .ply_export import ExportFrame
from .ply_import import _MAX_HEADER_BYTES, import_desc, parse_header, read_frame_json, read_ply_body

GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scale", "rot")
DEFAULT_LR = {"xyz": 0.00016, "f_dc": 0.0025, "f_rest": 0.0025 / 20, "opacity": 0.05, "scale": 0.005, "rot": 0.001}
BETAS = (0.9, 0.999)
EPS = 1e-15          # 3DGS's Adam eps


@dataclass
class RefineResult:
    """`records` float32 [n, P] on the device, in the input's layout; `loss` float32 [steps + 1] on the device: the
    context-view MSE before each step, and last the MSE of the refined records; `exp_avg` and `exp_avg_sq` the
    Adam moments in the records' layout (None after no step)."""
    records: Tensor
    loss: Tensor
    exp_avg: Optional[Tensor] = None
    exp_avg_sq: Optional[Tensor] = None


def group_of(name: str, sh_degree: int) -> Optional[str]:
    """The property group a column belongs to, or None for a column the unpack does not read."""
    if name in ("x", "y", "z"):
        return "xyz"
    if name in ("f_dc_0", "f_dc_1", "f_dc_2"):
        return "f_dc"
    if name.startswith("f_rest_") and name[7:].isdigit() and int(name[7:]) < 3 * ((sh_degree + 1) ** 2 - 1):
        return "f_rest"
    if name == "opacity":
        return "opacity"
    if name in ("scale_0", "scale_1", "scale_2"):
        return "scale"
    if name in ("rot_0", "rot_1", "rot_2", "rot_3"):
        return "rot"
    return None


def column_lr(properties, sh_degree: int, lr: Optional[dict] = None) -> list[float]:
    """Per column: the learning rate of its group (`lr` over DEFAULT_LR), 0 for a column the unpack does not read."""
    rates = dict(DEFAULT_LR)
    for k, v in (lr or {}).items():
        if k not in rates:
            raise ValueError(f"unknown learning-rate group {k!r}; the groups are {', '.join(GROUPS)}")
        if not (isinstance(v, (int, float)) and math.isfinite(v) and v >= 0):
            raise ValueError(f"learning rate of {k!r} must be a finite number >= 0, got {v!r}")
        rates[k] = float(v)
    groups = [group_of(p, sh_degree) for p in properties]
    return [0.0 if g is None else rates[g] for g in groups]


class RefineStep:
    """`ps_ply_refine_step` for the records of one scene: n records with `properties`, SH degree `sh_degree`,
    Gaussians of `sh_coeffs` coefficients per channel, `frame`, learning rates `lr` (groups over DEFAULT_LR).  The
    descriptor (columns, frame, SH blocks, per-column rates) is built once, here; each call only sets the step
    number and the pointers and enqueues the kernel, with nothing read back from the device."""

    def __init__(self, properties, sh_degree: int, n: int, *, sh_coeffs: Optional[int] = None,
                 frame: Optional[ExportFrame] = None, lr: Optional[dict] = None,
                 betas: tuple[float, float] = BETAS, eps: float = EPS):
        properties = list(properties)
        p = len(properties)
        if p > _lib.PLY_REFINE_MAX_PROPERTIES:
            raise ValueError(f"refine_step: {p} properties; at most {_lib.PLY_REFINE_MAX_PROPERTIES} can be refined")
        self.n, self.p = n, p
        self.coeffs = (sh_degree + 1) ** 2 if sh_coeffs is None else sh_coeffs
        self.desc = _lib.PlyRefineDesc(unpack=import_desc(properties, sh_degree, self.coeffs, n, frame),
                                       beta1=betas[0], beta2=betas[1], eps=eps)
        self.desc.lr[:p] = column_lr(properties, sh_degree, lr)

    def __call__(self, records: Tensor, exp_avg: Tensor, exp_avg_sq: Tensor, grads, out, step: int, *,
                 records_out: Optional[Tensor] = None, d_records: Optional[Tensor] = None) -> None:
        """Adam step number `step` (>= 1): `grads` (d_means [n, 3], d_covariances [n, 3, 3], d_harmonics
        [n, 3, C], d_opacities [n]) are the loss's gradients for `out` (a `Gaussians` of the same shapes, the unpack
        of `records`); `records_out` (default: `records`, in place) and the moments are updated, `out` receives the
        unpack of the updated records and `d_records`, when given, the records' gradient.  Every tensor is dense
        float32 on the records' device."""
        n, p, c, dev = self.n, self.p, self.coeffs, records.device
        if not isinstance(records, Tensor) or not records.is_cuda:
            raise ValueError("refine_step: `records` must be a CUDA tensor (pixelsplat_b200 has no CPU path)")
        records_out = records if records_out is None else records_out
        d_means, d_covariances, d_harmonics, d_opacities = grads
        checked = [("records", records, (n, p)), ("records_out", records_out, (n, p)), ("exp_avg", exp_avg, (n, p)),
                   ("exp_avg_sq", exp_avg_sq, (n, p)), ("d_records", d_records, (n, p)),
                   ("d_means", d_means, (n, 3)), ("d_covariances", d_covariances, (n, 3, 3)),
                   ("d_harmonics", d_harmonics, (n, 3, c)), ("d_opacities", d_opacities, (n,))] + \
            [(f"out.{k}", getattr(out, k), shape) for k, shape in (("means", (n, 3)), ("covariances", (n, 3, 3)),
                                                                   ("harmonics", (n, 3, c)), ("opacities", (n,)))]
        for name, t, shape in checked:
            if t is None and name == "d_records":
                continue
            if not isinstance(t, Tensor) or t.shape != shape or t.dtype != torch.float32 or t.device != dev \
                    or not t.is_contiguous():
                raise ValueError(f"refine_step: `{name}` must be a dense float32 {list(shape)} tensor on {dev}")
        d = self.desc
        d.step = step
        d.unpack.records = records.data_ptr()
        for name in ("means", "covariances", "harmonics", "opacities"):
            setattr(d.unpack, name, getattr(out, name).data_ptr())
        d.records_out, d.exp_avg, d.exp_avg_sq = records_out.data_ptr(), exp_avg.data_ptr(), exp_avg_sq.data_ptr()
        d.d_records = None if d_records is None else d_records.data_ptr()
        d.d_means, d.d_covariances = d_means.data_ptr(), d_covariances.data_ptr()
        d.d_harmonics, d.d_opacities = d_harmonics.data_ptr(), d_opacities.data_ptr()
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            rc = _lib.lib.ps_ply_refine_step(ctypes.byref(d), ctypes.c_void_p(stream.cuda_stream))
        _lib.check(rc, "ps_ply_refine_step")


def refine_step(records: Tensor, properties, sh_degree: int, exp_avg: Tensor, exp_avg_sq: Tensor, grads, out,
                step: int, *, frame: Optional[ExportFrame] = None, lr: Optional[dict] = None,
                records_out: Optional[Tensor] = None, d_records: Optional[Tensor] = None,
                betas: tuple[float, float] = BETAS, eps: float = EPS) -> None:
    """One `ps_ply_refine_step` (`RefineStep`, built for this one call).  A loop of steps over the same records
    builds one `RefineStep` and calls it once per step."""
    step_fn = RefineStep(properties, sh_degree, records.shape[0], sh_coeffs=out.harmonics.shape[-1], frame=frame,
                         lr=lr, betas=betas, eps=eps)
    step_fn(records, exp_avg, exp_avg_sq, grads, out, step, records_out=records_out, d_records=d_records)


def refine_records(records: Tensor, properties, sh_degree: int, *, frame: Optional[ExportFrame] = None,
                   extrinsics: Tensor, intrinsics: Tensor, near: Tensor, far: Tensor, images: Tensor,
                   background_color: Tensor, steps: int, lr: Optional[dict] = None) -> RefineResult:
    """`steps` Adam steps on `records` (float32 [n, P] on a CUDA device, from `ply_import.read_ply_body` or
    `ply_export.pack_viewer`, with `properties`) against the MSE of renders of the views (extrinsics [v, 4, 4],
    intrinsics [v, 3, 3], near / far [v], images [v, 3, h, w], background_color [3]) in the world of `frame`.
    `lr` maps groups (GROUPS) to learning rates over DEFAULT_LR.  The input is not modified; with steps=0 it is
    returned as it is."""
    from .decoder import Gaussians
    from .decoder.cuda_splatting import render_views_mse
    from .ply_import import unpack_records
    properties = list(properties)
    if isinstance(steps, bool) or not isinstance(steps, int) or steps < 0:
        raise ValueError(f"refine_records: `steps` must be an int >= 0, got {steps!r}")
    column_lr(properties, sh_degree, lr)
    dev = records.device
    v, _, h, w = images.shape
    views = [t.to(dev, torch.float32)[None] for t in (extrinsics, intrinsics, near, far)]
    target = images.to(dev, torch.float32)[None]
    background = background_color.to(dev, torch.float32).reshape(1, 1, 3).expand(1, v, 3)
    n, coeffs = records.shape[0], (sh_degree + 1) ** 2
    leaves = [torch.empty((1, n, 3), device=dev), torch.empty((1, n, 3, 3), device=dev),
              torch.empty((1, n, 3, coeffs), device=dev), torch.empty((1, n), device=dev)]
    out = Gaussians(*(t[0] for t in leaves))
    work = records if steps == 0 else records.clone().contiguous()
    unpack_records(work, properties, sh_degree, frame=frame, out=out)
    loss = torch.empty(steps + 1, device=dev)
    denom = float(v * 3 * h * w)

    def mse() -> Tensor:
        sse, _, _ = render_views_mse(*views, (h, w), background, *leaves, target=target, want_color=False)
        return sse.sum() / denom

    m = v2 = None
    if steps:
        m, v2 = torch.zeros_like(work), torch.zeros_like(work)
        step_fn = RefineStep(properties, sh_degree, n, sh_coeffs=coeffs, frame=frame, lr=lr)
        for leaf in leaves:
            leaf.requires_grad_(True)
        for t in range(1, steps + 1):
            value = mse()
            value.backward()
            loss[t - 1] = value.detach()
            grads = [leaf.grad[0].contiguous() for leaf in leaves]
            for leaf in leaves:
                leaf.grad = None
            step_fn(work, m, v2, grads, out, t)
    with torch.no_grad():
        loss[steps] = mse()
    return RefineResult(work, loss, m, v2)


def refine_ply(path: Union[Path, str], frame: Union[ExportFrame, Path, str, None], *, extrinsics: Tensor,
               intrinsics: Tensor, near: Tensor, far: Tensor, images: Tensor, background_color: Tensor, steps: int,
               out_path: Union[Path, str], lr: Optional[dict] = None, device=None) -> Optional[RefineResult]:
    """`refine_records` on the file at `path` (in the world of `frame`: an `ExportFrame`, a `<scene>.frame.json`
    path, or None for the file's own frame), written to `out_path` as the input's header bytes, unchanged, followed
    by the refined records: property order, extra properties and comments are kept.  With steps=0 the input's
    bytes are written as they are, without any device work, and the result is None."""
    path, out_path = Path(path), Path(out_path)
    with open(path, "rb") as f:
        head = f.read(_MAX_HEADER_BYTES)
    layout = parse_header(head, str(path))
    out_path.parent.mkdir(parents=True, exist_ok=True)
    if steps == 0:
        out_path.write_bytes(path.read_bytes())
        return None
    device = images.device if device is None else torch.device(device)
    if isinstance(frame, (str, Path)):
        frame = read_frame_json(frame, device)
    _, records = read_ply_body(path, device)
    result = refine_records(records, layout.properties, layout.sh_degree, frame=frame, extrinsics=extrinsics,
                            intrinsics=intrinsics, near=near, far=far, images=images,
                            background_color=background_color, steps=steps, lr=lr)
    body = result.records.cpu().numpy().astype("<f4", copy=False).tobytes()
    out_path.write_bytes(head[:layout.body_offset] + body)
    return result
