"""Test-time refinement of a 3D Gaussian splatting scene: Adam on the vertex records of a PLY file (or of
`ply_export.pack_viewer`), against a loss of renders of the scene's own views, as 3DGS optimises a scene.

The loss is the fused MSE over all views (`loss="mse"`, the default) or 3DGS's (1 - lambda) L1 + lambda D-SSIM
(`loss="l1_dssim"`, `loss.l1_dssim`, csrc/l1_dssim.cu), summed over the views: each view's gradient is then the one
3DGS's single-view step would give at that view.  Each step renders the views (with `render_views_mse`, or in colour
with `render_views` for L1 + D-SSIM; the unpacked Gaussians are the autograd leaves), then one kernel
(csrc/ply_import.cu, `ps_ply_refine_step`) differentiates the unpack, applies Adam with one learning rate per
property group and unpacks the updated records into the Gaussians the next step renders.  Records stay in the file's
layout throughout, so a refined file has the input's header and property order (with densification, a new vertex
count).

Learning rates are 3DGS's per-group rates.  The position rate is in the file's units: a viewer-format export
normalises the scene so that the 0.95 quantile of its centred means is 1 (`ply_export.export_frame`), which plays the
part of 3DGS's scene extent.  The position rate is constant unless `lr_xyz_final` is given; then it decays
exponentially from the xyz rate to `lr_xyz_final` over `lr_xyz_steps` steps, as 3DGS's schedule does (3DGS: 1.6e-6
over 30 000 steps).

With a `DensifyConfig`, the loop also runs 3DGS's adaptive density control (csrc/ply_densify.cu): each step before
`until_step` renders with a screen-space gradient holder and folds each view's projected-mean gradient norm into
per-Gaussian statistics; every `every` steps after `from_step` the records are cloned, split and pruned in 3DGS's
order, with the Adam moments carried along (zero for new rows); every `opacity_reset_every` steps the opacity logits
are clamped to logit(0.01).  The scene extent is 1 in a viewer-format export's units.  The gradient threshold is
3DGS's 2e-4, which was calibrated for its L1 + D-SSIM loss: with `loss="l1_dssim"` each view's statistic is the
quantity it was calibrated on; with the fused MSE over all context views the gradients are smaller, and the threshold
has not been tuned for that loss.

`refine_gaussians` refines one scene's encoder Gaussians in memory: the export, the refinement and the import that
`export-ply --write-frame`, `refine-ply` and `render-ply` chain through files, with the same bits.  `scene_report` and
`refine_report` build refine.json for both routes.
"""
from __future__ import annotations

import ctypes
import math
from dataclasses import asdict, dataclass
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
LOSSES = ("mse", "l1_dssim")


@dataclass
class RefineResult:
    """`records` float32 [n, P] on the device, in the input's layout; `loss` float32 [steps + 1] on the device: the
    loss before each step, and last the loss of the refined records (the context-view MSE, or with L1 + D-SSIM the
    mean per-view loss, the objective over the number of views); `exp_avg` and `exp_avg_sq` the Adam moments in the
    records' layout (None after no step)."""
    records: Tensor
    loss: Tensor
    exp_avg: Optional[Tensor] = None
    exp_avg_sq: Optional[Tensor] = None
    gaussians: Optional[list[int]] = None    # with densification: the record count at each entry of `loss`
    mse: Optional[Tensor] = None             # with L1 + D-SSIM: float32 [2], the context-view MSE before and after


@dataclass
class DensifyConfig:
    """3DGS's adaptive density control during refinement; the defaults are 3DGS's.  At step t (1-based):
    statistics are kept while t < until_step; clone / split / prune runs when from_step < t < until_step and
    t % every == 0; the opacity reset runs when opacity_reset_every > 0, t % opacity_reset_every == 0 and
    t < until_step; the world-size prune (max scale above 0.1 extent) is on once t > opacity_reset_every (with the
    reset on).  `extent` is the scene extent in the records' units; `seed` seeds the split copies' draws."""
    from_step: int = 500
    until_step: int = 15000
    every: int = 100
    grad_threshold: float = 2e-4
    percent_dense: float = 0.01
    min_opacity: float = 0.005
    opacity_reset_every: int = 3000
    extent: float = 1.0
    seed: int = 0

    def __post_init__(self):
        for k in ("from_step", "until_step", "every", "opacity_reset_every", "seed"):
            v = getattr(self, k)
            if isinstance(v, bool) or not isinstance(v, int) or v < (1 if k == "every" else 0):
                raise ValueError(f"DensifyConfig.{k} must be an int >= {1 if k == 'every' else 0}, got {v!r}")
        for k in ("grad_threshold", "percent_dense", "min_opacity", "extent"):
            v = getattr(self, k)
            if not (isinstance(v, (int, float)) and math.isfinite(v) and v >= 0) or (k == "extent" and v <= 0):
                raise ValueError(f"DensifyConfig.{k} must be a finite number {'> 0' if k == 'extent' else '>= 0'}, "
                                 f"got {v!r}")

    def stats_at(self, t: int) -> bool:
        return t < self.until_step

    def densifies_at(self, t: int) -> bool:
        return self.from_step < t < self.until_step and t % self.every == 0

    def resets_at(self, t: int) -> bool:
        return self.opacity_reset_every > 0 and t % self.opacity_reset_every == 0 and t < self.until_step

    def prunes_world_at(self, t: int) -> bool:
        return self.opacity_reset_every > 0 and t > self.opacity_reset_every


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
    number, the pointers and, when given, the rate of the position columns, and enqueues the kernel, with nothing
    read back from the device."""

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
        self.xyz_columns = [i for i, name in enumerate(properties) if group_of(name, sh_degree) == "xyz"]

    def __call__(self, records: Tensor, exp_avg: Tensor, exp_avg_sq: Tensor, grads, out, step: int, *,
                 records_out: Optional[Tensor] = None, d_records: Optional[Tensor] = None,
                 lr_xyz: Optional[float] = None) -> None:
        """Adam step number `step` (>= 1): `grads` (d_means [n, 3], d_covariances [n, 3, 3], d_harmonics
        [n, 3, C], d_opacities [n]) are the loss's gradients for `out` (a `Gaussians` of the same shapes, the unpack
        of `records`); `records_out` (default: `records`, in place) and the moments are updated, `out` receives the
        unpack of the updated records and `d_records`, when given, the records' gradient.  `lr_xyz`, when given,
        is the position columns' rate from this call on.  Every tensor is dense float32 on the records' device."""
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
        if lr_xyz is not None:
            for c in self.xyz_columns:
                d.lr[c] = lr_xyz
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


MAX_GAUSSIANS = 2 ** 31 - 1    # the rasterizer's int32 n_gaussians
OPACITY_RESET_LOGIT = math.log(0.01 / 0.99)


def _stream(dev) -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _dense(name: str, t: Tensor, shape, dtype, dev) -> None:
    if not isinstance(t, Tensor) or tuple(t.shape) != tuple(shape) or t.dtype != dtype or t.device != dev \
            or not t.is_contiguous():
        raise ValueError(f"densify: `{name}` must be a dense {str(dtype)[6:]} {list(shape)} tensor on {dev}")


def densify_stats(d_means2d: Tensor, radii: Tensor, accum: Tensor, count: Tensor) -> None:
    """`ps_ply_densify_stats`: for each view v where radii[v, i] > 0, accum[i] += |d_means2d[v, i, :2]| and
    count[i] += 1, in place.  d_means2d float32 [V, n, 3], radii int32 [V, n], accum float32 [n], count int32 [n]."""
    v, n = radii.shape
    dev = accum.device
    _dense("d_means2d", d_means2d, (v, n, 3), torch.float32, dev)
    _dense("radii", radii, (v, n), torch.int32, dev)
    _dense("accum", accum, (n,), torch.float32, dev)
    _dense("count", count, (n,), torch.int32, dev)
    with torch.cuda.device(dev):
        rc = _lib.lib.ps_ply_densify_stats(n, v, d_means2d.data_ptr(), radii.data_ptr(), accum.data_ptr(),
                                           count.data_ptr(), _stream(dev))
    _lib.check(rc, "ps_ply_densify_stats")


def densify_desc(properties, n: int, cfg: DensifyConfig, prune_world: bool) -> _lib.PlyDensifyDesc:
    col = {name: i for i, name in enumerate(properties)}
    need = ["x", "y", "z", "opacity"] + [f"scale_{k}" for k in range(3)] + [f"rot_{k}" for k in range(4)]
    missing = [k for k in need if k not in col]
    if missing:
        raise ValueError(f"densify: the records have no {', '.join(missing)} property")
    return _lib.PlyDensifyDesc(
        n_gaussians=n, n_props=len(properties), prune_world=int(prune_world),
        col_xyz=(ctypes.c_int32 * 3)(*(col[k] for k in "xyz")), col_opacity=col["opacity"],
        col_scale=(ctypes.c_int32 * 3)(*(col[f"scale_{k}"] for k in range(3))),
        col_rot=(ctypes.c_int32 * 4)(*(col[f"rot_{k}"] for k in range(4))),
        grad_threshold=cfg.grad_threshold, percent_dense=cfg.percent_dense, min_opacity=cfg.min_opacity,
        extent=cfg.extent)


def densify_workspace_bytes(n: int) -> int:
    out = ctypes.c_size_t()
    _lib.check(_lib.lib.ps_ply_densify_workspace_bytes(n, ctypes.byref(out)), "ps_ply_densify_workspace_bytes")
    return out.value


def densify_records(records: Tensor, exp_avg: Tensor, exp_avg_sq: Tensor, accum: Tensor, count: Tensor, properties,
                    cfg: DensifyConfig, *, prune_world: bool, eps: Tensor, out=None):
    """3DGS's clone / split / prune of `records` [n, P] with their Adam moments (`ps_ply_densify_count`, one read of
    the new count, then `ps_ply_densify_apply`), from the statistics accum [n] / count [n] and the split draws `eps`
    float32 [2, n, 3].  -> (records, exp_avg, exp_avg_sq) [n_new, P]: kept originals, clones, first and second split
    copies.  `out`, when given, is three float32 [>= n_new, P] tensors to write instead of new ones.  Raises
    ValueError, with nothing written, when n_new would be 0 or above the rasterizer's MAX_GAUSSIANS."""
    n, p = records.shape
    dev = records.device
    if not records.is_cuda:
        raise ValueError("densify: `records` must be a CUDA tensor (pixelsplat_b200 has no CPU path)")
    for name, t in (("records", records), ("exp_avg", exp_avg), ("exp_avg_sq", exp_avg_sq)):
        _dense(name, t, (n, p), torch.float32, dev)
    _dense("accum", accum, (n,), torch.float32, dev)
    _dense("count", count, (n,), torch.int32, dev)
    _dense("eps", eps, (2, n, 3), torch.float32, dev)
    desc = densify_desc(properties, n, cfg, prune_world)
    ws = torch.empty(densify_workspace_bytes(n), dtype=torch.uint8, device=dev)
    counts = torch.empty(4, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.lib.ps_ply_densify_count(ctypes.byref(desc), records.data_ptr(), accum.data_ptr(), count.data_ptr(),
                                           ws.data_ptr(), ws.numel(), counts.data_ptr(), _stream(dev))
    _lib.check(rc, "ps_ply_densify_count")
    n_new = int(counts[3].item())      # the one device-to-host synchronisation of a densification
    if n_new == 0:
        raise ValueError("densify: every Gaussian would be pruned; lower min_opacity or densify less often")
    if n_new > MAX_GAUSSIANS:
        raise ValueError(f"densify: {n_new} Gaussians are more than the rasterizer takes ({MAX_GAUSSIANS})")
    if out is None:
        out = [torch.empty((n_new, p), device=dev) for _ in range(3)]
    for name, t in zip(("records_out", "exp_avg_out", "exp_avg_sq_out"), out):
        if not isinstance(t, Tensor) or t.dim() != 2 or t.shape[0] < n_new or t.shape[1] != p \
                or t.dtype != torch.float32 or t.device != dev or not t.is_contiguous():
            raise ValueError(f"densify: `{name}` must be a dense float32 [>= {n_new}, {p}] tensor on {dev}")
    with torch.cuda.device(dev):
        rc = _lib.lib.ps_ply_densify_apply(ctypes.byref(desc), records.data_ptr(), exp_avg.data_ptr(),
                                           exp_avg_sq.data_ptr(), eps.data_ptr(), ws.data_ptr(), ws.numel(),
                                           counts.data_ptr(), *(t.data_ptr() for t in out), _stream(dev))
    _lib.check(rc, "ps_ply_densify_apply")
    return tuple(t[:n_new] for t in out)


def reset_opacity(records: Tensor, exp_avg: Tensor, exp_avg_sq: Tensor, properties) -> None:
    """3DGS's opacity reset, in place: o = min(o, logit(0.01)) and the opacity column's moments set to 0."""
    c = list(properties).index("opacity")
    records[:, c].clamp_(max=OPACITY_RESET_LOGIT)
    exp_avg[:, c] = 0.0
    exp_avg_sq[:, c] = 0.0


def refine_step(records: Tensor, properties, sh_degree: int, exp_avg: Tensor, exp_avg_sq: Tensor, grads, out,
                step: int, *, frame: Optional[ExportFrame] = None, lr: Optional[dict] = None,
                records_out: Optional[Tensor] = None, d_records: Optional[Tensor] = None,
                betas: tuple[float, float] = BETAS, eps: float = EPS) -> None:
    """One `ps_ply_refine_step` (`RefineStep`, built for this one call).  A loop of steps over the same records
    builds one `RefineStep` and calls it once per step."""
    step_fn = RefineStep(properties, sh_degree, records.shape[0], sh_coeffs=out.harmonics.shape[-1], frame=frame,
                         lr=lr, betas=betas, eps=eps)
    step_fn(records, exp_avg, exp_avg_sq, grads, out, step, records_out=records_out, d_records=d_records)


def xyz_lr_at(step: int, lr_xyz: float, lr_xyz_final: float, lr_xyz_steps: int) -> float:
    """The position rate at `step` (1-based) of 3DGS's exponential decay (get_expon_lr_func with no delay), in
    float64: exp((1 - u) ln lr_xyz + u ln lr_xyz_final), u = clip(step / lr_xyz_steps, 0, 1)."""
    u = min(max(step / lr_xyz_steps, 0.0), 1.0)
    return math.exp((1.0 - u) * math.log(lr_xyz) + u * math.log(lr_xyz_final))


def _check_schedule(lr: Optional[dict], lr_xyz_final, lr_xyz_steps) -> None:
    if lr_xyz_final is None:
        if lr_xyz_steps is not None:
            raise ValueError("refine_records: `lr_xyz_steps` needs `lr_xyz_final`")
        return
    if isinstance(lr_xyz_final, bool) or not isinstance(lr_xyz_final, (int, float)) \
            or not (math.isfinite(lr_xyz_final) and lr_xyz_final > 0):
        raise ValueError(f"refine_records: `lr_xyz_final` must be a finite number > 0, got {lr_xyz_final!r}")
    if not dict(DEFAULT_LR, **(lr or {}))["xyz"] > 0:
        raise ValueError("refine_records: the position rate decays only from an xyz rate > 0")
    if lr_xyz_steps is not None and (isinstance(lr_xyz_steps, bool) or not isinstance(lr_xyz_steps, int)
                                     or lr_xyz_steps < 1):
        raise ValueError(f"refine_records: `lr_xyz_steps` must be an int >= 1, got {lr_xyz_steps!r}")


def _check_options(steps, lr: Optional[dict], densify, loss, lambda_dssim, lr_xyz_final, lr_xyz_steps) -> None:
    """What `refine_records` refuses in its arguments, checked on the host before any launch."""
    if isinstance(steps, bool) or not isinstance(steps, int) or steps < 0:
        raise ValueError(f"refine_records: `steps` must be an int >= 0, got {steps!r}")
    column_lr((), 0, lr)
    if densify is not None and not isinstance(densify, DensifyConfig):
        raise ValueError(f"refine_records: `densify` must be a DensifyConfig or None, got {densify!r}")
    if loss not in LOSSES:
        raise ValueError(f"refine_records: `loss` must be one of {', '.join(LOSSES)}, got {loss!r}")
    if isinstance(lambda_dssim, bool) or not isinstance(lambda_dssim, (int, float)) or not 0 <= lambda_dssim <= 1:
        raise ValueError(f"refine_records: `lambda_dssim` must be a number in [0, 1], got {lambda_dssim!r}")
    _check_schedule(lr, lr_xyz_final, lr_xyz_steps)


def refine_records(records: Tensor, properties, sh_degree: int, *, frame: Optional[ExportFrame] = None,
                   extrinsics: Tensor, intrinsics: Tensor, near: Tensor, far: Tensor, images: Tensor,
                   background_color: Tensor, steps: int, lr: Optional[dict] = None,
                   densify: Optional[DensifyConfig] = None, loss: str = "mse", lambda_dssim: float = 0.2,
                   lr_xyz_final: Optional[float] = None, lr_xyz_steps: Optional[int] = None) -> RefineResult:
    """`steps` Adam steps on `records` (float32 [n, P] on a CUDA device, from `ply_import.read_ply_body` or
    `ply_export.pack_viewer`, with `properties`) against a loss of renders of the views (extrinsics [v, 4, 4],
    intrinsics [v, 3, 3], near / far [v], images [v, 3, h, w], background_color [3]) in the world of `frame`.
    `loss` is "mse" (the fused MSE over the views) or "l1_dssim" (the sum over the views of 3DGS's
    (1 - lambda_dssim) L1 + lambda_dssim D-SSIM; the result's `mse` then holds the context MSE before and after).
    `lr` maps groups (GROUPS) to learning rates over DEFAULT_LR.  With `lr_xyz_final`, the position rate at step t is
    `xyz_lr_at(t, lr["xyz"], lr_xyz_final, lr_xyz_steps or steps)`.  With `densify`, 3DGS's densification, pruning
    and opacity reset run after each step's Adam update as the config schedules them, and the result's `gaussians`
    holds the count at each loss entry.  The input is not modified; with steps=0 it is returned as it is."""
    from .decoder import Gaussians
    from .decoder.cuda_splatting import render_views, render_views_means2d, render_views_mse, render_views_mse_means2d
    from .loss import l1_dssim
    from .ply_import import unpack_records
    properties = list(properties)
    _check_options(steps, lr, densify, loss, lambda_dssim, lr_xyz_final, lr_xyz_steps)
    lr_xyz = dict(DEFAULT_LR, **(lr or {}))["xyz"]
    decay_steps = steps if lr_xyz_steps is None else lr_xyz_steps
    dev = records.device
    v, _, h, w = images.shape
    views = [t.to(dev, torch.float32)[None] for t in (extrinsics, intrinsics, near, far)]
    target = images.to(dev, torch.float32)[None]
    background = background_color.to(dev, torch.float32).reshape(1, 1, 3).expand(1, v, 3)
    n, coeffs = records.shape[0], (sh_degree + 1) ** 2

    def gaussians_for(count: int):
        leaves = [torch.empty((1, count, 3), device=dev), torch.empty((1, count, 3, 3), device=dev),
                  torch.empty((1, count, 3, coeffs), device=dev), torch.empty((1, count), device=dev)]
        return leaves, Gaussians(*(t[0] for t in leaves))

    leaves, out = gaussians_for(n)
    work = records if steps == 0 else records.clone().contiguous()
    unpack_records(work, properties, sh_degree, frame=frame, out=out)
    losses = torch.empty(steps + 1, device=dev)
    denom = float(v * 3 * h * w)

    def mse() -> Tensor:
        sse, _, _ = render_views_mse(*views, (h, w), background, *leaves, target=target, want_color=False)
        return sse.sum() / denom

    def photometric(means2d: Optional[Tensor] = None):
        """The L1 + D-SSIM objective (the sum over the views) and, with the holder `means2d`, the radii."""
        if means2d is None:
            color, radii = render_views(*views, (h, w), background, *leaves), None
        else:
            color, radii = render_views_means2d(*views, (h, w), background, *leaves, means2d=means2d)
        return l1_dssim(color[0], target[0], lambda_dssim).sum(), radii

    dssim = loss == "l1_dssim"
    mse_before = None
    if dssim:
        with torch.no_grad():
            mse_before = mse()
    m = v2 = None
    counts = None if densify is None else [n]
    if steps:
        m, v2 = torch.zeros_like(work), torch.zeros_like(work)
        step_fn = RefineStep(properties, sh_degree, n, sh_coeffs=coeffs, frame=frame, lr=lr)
        for leaf in leaves:
            leaf.requires_grad_(True)
        if densify is not None:
            accum = torch.zeros(n, device=dev)
            seen = torch.zeros(n, dtype=torch.int32, device=dev)
            draws = torch.Generator(dev).manual_seed(densify.seed)
        for t in range(1, steps + 1):
            if densify is not None and densify.stats_at(t):
                means2d = torch.zeros((v, n, 3), device=dev, requires_grad=True)
                if dssim:
                    value, radii = photometric(means2d)
                else:
                    sse, _, _, radii = render_views_mse_means2d(*views, (h, w), background, *leaves, target=target,
                                                                means2d=means2d, want_color=False)
                    value = sse.sum() / denom
                value.backward()
                densify_stats(means2d.grad, radii, accum, seen)
            else:
                value = photometric()[0] if dssim else mse()
                value.backward()
            losses[t - 1] = value.detach() / v if dssim else value.detach()
            grads = [leaf.grad[0].contiguous() for leaf in leaves]
            for leaf in leaves:
                leaf.grad = None
            step_fn(work, m, v2, grads, out, t,
                    lr_xyz=None if lr_xyz_final is None else xyz_lr_at(t, lr_xyz, lr_xyz_final, decay_steps))
            if densify is None:
                continue
            if densify.densifies_at(t):
                eps = torch.randn((2, n, 3), device=dev, generator=draws)
                work, m, v2 = densify_records(work, m, v2, accum, seen, properties, densify,
                                              prune_world=densify.prunes_world_at(t), eps=eps)
                n = work.shape[0]
                accum, seen = torch.zeros(n, device=dev), torch.zeros(n, dtype=torch.int32, device=dev)
                leaves, out = gaussians_for(n)
                step_fn = RefineStep(properties, sh_degree, n, sh_coeffs=coeffs, frame=frame, lr=lr)
            if densify.resets_at(t):
                reset_opacity(work, m, v2, properties)
            if densify.densifies_at(t) or densify.resets_at(t):
                unpack_records(work, properties, sh_degree, frame=frame, out=out)
                for leaf in leaves:
                    leaf.requires_grad_(True)
            counts.append(n)
    with torch.no_grad():
        if dssim:
            losses[steps] = photometric()[0] / v
            mse_after = mse_before if steps == 0 else mse()
            return RefineResult(work, losses, m, v2, counts, torch.stack([mse_before, mse_after]))
        losses[steps] = mse()
    return RefineResult(work, losses, m, v2, counts)


OPTIONS = ("lr", "densify", "loss", "lambda_dssim", "lr_xyz_final", "lr_xyz_steps")   # refine_records' options


def check_refine_options(steps, **options) -> None:
    """Refuses, on the host, what `refine_records` would refuse in `steps` and its `options` (OPTIONS), and any
    other option."""
    unknown = sorted(set(options) - set(OPTIONS))
    if unknown:
        raise ValueError(f"refine: unknown option {', '.join(unknown)}; the options are {', '.join(OPTIONS)}")
    _check_options(steps, options.get("lr"), options.get("densify"), options.get("loss", "mse"),
                   options.get("lambda_dssim", 0.2), options.get("lr_xyz_final"), options.get("lr_xyz_steps"))


def refine_gaussians(gaussians, extrinsics: Tensor, *, context_extrinsics: Tensor, intrinsics: Tensor, near: Tensor,
                     far: Tensor, images: Tensor, background_color: Tensor, steps: int, **options):
    """One scene's Gaussians as the encoder returns them (batch 1), refined in memory as `export-ply --write-frame`,
    `refine-ply` and `render-ply` refine and load them from files: `ply_export.pack_viewer` at its default degree
    with context view 0's pose `extrinsics` [4, 4], `refine_records` in the world of
    `ply_export.export_frame(means, extrinsics)` against the context views (context_extrinsics [v, 4, 4],
    intrinsics [v, 3, 3], near / far [v], images [v, 3, h, w]), and `ply_import.unpack_records` with the file's
    (d + 1)^2 coefficients.  `options` are refine_records' (OPTIONS).  -> (batch-1 `Gaussians` for the decoder,
    the `RefineResult`); with steps=0, the export round trip alone and the context loss once.  Runs with autograd
    on whatever the caller's grad mode; refuses bad arguments before any launch."""
    from .decoder import Gaussians
    from .ply_export import export_frame, pack_viewer
    from .ply_import import unpack_records
    check_refine_options(steps, **options)
    means = getattr(gaussians, "means", None)
    if not isinstance(means, Tensor) or means.dim() != 3 or means.shape[0] != 1:
        shape = list(means.shape) if isinstance(means, Tensor) else None
        raise ValueError(f"refine_gaussians: `gaussians` must hold one scene with a batch dimension of 1 (means "
                         f"[1, n, 3]), got means of shape {shape}")
    records, properties = pack_viewer(gaussians, extrinsics)
    frame = export_frame(means[0], extrinsics)
    sh_degree = math.isqrt(sum(p.startswith("f_rest_") for p in properties) // 3 + 1) - 1
    with torch.enable_grad():
        result = refine_records(records, properties, sh_degree, frame=frame, extrinsics=context_extrinsics,
                                intrinsics=intrinsics, near=near, far=far, images=images,
                                background_color=background_color, steps=steps, **options)
    g = unpack_records(result.records, properties, sh_degree, frame=frame)
    return Gaussians(*(t[None] for t in (g.means, g.covariances, g.harmonics, g.opacities))), result


def scene_report(result: RefineResult, steps: int, loss: str = "mse",
                 densify: Optional[DensifyConfig] = None) -> dict:
    """One scene's entry of refine.json: the context MSE before and after and the steps; with L1 + D-SSIM also the
    mean per-view loss before and after (the MSE then comes from the result's `mse`); with densification the
    Gaussian count before and after (the records' count when the result kept no counts)."""
    history = result.loss.tolist()
    if loss == "mse":
        out = {"mse_before": history[0], "mse_after": history[-1], "steps": steps}
    else:
        mse = result.mse.tolist()
        out = {"mse_before": mse[0], "mse_after": mse[-1], "steps": steps, "loss_before": history[0],
               "loss_after": history[-1]}
    if densify is not None:
        before, after = (result.gaussians[0], result.gaussians[-1]) if result.gaussians else \
            (result.records.shape[0],) * 2
        out.update(gaussians_before=before, gaussians_after=after)
    return out


def refine_report(scenes: dict, steps: int, lr: Optional[dict] = None, densify: Optional[DensifyConfig] = None,
                  loss: str = "mse", lambda_dssim: float = 0.2, lr_xyz_final: Optional[float] = None,
                  lr_xyz_steps: Optional[int] = None) -> dict:
    """refine.json: the settings (every group's rate) and each scene's entry (`scene_report`); the densification,
    the loss and the decay are recorded only when not off."""
    out = {"steps": steps, "lr": dict(DEFAULT_LR, **(lr or {})), "scenes": scenes}
    if densify is not None:
        out["densify"] = asdict(densify)
    if loss != "mse":
        out.update(loss=loss, lambda_dssim=lambda_dssim)
    if lr_xyz_final is not None:
        out.update(lr_xyz_final=lr_xyz_final, lr_xyz_steps=steps if lr_xyz_steps is None else lr_xyz_steps)
    return out


def rewrite_vertex_count(head: bytes, count: int) -> bytes:
    """The header bytes `head` (up to and including end_header) with the `element vertex N` line's N set to `count`;
    every other byte is kept."""
    start = head.index(b"\nelement vertex ") + len(b"\nelement vertex ")
    end = head.index(b"\n", start)
    return head[:start] + str(count).encode() + head[end:]


def refine_ply(path: Union[Path, str], frame: Union[ExportFrame, Path, str, None], *, extrinsics: Tensor,
               intrinsics: Tensor, near: Tensor, far: Tensor, images: Tensor, background_color: Tensor, steps: int,
               out_path: Union[Path, str], lr: Optional[dict] = None, device=None,
               densify: Optional[DensifyConfig] = None, loss: str = "mse", lambda_dssim: float = 0.2,
               lr_xyz_final: Optional[float] = None, lr_xyz_steps: Optional[int] = None) -> Optional[RefineResult]:
    """`refine_records` on the file at `path` (in the world of `frame`: an `ExportFrame`, a `<scene>.frame.json`
    path, or None for the file's own frame), written to `out_path` as the input's header bytes followed by the
    refined records: property order, extra properties and comments are kept, and only the `element vertex` count
    changes when densification changed it.  With steps=0 the input's bytes are written as they are, without any
    device work, and the result is None."""
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
                            background_color=background_color, steps=steps, lr=lr, densify=densify, loss=loss,
                            lambda_dssim=lambda_dssim, lr_xyz_final=lr_xyz_final, lr_xyz_steps=lr_xyz_steps)
    body = result.records.cpu().numpy().astype("<f4", copy=False).tobytes()
    header = head[:layout.body_offset]
    if result.records.shape[0] != layout.count:
        header = rewrite_vertex_count(header, result.records.shape[0])
    out_path.write_bytes(header + body)
    return result
