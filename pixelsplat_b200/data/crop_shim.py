"""The reference's crop shim (src/dataset/shims/crop_shim.py) on the GPU.

The reference resizes every view on the host: float -> uint8 -> PIL `Image.resize(..., Image.LANCZOS)` -> / 255,
then centre-crops and rescales fx, fy.  Here one launch of csrc/image_resample.cu does the flip, the resample, the
crop and the conversion for a whole batch of uint8 views, with Pillow's result bit for bit: the kernel runs
Pillow's integer passes on coefficient tables this module builds on the host, in float64 with libm's `sin`
(`math.sin`), exactly as Pillow's `precompute_coeffs` / `normalize_coeffs_8bpc` do.

- `rescale_and_crop_u8` takes decoded uint8 views [..., h, w, 3] (what the data loader yields) and the flip flags.
- `rescale`, `center_crop`, `rescale_and_crop` and `apply_crop_shim` are drop-ins for the reference's functions on
  float CUDA tensors.
- `device_shim` is the one call after the DataLoader of `DatasetRE10k`: it returns the reference's batch layout.
CPU tensors raise ValueError: there is no host path.
"""
from __future__ import annotations

import functools
import math

import numpy as np
import torch
from torch import Tensor

PRECISION_BITS = 22
LANCZOS_SUPPORT = 3.0


def _sinc(x: float) -> float:
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x: float) -> float:
    if -LANCZOS_SUPPORT <= x < LANCZOS_SUPPORT:
        return _sinc(x) * _sinc(x / LANCZOS_SUPPORT)
    return 0.0


@functools.lru_cache(maxsize=None)
def resample_table(in_size: int, out_size: int, offset: int = 0, length: int | None = None
                   ) -> tuple[np.ndarray, np.ndarray]:
    """Pillow's LANCZOS coefficients for resizing an axis of `in_size` pixels to `out_size`, for output pixels
    [offset, offset + length) (the crop): bounds int32 [length, 2] (first input pixel, count) and weights int32
    [length, taps] (22 fraction bits, zero past a window's count).  An axis that keeps its size, which Pillow does
    not resample, gets the identity (one tap of 2^22).  Read-only arrays, cached per argument tuple."""
    length = out_size - offset if length is None else length
    if not (1 <= out_size <= in_size and 0 <= offset and length >= 1 and offset + length <= out_size):
        raise ValueError(f"resample_table: bad sizes in {in_size}, out {out_size}, crop [{offset}, +{length})")
    if out_size == in_size:
        bounds = np.stack([np.arange(offset, offset + length), np.ones(length, np.int64)], 1).astype(np.int32)
        weights = np.full((length, 1), 1 << PRECISION_BITS, np.int32)
    else:
        scale = in_size / out_size
        filterscale = max(scale, 1.0)
        support = LANCZOS_SUPPORT * filterscale
        ss = 1.0 / filterscale
        rows = []
        for xx in range(offset, offset + length):
            center = (xx + 0.5) * scale
            xmin = max(int(center - support + 0.5), 0)          # int() truncates toward zero, as C's cast
            xmax = min(int(center + support + 0.5), in_size) - xmin
            k = [_lanczos((x + xmin - center + 0.5) * ss) for x in range(xmax)]
            ww = 0.0
            for w in k:                                         # in order: Python's sum() is compensated
                ww += w
            if ww != 0.0:
                k = [w / ww for w in k]
            fixed = [int(-0.5 + w * (1 << PRECISION_BITS)) if w < 0 else int(0.5 + w * (1 << PRECISION_BITS))
                     for w in k]
            rows.append((xmin, fixed))
        taps = max(len(f) for _, f in rows)
        bounds = np.array([(xmin, len(f)) for xmin, f in rows], np.int32)
        weights = np.zeros((length, taps), np.int32)
        for i, (_, f) in enumerate(rows):
            weights[i, :len(f)] = f
    bounds.setflags(write=False)
    weights.setflags(write=False)
    return bounds, weights


_DEVICE_TABLES: dict = {}


def _device_table(in_size: int, out_size: int, offset: int, length: int, device: torch.device):
    """resample_table on `device`, uploaded once (so later calls, and a graph capture, copy nothing)."""
    key = (in_size, out_size, offset, length, str(device))
    t = _DEVICE_TABLES.get(key)
    if t is None:
        b, w = resample_table(in_size, out_size, offset, length)
        t = (torch.from_numpy(b.copy()).to(device), torch.from_numpy(w.copy()).to(device))
        _DEVICE_TABLES[key] = t
    return t


def scaled_shape(h_in: int, w_in: int, shape: tuple[int, int]) -> tuple[int, int]:
    """The reference's rescale_and_crop sizes: scale by the larger ratio (rounded), so one axis matches `shape`."""
    h_out, w_out = shape
    if not (h_out <= h_in and w_out <= w_in):
        raise ValueError(f"crop shim: output {shape} is larger than the input {(h_in, w_in)}")
    scale_factor = max(h_out / h_in, w_out / w_in)
    h_scaled, w_scaled = round(h_in * scale_factor), round(w_in * scale_factor)
    if not (h_scaled == h_out or w_scaled == w_out):
        raise ValueError(f"crop shim: scaled size {(h_scaled, w_scaled)} matches neither side of {shape}")
    return h_scaled, w_scaled


def _check_cuda(what: str, *tensors: Tensor) -> None:
    for t in tensors:
        if not t.is_cuda:
            raise ValueError(f"{what}: expected CUDA tensors, got one on {t.device}; there is no CPU path")


def resample_u8(images: Tensor, scaled: tuple[int, int], crop: tuple[int, int, int, int],
                flip: Tensor | None = None) -> Tensor:
    """images uint8 [n, h, w, 3] (CUDA) resized to `scaled` = (h_s, w_s) as Pillow's LANCZOS does, flipped first
    where flip [n] is set, cropped to crop = (row, col, h_out, w_out): float32 [n, 3, h_out, w_out] = u / 255."""
    from .. import _lib
    _check_cuda("resample_u8", images, *([] if flip is None else [flip]))
    if images.dtype != torch.uint8 or images.dim() != 4 or images.shape[-1] != 3:
        raise ValueError(f"resample_u8: expected uint8 [n, h, w, 3], got {images.dtype} {tuple(images.shape)}")
    n, h, w, _ = images.shape
    (h_s, w_s), (row, col, h_out, w_out) = scaled, crop
    if h_s > h or w_s > w:
        raise ValueError(f"resample_u8: scaled size {scaled} is larger than the input {(h, w)}")
    images = images.contiguous()
    bh, wh = _device_table(w, w_s, col, w_out, images.device)
    bv, wv = _device_table(h, h_s, row, h_out, images.device)
    if flip is not None:
        if flip.shape != (n,):
            raise ValueError(f"resample_u8: flip must be [{n}], got {tuple(flip.shape)}")
        flip = flip.to(torch.uint8).contiguous()
    out = torch.empty(n, 3, h_out, w_out, dtype=torch.float32, device=images.device)
    desc = _lib.ResampleDesc(n, h, w, h_out, w_out, wh.shape[1], wv.shape[1], images.data_ptr(),
                             0 if flip is None else flip.data_ptr(), bh.data_ptr(), wh.data_ptr(), bv.data_ptr(),
                             wv.data_ptr())
    stream = torch.cuda.current_stream(images.device).cuda_stream
    _lib.check(_lib.on_device(images.device, _lib.lib.ps_image_resample, desc, out.data_ptr(), stream),
               "ps_image_resample")
    return out


def crop_shim_intrinsics(intrinsics: Tensor, in_shape: tuple[int, int], shape: tuple[int, int]) -> Tensor:
    """The intrinsics apply_crop_shim gives views of in_shape (h, w) cropped to shape, without the images."""
    return _crop_intrinsics(intrinsics, scaled_shape(*in_shape, shape), shape)


def _crop_intrinsics(intrinsics: Tensor, scaled: tuple[int, int], shape: tuple[int, int]) -> Tensor:
    """center_crop's intrinsics update, with the rescaled size as its input size."""
    intrinsics = intrinsics.clone()
    intrinsics[..., 0, 0] *= scaled[1] / shape[1]  # fx
    intrinsics[..., 1, 1] *= scaled[0] / shape[0]  # fy
    return intrinsics


def rescale_and_crop_u8(images_u8: Tensor, intrinsics: Tensor, shape: tuple[int, int],
                        flip: Tensor | None = None) -> tuple[Tensor, Tensor]:
    """Decoded views uint8 [*batch, h, w, 3] -> (float32 [*batch, 3, h_out, w_out], intrinsics [*batch, 3, 3]):
    the reference's augmentation flip (where flip [*batch] is set), rescale and center_crop in one launch."""
    *batch, h_in, w_in, c = images_u8.shape
    if c != 3:
        raise ValueError(f"rescale_and_crop_u8: expected 3 channels last, got {tuple(images_u8.shape)}")
    h_out, w_out = shape
    h_s, w_s = scaled_shape(h_in, w_in, shape)
    crop = ((h_s - h_out) // 2, (w_s - w_out) // 2, h_out, w_out)
    f = None if flip is None else flip.expand(batch).reshape(-1)
    out = resample_u8(images_u8.reshape(-1, h_in, w_in, 3), (h_s, w_s), crop, f)
    return out.reshape(*batch, 3, h_out, w_out), _crop_intrinsics(intrinsics, (h_s, w_s), shape)


def _to_u8_hwc(images: Tensor) -> Tensor:
    """The reference's float -> uint8 step, (x * 255).clip(0, 255).type(uint8), channels last."""
    if images.shape[-3] != 3:
        raise ValueError(f"crop shim: expected 3 channels, got {tuple(images.shape)}")
    return (images * 255).clip(min=0, max=255).type(torch.uint8).movedim(-3, -1)


def _as_dtype(out: Tensor, dtype: torch.dtype) -> Tensor:
    """u / 255 in `dtype` as the reference forms it (float64 u / 255, then cast); float32 is the kernel's own."""
    if dtype == torch.float32:
        return out
    u = (out.double() * 255).round()
    # a device divisor: torch turns division by a host scalar into a multiplication by its reciprocal
    return (u / torch.tensor(255.0, dtype=torch.float64, device=u.device)).to(dtype)


def rescale(image: Tensor, shape: tuple[int, int]) -> Tensor:
    """Drop-in for the reference's rescale: float [3, h_in, w_in] (CUDA) -> [3, h_out, w_out]."""
    _check_cuda("rescale", image)
    h, w = shape
    out = resample_u8(_to_u8_hwc(image.detach())[None], (h, w), (0, 0, h, w))
    return _as_dtype(out[0], image.dtype)


def center_crop(images: Tensor, intrinsics: Tensor, shape: tuple[int, int]) -> tuple[Tensor, Tensor]:
    """Drop-in for the reference's center_crop."""
    _check_cuda("center_crop", images)
    *_, h_in, w_in = images.shape
    h_out, w_out = shape
    row, col = (h_in - h_out) // 2, (w_in - w_out) // 2
    return images[..., :, row:row + h_out, col:col + w_out], _crop_intrinsics(intrinsics, (h_in, w_in), shape)


def rescale_and_crop(images: Tensor, intrinsics: Tensor, shape: tuple[int, int]) -> tuple[Tensor, Tensor]:
    """Drop-in for the reference's rescale_and_crop: float [*batch, 3, h, w] (CUDA), one launch for the batch."""
    _check_cuda("rescale_and_crop", images)
    out, intrinsics = rescale_and_crop_u8(_to_u8_hwc(images.detach()), intrinsics, shape)
    return _as_dtype(out, images.dtype), intrinsics


def apply_crop_shim_to_views(views: dict, shape: tuple[int, int]) -> dict:
    images, intrinsics = rescale_and_crop(views["image"], views["intrinsics"], shape)
    return {**views, "image": images, "intrinsics": intrinsics}


def apply_crop_shim(example: dict, shape: tuple[int, int]) -> dict:
    """Drop-in for the reference's apply_crop_shim (context and target are resized in one launch each)."""
    return {**example, "context": apply_crop_shim_to_views(example["context"], shape),
            "target": apply_crop_shim_to_views(example["target"], shape)}


def device_shim(batch: dict, image_shape: tuple[int, int], device: torch.device | str | None = None) -> dict:
    """The call after DatasetRE10k's DataLoader: moves the batch to `device` (default: the current CUDA device;
    host images through pinned memory, without blocking), flips, resamples and crops context and target views in
    one launch, and updates the intrinsics.  Returns the batch the reference's loader + apply_crop_shim give
    ("flip" is consumed), so a model's data shims and step take it unchanged."""
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if device.type != "cuda":
        raise ValueError(f"device_shim: expected a CUDA device, got {device}; there is no CPU path")

    def move(x: Tensor) -> Tensor:
        if x.device == device:
            return x
        if not x.is_cuda and not x.is_pinned():
            x = x.contiguous().pin_memory()
        return x.to(device, non_blocking=True)

    ctx, tgt = batch["context"], batch["target"]
    b, vc, h, w, _ = ctx["image"].shape
    vt = tgt["image"].shape[1]
    if tgt["image"].shape[0] != b or tgt["image"].shape[2:] != ctx["image"].shape[2:]:
        raise ValueError(f"device_shim: context {tuple(ctx['image'].shape)} and target {tuple(tgt['image'].shape)} "
                         "views differ in batch or image size")
    images = torch.empty(b * (vc + vt), h, w, 3, dtype=torch.uint8, device=device)
    images[:b * vc].copy_(move(ctx["image"]).reshape(b * vc, h, w, 3), non_blocking=True)
    images[b * vc:].copy_(move(tgt["image"]).reshape(b * vt, h, w, 3), non_blocking=True)
    flip = move(batch["flip"]).to(torch.uint8)
    flip = torch.cat([flip[:, None].expand(b, vc).reshape(-1), flip[:, None].expand(b, vt).reshape(-1)])
    intrinsics = torch.cat([move(ctx["intrinsics"]).reshape(-1, 3, 3), move(tgt["intrinsics"]).reshape(-1, 3, 3)])
    out, intrinsics = rescale_and_crop_u8(images, intrinsics, tuple(image_shape), flip)

    def views(v: dict, lo: int, hi: int, n: int) -> dict:
        rest = {k: move(x) if isinstance(x, Tensor) else x for k, x in v.items() if k not in ("image", "intrinsics")}
        return {**rest, "image": out[lo:hi].reshape(b, n, *out.shape[1:]),
                "intrinsics": intrinsics[lo:hi].reshape(b, n, 3, 3)}

    result = {k: v for k, v in batch.items() if k not in ("context", "target", "flip")}
    result["context"] = views(ctx, 0, b * vc, vc)
    result["target"] = views(tgt, b * vc, b * (vc + vt), vt)
    return result
