"""The 8-bit frame pass of csrc/eval_images.cu: renders -> the uint8 frames the reference writes as PNGs, the float
planes ToTensor reads back from them, and per image the squared error against a target.

`frame_pass` takes either float32 renders [n, 3, h, w] (render mode: quantised as prep_image does) or uint8 frames
[n, h, w, 3] (frame mode: decoded PNG bytes).  Chunks of PS_EVAL_MAX_IMAGES images go to one launch each.  CUDA
tensors only: there is no host path.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import Optional

import torch
from torch import Tensor


@dataclass
class FramePass:
    frames: Optional[Tensor]   # uint8 [n, h, w, 3] (render mode, when asked for)
    planes: Optional[Tensor]   # float32 [n, 3, h, w] = u / 255
    sse: Optional[Tensor]      # float64 [n]: sum of (u / 255 - clip(target, 0, 1))^2


def workspace_bytes(n: int, h: int, w: int) -> int:
    from .. import _lib
    size = ctypes.c_size_t()
    _lib.check(_lib.lib.ps_eval_images_workspace_bytes(n, h, w, ctypes.byref(size)), "ps_eval_images_workspace_bytes")
    return size.value


def frame_pass(images: Tensor, target: Tensor | None = None, frames: bool = True, planes: bool = True) -> FramePass:
    """One pass over `images` (float32 renders [n, 3, h, w] or uint8 frames [n, h, w, 3]) that writes the requested
    outputs: `frames` (render mode only), `planes`, and `sse` when `target` (float32 [n, 3, h, w]) is given."""
    from .. import _lib
    render = images.dtype == torch.float32
    if render:
        if images.dim() != 4 or images.shape[1] != 3:
            raise ValueError(f"frame_pass: renders must be float32 [n, 3, h, w], got {tuple(images.shape)}")
        n, _, h, w = images.shape
    elif images.dtype == torch.uint8:
        if images.dim() != 4 or images.shape[3] != 3:
            raise ValueError(f"frame_pass: frames must be uint8 [n, h, w, 3], got {tuple(images.shape)}")
        n, h, w, _ = images.shape
        frames = False
    else:
        raise ValueError(f"frame_pass: expected float32 renders or uint8 frames, got {images.dtype}")
    if not images.is_cuda:
        raise ValueError(f"frame_pass: expected a CUDA tensor, got one on {images.device}; there is no CPU path")
    if target is not None:
        if target.shape != (n, 3, h, w) or target.dtype != torch.float32 or target.device != images.device:
            raise ValueError(f"frame_pass: target must be float32 [{n}, 3, {h}, {w}] on {images.device}, got "
                             f"{target.dtype} {tuple(target.shape)} on {target.device}")
        target = target.contiguous()
    images = images.contiguous()
    dev = images.device
    out_frames = torch.empty(n, h, w, 3, dtype=torch.uint8, device=dev) if frames else None
    out_planes = torch.empty(n, 3, h, w, dtype=torch.float32, device=dev) if planes else None
    out_sse = torch.empty(n, dtype=torch.float64, device=dev) if target is not None else None
    if n == 0:
        return FramePass(out_frames, out_planes, out_sse)
    chunk = _lib.EVAL_MAX_IMAGES
    ws = None
    if target is not None:
        ws = torch.empty(workspace_bytes(min(n, chunk), h, w), dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    ptr = lambda t, i: 0 if t is None else t[i:i + chunk].data_ptr()
    for i in range(0, n, chunk):
        k = min(chunk, n - i)
        desc = _lib.EvalDesc(_lib.PS_EVAL_RENDER if render else _lib.PS_EVAL_FRAME, k, h, w,
                             ptr(images, i) if render else 0, 0 if render else ptr(images, i), ptr(target, i),
                             ptr(out_frames, i), ptr(out_planes, i), ptr(out_sse, i))
        _lib.check(_lib.on_device(dev, _lib.lib.ps_eval_images, desc, 0 if ws is None else ws.data_ptr(),
                                  0 if ws is None else ws.numel(), stream), "ps_eval_images")
    return FramePass(out_frames, out_planes, out_sse)


def psnr_from_sse(sse: Tensor, h: int, w: int) -> Tensor:
    """-10 log10(sse / (3 h w)) in float64, returned as float32 (the reference's dtype); sse = 0 gives inf."""
    return (-10 * (sse / (3 * h * w)).log10()).float()
