"""Drop-ins for the reference's src/misc/image_io.py: `prep_image`, `save_image` and `load_image`.

The quantisation (clip, * 255, truncation) runs in the frame pass of csrc/eval_images.cu, so only uint8 bytes reach
the host; PNG encoding and decoding go through PIL on the host, as in the reference.  `load_image` uploads the
decoded bytes and dequantises them on the device (frame mode), so the float image never exists on the host.
Images must be CUDA tensors: there is no host path.
"""
from __future__ import annotations

from pathlib import Path
from typing import Union

import numpy as np
import torch
from PIL import Image
from torch import Tensor

from .frames import frame_pass


def quantise(image: Tensor) -> Tensor:
    """float32 [3, h, w] or [n, 3, h, w] (CUDA) -> uint8 [h, w, 3] or [n, h, w, 3] on the device, prep_image's
    bytes.  Other float types would be multiplied by 255 in their own precision by the reference; they raise."""
    if image.dtype != torch.float32:
        raise ValueError(f"quantise: expected a float32 image, got {image.dtype}")
    batched = image.dim() == 4
    x = image.detach()
    frames = frame_pass(x if batched else x[None], planes=False).frames
    return frames if batched else frames[0]


def prep_image(image: Tensor) -> np.ndarray:
    """The reference's prep_image: [h, w], [c, h, w] or [b, c, h, w] (c = 1, 3 or 4; batches side by side) ->
    uint8 [h, w, c'] on the host, c' = 3 or 4."""
    if image.dim() == 4:
        image = image.permute(1, 2, 0, 3).reshape(image.shape[1], image.shape[2], -1)   # b c h w -> c h (b w)
    if image.dim() == 2:
        image = image[None]
    if image.shape[0] == 1:
        image = image.expand(3, -1, -1)
    if image.shape[0] not in (3, 4):
        raise ValueError(f"prep_image: expected 1, 3 or 4 channels, got {tuple(image.shape)}")
    if not image.is_cuda:
        raise ValueError(f"prep_image: expected a CUDA tensor, got one on {image.device}; there is no CPU path")
    if image.shape[0] == 3:
        return quantise(image).cpu().numpy()
    # alpha goes through the same pass as a second (grey) image
    pair = torch.stack([image[:3], image[3:].expand(3, -1, -1)])
    frames = quantise(pair)
    return torch.cat([frames[0], frames[1, ..., :1]], dim=-1).cpu().numpy()


def save_frame(frame: np.ndarray, path: Union[Path, str]) -> None:
    """Writes uint8 [h, w, 3 | 4] as a PNG (or whatever the suffix names), creating the parent directory."""
    path = Path(path)
    path.parent.mkdir(exist_ok=True, parents=True)
    Image.fromarray(frame).save(path)


def save_image(image: Tensor, path: Union[Path, str]) -> None:
    """The reference's save_image: the image (assumed in [0, 1]) through prep_image, written by PIL."""
    save_frame(prep_image(image), path)


def read_frame(path: Union[Path, str]) -> np.ndarray:
    """A decoded image file's first three channels, uint8 [h, w, 3] (ToTensor(Image.open(path))[:3] times 255).
    RGB and RGBA images only."""
    with Image.open(path) as im:
        if im.mode not in ("RGB", "RGBA"):
            raise ValueError(f"read_frame: {path} is a {im.mode} image; expected RGB or RGBA")
        return np.ascontiguousarray(np.asarray(im)[..., :3])


def load_frames(paths, device: torch.device | str = "cuda") -> Tensor:
    """The decoded frames of `paths`, uint8 [n, h, w, 3] on `device` (one host-to-device copy of bytes)."""
    frames = np.stack([read_frame(p) for p in paths])
    return torch.from_numpy(frames).pin_memory().to(device, non_blocking=True)


def load_image(path: Union[Path, str], device: torch.device | str = "cuda") -> Tensor:
    """The reference's load_image, ToTensor(Image.open(path))[:3]: float32 [3, h, w] = u / 255, on `device`."""
    return frame_pass(load_frames([path], device), frames=False).planes[0]
