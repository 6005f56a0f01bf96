"""Numpy restatement of Pillow's 8-bit resample passes (libImaging/Resample.c, ImagingResampleHorizontal_8bpc /
ImagingResampleVertical_8bpc) over the coefficient tables of pixelsplat_b200.data.crop_shim.resample_table.

TEST INFRASTRUCTURE ONLY: the CPU tests pin the tables (and this restatement) to PIL.Image.resize bit for bit, and
the GPU tests pin csrc/image_resample.cu to the same result.  Integer arithmetic throughout (int64 here; Pillow's
int32 sums never overflow for 8-bit input), so the order of the sums does not matter."""
from __future__ import annotations

import numpy as np

PRECISION_BITS = 22


def _clip8(s: np.ndarray) -> np.ndarray:
    return np.clip(s >> PRECISION_BITS, 0, 255).astype(np.uint8)


def _pass(img: np.ndarray, bounds: np.ndarray, weights: np.ndarray, axis: int) -> np.ndarray:
    """One pass along `axis` (1: columns, 0: rows) of an [h, w, 3] uint8 image; output pixel j reads input
    pixels bounds[j, 0] + [0, bounds[j, 1]) with weights[j]."""
    size = img.shape[axis]
    taps = weights.shape[1]
    idx = bounds[:, :1].astype(np.int64) + np.arange(taps)                   # [out, taps]
    w = np.where(np.arange(taps) < bounds[:, 1:], weights, 0).astype(np.int64)
    idx = np.minimum(idx, size - 1)
    x = np.take(img.astype(np.int64), idx, axis=axis)                        # axis 1: [h, out, taps, 3]
    if axis == 1:
        s = np.einsum("hotc,ot->hoc", x, w)
    else:
        s = np.einsum("otwc,ot->owc", x, w)
    return _clip8(s + (1 << (PRECISION_BITS - 1)))


def resample_and_crop(img: np.ndarray, scaled: tuple[int, int], crop: tuple[int, int, int, int],
                      flip: bool = False) -> np.ndarray:
    """uint8 [h, w, 3] -> uint8 [h_out, w_out, 3]: flip, Pillow's LANCZOS resize to `scaled`, crop (row, col,
    h_out, w_out), with the tables the kernel receives (horizontal pass first, as Pillow)."""
    from pixelsplat_b200.data.crop_shim import resample_table
    h, w, _ = img.shape
    row, col, h_out, w_out = crop
    if flip:
        img = img[:, ::-1]
    bh, wh = resample_table(w, scaled[1], col, w_out)
    bv, wv = resample_table(h, scaled[0], row, h_out)
    return _pass(_pass(img, bh, wh, 1), bv, wv, 0)
