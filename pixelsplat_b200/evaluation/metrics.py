"""Per-image PSNR, SSIM and LPIPS of 8-bit frames: what the reference's metric computer measures on the PNGs its
test step wrote, computed without a PNG or a float image on the host.

`frame_metrics(ground_truth, rendered)` takes float32 renders [n, 3, h, w] (quantised as prep_image does) or uint8
frames [n, h, w, 3] (decoded PNG bytes).  One pass of csrc/eval_images.cu gives the dequantised planes u / 255 and
each image's squared error; PSNR is -10 log10(sse / (3 h w)) (identical images: inf, as in the reference), SSIM is
`compute_ssim` and LPIPS is `compute_lpips`'s network on the planes.
"""
from __future__ import annotations

import torch
from torch import Tensor, nn

from ..loss import compute_ssim, get_lpips
from .frames import frame_pass, psnr_from_sse


@torch.no_grad()
def frame_metrics(ground_truth: Tensor, rendered: Tensor, lpips: nn.Module | None = None,
                  return_frames: bool = False) -> dict[str, Tensor]:
    """{"psnr", "ssim", "lpips"}: float32 [n] each, of the 8-bit frames of `rendered` against `ground_truth`
    (float32 [n, 3, h, w] in [0, 1]).  `lpips` is an `Lpips` module (default: `Lpips.from_files()` on the device),
    used in eval mode.  With `return_frames` (renders only) the dict also holds "frames", uint8 [n, h, w, 3]."""
    n, c, h, w = ground_truth.shape
    fp = frame_pass(rendered, target=ground_truth, frames=return_frames)
    model = (lpips if lpips is not None else get_lpips(ground_truth.device)).eval()
    out = {"psnr": psnr_from_sse(fp.sse, h, w),
           "ssim": compute_ssim(ground_truth, fp.planes),
           "lpips": model(ground_truth, fp.planes, normalize=True)[:, 0, 0, 0].float()}
    if return_frames:
        out["frames"] = fp.frames
    return out


CHUNK = 32   # the reference's test step renders 32 targets at a time


@torch.no_grad()
def frame_metrics_chunked(ground_truth: Tensor, rendered: Tensor, lpips: nn.Module | None = None,
                          return_frames: bool = False, chunk: int = CHUNK) -> dict[str, Tensor]:
    """`frame_metrics` over slices of `chunk` images, concatenated.  The evaluator and the metric computer both
    score through here, so a scene's numbers from its renders and from its written frames are the same bits."""
    parts = [frame_metrics(ground_truth[i:i + chunk], rendered[i:i + chunk], lpips, return_frames)
             for i in range(0, ground_truth.shape[0], chunk)]
    return {k: torch.cat([p[k] for p in parts]) for k in parts[0]}
