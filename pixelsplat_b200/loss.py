"""Loss / metric of the training step (SURVEY.md 8 row f-4).

Drop-ins for /root/reference/src/loss/loss_mse.py:12-31 (`LossMse`, `LossMseCfg`, `LossMseCfgWrapper`) and
/root/reference/src/evaluation/metrics.py:11-19 (`compute_psnr`), plus the fused route: the compositor's
epilogue already returns, per view, sse = sum (C - t)^2 and sse_clipped = sum (clip C - clip t)^2
(`DecoderSplattingCUDA.forward_mse`), from which

    LossMse          = weight * sse.sum() / (b v 3 h w)                       (mse_from_sse)
    compute_psnr     = -10 log10(sse_clipped / (3 h w))                       (psnr_from_sse)

with the rendered image never re-read for the loss and dL/dC never written as a tensor.

`LossDepth` / `LossDepthCfg` / `LossDepthCfgWrapper` are the drop-in for /root/reference/src/loss/loss_depth.py: an
edge-aware smoothness penalty on the rendered depth map (`DecoderOutput.depth`), which the fused depth channel
(`DecoderSplattingCUDA.forward(depth_mode=...)`) provides.
"""
from __future__ import annotations

from dataclasses import dataclass, fields

import torch
from torch import Tensor, nn


@dataclass
class LossMseCfg:
    weight: float


@dataclass
class LossMseCfgWrapper:
    mse: LossMseCfg


class LossMse(nn.Module):
    """Same constructor and forward signature as the reference's LossMse (prediction has `.color`,
    batch["target"]["image"] is the ground truth)."""

    def __init__(self, cfg: LossMseCfgWrapper) -> None:
        super().__init__()
        (field,) = fields(type(cfg))
        self.cfg = getattr(cfg, field.name)
        self.name = field.name

    def forward(self, prediction, batch, gaussians=None, global_step: int = 0) -> Tensor:
        delta = prediction.color - batch["target"]["image"]
        return self.cfg.weight * (delta ** 2).mean()

    def from_sse(self, sse: Tensor, image_shape: tuple[int, int]) -> Tensor:
        """The same number from the fused epilogue's per-view sums [b, v]."""
        return mse_from_sse(sse, image_shape, self.cfg.weight)


def mse_from_sse(sse: Tensor, image_shape: tuple[int, int], weight: float = 1.0) -> Tensor:
    h, w = image_shape
    return weight * sse.sum() / (sse.numel() * 3 * h * w)


@torch.no_grad()
def compute_psnr(ground_truth: Tensor, predicted: Tensor) -> Tensor:
    """[batch, c, h, w] x 2 -> [batch] (metrics.py:11-19)."""
    ground_truth = ground_truth.clip(min=0, max=1)
    predicted = predicted.clip(min=0, max=1)
    mse = ((ground_truth - predicted) ** 2).mean(dim=(1, 2, 3))
    return -10 * mse.log10()


@torch.no_grad()
def psnr_from_sse(sse_clipped: Tensor, image_shape: tuple[int, int], channels: int = 3) -> Tensor:
    h, w = image_shape
    return -10 * (sse_clipped / (channels * h * w)).log10()


@dataclass
class LossDepthCfg:
    weight: float
    sigma_image: float | None
    use_second_derivative: bool


@dataclass
class LossDepthCfgWrapper:
    depth: LossDepthCfg


def depth_smoothness(depth: Tensor, near: Tensor, far: Tensor, image: Tensor | None, sigma_image: float | None,
                     second_derivative: bool) -> Tensor:
    """Mean absolute finite difference of the depth map along x plus the same along y (first or second order),
    each difference down-weighted by exp(-sigma * colour edge) when `sigma_image` is set.  The depth map [b, v, h, w]
    is first clamped to [log near, log far] and mapped to [0, 1] on that interval (near / far [b, v]; `image`
    [b, v, c, h, w] is the ground truth whose largest per-channel difference is the edge)."""
    lo, hi = near.log()[..., None, None], far.log()[..., None, None]
    d = (depth.minimum(hi).maximum(lo) - lo) / (hi - lo)
    order = 2 if second_derivative else 1
    dx, dy = d.diff(n=order, dim=-1), d.diff(n=order, dim=-2)
    if sigma_image is not None:
        ex = image.diff(dim=-1).amax(dim=-3)           # [b, v, h, w - 1]
        ey = image.diff(dim=-2).amax(dim=-3)           # [b, v, h - 1, w]
        if second_derivative:                          # the larger edge of the two differences a term spans
            ex = torch.maximum(ex[..., :, 1:], ex[..., :, :-1])
            ey = torch.maximum(ey[..., 1:, :], ey[..., :-1, :])
        dx = dx * torch.exp(-sigma_image * ex)
        dy = dy * torch.exp(-sigma_image * ey)
    return dx.abs().mean() + dy.abs().mean()


class LossDepth(nn.Module):
    """Same constructor and forward signature as the reference's LossDepth: prediction.depth [b, v, h, w],
    batch["target"]["near"] / ["far"] [b, v] and ["image"] [b, v, 3, h, w]."""

    def __init__(self, cfg: LossDepthCfgWrapper) -> None:
        super().__init__()
        (field,) = fields(type(cfg))
        self.cfg = getattr(cfg, field.name)
        self.name = field.name

    def forward(self, prediction, batch, gaussians=None, global_step: int = 0) -> Tensor:
        t = batch["target"]
        return self.cfg.weight * depth_smoothness(prediction.depth, t["near"], t["far"], t["image"],
                                                  self.cfg.sigma_image, self.cfg.use_second_derivative)
