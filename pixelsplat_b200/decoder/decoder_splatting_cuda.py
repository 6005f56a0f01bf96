"""Drop-in for /root/reference/src/model/decoder/decoder_splatting_cuda.py:20-91 and the
`Decoder` / `DecoderOutput` / `Gaussians` types it uses (decoder.py:20-45, model/types.py:8-12).
Same constructor, forward signature and registry key ("splatting_cuda"); the per-view `repeat`
of the Gaussian tensors is gone (V cameras share one Gaussian set inside the kernels)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, Literal, Optional

import torch
from torch import Tensor, nn

from .cuda_splatting import (DepthRenderingMode, render_depth_views, render_views, render_views_mse,
                             render_views_mse_with_depth, render_views_with_depth)


@dataclass
class Gaussians:
    means: Tensor        # [batch, gaussian, 3]
    covariances: Tensor  # [batch, gaussian, 3, 3]
    harmonics: Tensor    # [batch, gaussian, 3, d_sh]
    opacities: Tensor    # [batch, gaussian]


@dataclass
class DecoderOutput:
    color: Tensor            # [batch, view, 3, height, width]
    depth: Optional[Tensor]  # [batch, view, height, width]


@dataclass
class DecoderSplattingCUDACfg:
    name: Literal["splatting_cuda"]


class DecoderSplattingCUDA(nn.Module):
    background_color: Tensor

    def __init__(self, cfg: DecoderSplattingCUDACfg, dataset_cfg: Any) -> None:
        """`dataset_cfg` only needs a `.background_color` (list of 3 floats), like the reference's
        DatasetCfg (decoder_splatting_cuda.py:29-33)."""
        super().__init__()
        self.cfg = cfg
        self.dataset_cfg = dataset_cfg
        self.register_buffer("background_color",
                             torch.tensor(dataset_cfg.background_color, dtype=torch.float32),
                             persistent=False)

    def forward(self, gaussians: Gaussians, extrinsics: Tensor, intrinsics: Tensor, near: Tensor,
                far: Tensor, image_shape: tuple[int, int],
                depth_mode: DepthRenderingMode | None = None) -> DecoderOutput:
        b, v, _, _ = extrinsics.shape
        args = (extrinsics, intrinsics, near, far, image_shape, self.background_color.expand(b, v, 3),
                gaussians.means, gaussians.covariances, gaussians.harmonics, gaussians.opacities)
        if depth_mode is None:
            return DecoderOutput(render_views(*args), None)
        # the depth map is a channel of the colour pass (two passes under the legacy compositor)
        return DecoderOutput(*render_views_with_depth(*args, mode=depth_mode))

    def forward_mse(self, gaussians: Gaussians, extrinsics: Tensor, intrinsics: Tensor, near: Tensor, far: Tensor,
                    image_shape: tuple[int, int], target: Tensor, want_color: bool = True,
                    depth_mode: DepthRenderingMode | None = None):
        """`forward` with LossMse / PSNR sums taken in the compositor's epilogue (row f-4):
        -> (DecoderOutput (color detached, or None when want_color=False), sse [b, v], sse_clipped [b, v]).
        pixelsplat_b200.loss.mse_from_sse / psnr_from_sse turn the sums into the reference's numbers.
        With `depth_mode`, DecoderOutput.depth is the (differentiable) depth channel of the same pass."""
        b, v, _, _ = extrinsics.shape
        args = (extrinsics, intrinsics, near, far, image_shape, self.background_color.expand(b, v, 3),
                gaussians.means, gaussians.covariances, gaussians.harmonics, gaussians.opacities, target)
        if depth_mode is None:
            sse, sse_clipped, color = render_views_mse(*args, want_color=want_color)
            return DecoderOutput(color, None), sse, sse_clipped
        sse, sse_clipped, color, depth = render_views_mse_with_depth(*args, mode=depth_mode, want_color=want_color)
        return DecoderOutput(color, depth), sse, sse_clipped

    def render_depth(self, gaussians: Gaussians, extrinsics: Tensor, intrinsics: Tensor, near: Tensor,
                     far: Tensor, image_shape: tuple[int, int],
                     mode: DepthRenderingMode = "depth") -> Tensor:
        return render_depth_views(extrinsics, intrinsics, near, far, image_shape, gaussians.means,
                                  gaussians.covariances, gaussians.opacities, mode=mode)


DECODERS = {"splatting_cuda": DecoderSplattingCUDA}


def get_decoder(decoder_cfg: DecoderSplattingCUDACfg, dataset_cfg: Any) -> DecoderSplattingCUDA:
    return DECODERS[decoder_cfg.name](decoder_cfg, dataset_cfg)
