"""pixelSplat's whole encoder: the reference's `EncoderEpipolar` (src/model/encoder/encoder_epipolar.py), images ->
Gaussians.  backbone -> backbone_projection (ReLU + Linear) -> EpipolarTransformer (if use_epipolar_transformer)
-> the tail (`EncoderEpipolarTail`: high-resolution skip, depth predictor, to_gaussians, fused GaussianAdapter).

Child modules sit at the top level under the reference's names (`backbone`, `backbone_projection`,
`epipolar_transformer`, `depth_predictor`, `to_gaussians`, `gaussian_adapter`, `high_resolution_skip`,
`to_opacity`), so a reference `EncoderEpipolar` state dict loads with strict=True.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, Literal, Optional

import torch
from torch import Tensor, nn

from ..decoder.decoder_splatting_cuda import Gaussians
from .backbone import BackboneCfg, get_backbone
from .encoder_tail import EncoderEpipolarTail, EncoderTailCfg, OpacityMappingCfg
from .epipolar_transformer import EpipolarTransformer, EpipolarTransformerCfg
from .gaussian_adapter import GaussianAdapterCfg


@dataclass
class EncoderEpipolarCfg:
    name: Literal["epipolar"]
    d_feature: int
    num_monocular_samples: int
    num_surfaces: int
    predict_opacity: bool
    backbone: BackboneCfg
    visualizer: Any
    near_disparity: float
    gaussian_adapter: GaussianAdapterCfg
    apply_bounds_shim: bool
    epipolar_transformer: EpipolarTransformerCfg
    opacity_mapping: OpacityMappingCfg
    gaussians_per_pixel: int
    use_epipolar_transformer: bool
    use_transmittance: bool


class EncoderEpipolar(EncoderEpipolarTail):
    def __init__(self, cfg: EncoderEpipolarCfg, num_context_views: Optional[int] = None) -> None:
        """`num_context_views` as for EpipolarTransformer: inside the reference tree it is read from the global
        config, as the reference does."""
        super().__init__(EncoderTailCfg(cfg.d_feature, cfg.num_monocular_samples, cfg.num_surfaces,
                                        cfg.predict_opacity, cfg.gaussians_per_pixel, cfg.use_transmittance,
                                        cfg.gaussian_adapter, cfg.opacity_mapping))
        self.cfg = cfg
        self.backbone = get_backbone(cfg.backbone, 3)
        self.backbone_projection = nn.Sequential(nn.ReLU(), nn.Linear(self.backbone.d_out, cfg.d_feature))
        if cfg.use_epipolar_transformer:
            self.epipolar_transformer = EpipolarTransformer(cfg.epipolar_transformer, cfg.d_feature,
                                                            num_context_views=num_context_views)
        else:
            self.epipolar_transformer = None

    def trunk(self, context: dict) -> tuple[Tensor, Optional[Any]]:
        """The part of `forward` before the tail: backbone -> backbone_projection -> epipolar transformer.  Returns
        the features the tail takes [b, v, d_feature, h, w] and the transformer's sampling (None without one).
        Neither `global_step` nor `deterministic` reaches it, and with two context views it draws no random numbers
        (with more, the transformer draws one permutation of its view embeddings), so one trunk can feed several
        calls of the tail, `EncoderEpipolarTail.forward(encoder, features, context, ...)`."""
        features = self.backbone(context)                                           # [b, v, c, h, w]
        features = self.backbone_projection(features.permute(0, 1, 3, 4, 2)).permute(0, 1, 4, 2, 3)
        sampling = None
        if self.cfg.use_epipolar_transformer:
            features, sampling = self.epipolar_transformer(features, context["extrinsics"], context["intrinsics"],
                                                           context["near"], context["far"])
        return features, sampling

    def forward(self, context: dict, global_step: int, deterministic: bool = False,
                visualization_dump: Optional[dict] = None) -> Gaussians:
        features, sampling = self.trunk(context)
        gaussians = super().forward(features, context, global_step, deterministic, visualization_dump)
        if visualization_dump is not None and sampling is not None:
            visualization_dump["sampling"] = sampling
        return gaussians

    def get_data_shim(self):
        def data_shim(batch: dict) -> dict:
            batch = apply_patch_shim(batch, patch_size=self.cfg.epipolar_transformer.self_attention.patch_size
                                     * self.cfg.epipolar_transformer.downscale)
            if self.cfg.apply_bounds_shim:
                _, _, _, h, w = batch["context"]["image"].shape
                batch = apply_bounds_shim(batch, self.cfg.near_disparity * min(h, w), 0.5)
            return batch

        return data_shim

    @property
    def sampler(self):
        return self.epipolar_transformer.epipolar_sampler


# ---- the reference's data shims (src/dataset/shims/{patch_shim,bounds_shim}.py), restated


def _patch_shim_views(views: dict, patch_size: int) -> dict:
    _, _, _, h, w = views["image"].shape
    assert h % 2 == 0 and w % 2 == 0          # even, so that the centre crop does not misalign
    h_new = (h // patch_size) * patch_size
    row = (h - h_new) // 2
    w_new = (w // patch_size) * patch_size
    col = (w - w_new) // 2
    intrinsics = views["intrinsics"].clone()
    intrinsics[:, :, 0, 0] *= w / w_new
    intrinsics[:, :, 1, 1] *= h / h_new
    return {**views, "image": views["image"][:, :, :, row:row + h_new, col:col + w_new], "intrinsics": intrinsics}


def apply_patch_shim(batch: dict, patch_size: int) -> dict:
    """Centre-crops every view to a multiple of `patch_size` and rescales fx, fy to match."""
    return {**batch, "context": _patch_shim_views(batch["context"], patch_size),
            "target": _patch_shim_views(batch["target"], patch_size)}


def compute_depth_for_disparity(extrinsics: Tensor, intrinsics: Tensor, image_shape: tuple[int, int],
                                disparity: float, delta_min: float = 1e-6) -> Tensor:
    """[b]: the depth at which the largest camera baseline moves a point by `disparity` pixels."""
    origins = extrinsics[:, :, :3, 3]
    deltas = (origins[:, None, :, :] - origins[:, :, None, :]).norm(dim=-1).clip(min=delta_min)
    baselines = deltas.flatten(1).amax(dim=1)
    h, w = image_shape
    pixel_size = 1 / torch.tensor((w, h), dtype=torch.float32, device=extrinsics.device)
    pixel_size = torch.einsum("...ij,j->...i", intrinsics[..., :2, :2].inverse(), pixel_size)
    return baselines / (disparity * pixel_size.flatten(1).mean(dim=1))


def apply_bounds_shim(batch: dict, near_disparity: float, far_disparity: float) -> dict:
    """near / far of every view from the context cameras' baseline."""
    context, target = batch["context"], batch["target"]
    _, cv, _, h, w = context["image"].shape
    tv = target["image"].shape[1]
    near = compute_depth_for_disparity(context["extrinsics"], context["intrinsics"], (h, w), near_disparity)
    far = compute_depth_for_disparity(context["extrinsics"], context["intrinsics"], (h, w), far_disparity)
    return {**batch,
            "context": {**context, "near": near[:, None].expand(-1, cv), "far": far[:, None].expand(-1, cv)},
            "target": {**target, "near": near[:, None].expand(-1, tv), "far": far[:, None].expand(-1, tv)}}
