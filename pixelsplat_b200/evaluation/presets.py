"""The reference's RE10k and ACID test configurations as Python values: config/model/encoder/epipolar.yaml with the
dino backbone (config/model/encoder/backbone/dino.yaml), as config/experiment/{re10k,acid}.yaml select it, the
re10k dataset (config/dataset/re10k.yaml) at 256 x 256 with the evaluation view sampler, and the CUDA splatting
decoder.  RE10k and ACID differ only in their data, so both presets build the same model."""
from __future__ import annotations

from pathlib import Path

from ..data import DatasetRE10k, DatasetRE10kCfg, ViewSamplerEvaluationCfg, get_view_sampler
from ..decoder import DecoderSplattingCUDA, DecoderSplattingCUDACfg
from ..encoder import EpipolarTransformerCfg, GaussianAdapterCfg, ImageSelfAttentionCfg
from ..encoder.backbone import BackboneDinoCfg
from ..encoder.encoder_epipolar import EncoderEpipolar, EncoderEpipolarCfg, OpacityMappingCfg

PRESETS = ("re10k", "acid")
IMAGE_SHAPE = (256, 256)
NUM_CONTEXT_VIEWS = 2
SEED = 111123   # config/main.yaml


def encoder_cfg(preset: str) -> EncoderEpipolarCfg:
    if preset not in PRESETS:
        raise ValueError(f"unknown preset {preset!r}; expected one of {PRESETS}")
    return EncoderEpipolarCfg(
        name="epipolar", d_feature=128, num_monocular_samples=32, num_surfaces=1, predict_opacity=False,
        backbone=BackboneDinoCfg("dino", "dino_vitb8", 512), visualizer=None, near_disparity=3.0,
        gaussian_adapter=GaussianAdapterCfg(0.5, 15.0, 4), apply_bounds_shim=True,
        epipolar_transformer=EpipolarTransformerCfg(ImageSelfAttentionCfg(4, 10, 2, 4, 128, 128, 256),
                                                    10, 2, 4, 32, 128, 256, 4),
        opacity_mapping=OpacityMappingCfg(0.0, 0.0, 1), gaussians_per_pixel=3, use_epipolar_transformer=True,
        use_transmittance=False)


def dataset_cfg(root: Path | str, index_path: Path | str,
                image_shape: tuple[int, int] = IMAGE_SHAPE) -> DatasetRE10kCfg:
    vs = ViewSamplerEvaluationCfg("evaluation", Path(index_path), NUM_CONTEXT_VIEWS)
    return DatasetRE10kCfg(image_shape=list(image_shape), background_color=[0.0, 0.0, 0.0],
                           cameras_are_circular=False, overfit_to_scene=None, view_sampler=vs, name="re10k",
                           roots=[Path(root)], baseline_epsilon=1e-3, max_fov=100.0, make_baseline_1=True,
                           augment=True)


def make_test_dataset(cfg: DatasetRE10kCfg) -> DatasetRE10k:
    return DatasetRE10k(cfg, "test", get_view_sampler(cfg.view_sampler, "test", False, False, None))


def build_model(preset: str, dataset: DatasetRE10kCfg) -> tuple[EncoderEpipolar, DecoderSplattingCUDA]:
    """A randomly initialised encoder (no backbone weights are read: a checkpoint holds them all) and the decoder."""
    encoder = EncoderEpipolar(encoder_cfg(preset), num_context_views=NUM_CONTEXT_VIEWS)
    return encoder, DecoderSplattingCUDA(DecoderSplattingCUDACfg("splatting_cuda"), dataset)
