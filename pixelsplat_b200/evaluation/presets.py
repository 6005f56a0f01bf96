"""The reference's RE10k and ACID test configurations as Python values: config/model/encoder/epipolar.yaml with the
dino backbone (config/model/encoder/backbone/dino.yaml), as config/experiment/*.yaml select it, the re10k dataset
(config/dataset/re10k.yaml) at 256 x 256 with the evaluation view sampler, and the CUDA splatting decoder.

One preset per experiment file that builds a model:

    re10k, acid, re10k_depth_loss             the paper's model (the three differ only in data and losses)
    re10k_ablation_no_epipolar_transformer    use_epipolar_transformer: false
    re10k_ablation_no_probabilistic_sampling  num_monocular_samples: 1, gaussians_per_pixel: 1
    re10k_ablation_no_depth_encoding          epipolar_transformer.num_octaves: 0 (the self-attention keeps its 10)
    re10k_3_view                              the paper's model with 3 context views (view_embeddings); at test
                                              time the index's two views plus (left + right) // 2

The number of context views is a property of the preset (`num_context_views`): the evaluation sampler and the
encoder's EpipolarTransformer both take it from there."""
from __future__ import annotations

from dataclasses import replace
from pathlib import Path

from ..data import DatasetRE10k, DatasetRE10kCfg, ViewSamplerEvaluationCfg, get_view_sampler
from ..decoder import DecoderSplattingCUDA, DecoderSplattingCUDACfg
from ..encoder import EpipolarTransformerCfg, GaussianAdapterCfg, ImageSelfAttentionCfg
from ..encoder.backbone import BackboneDinoCfg
from ..encoder.encoder_epipolar import EncoderEpipolar, EncoderEpipolarCfg, OpacityMappingCfg

PRESETS = ("re10k", "acid", "re10k_depth_loss", "re10k_ablation_no_epipolar_transformer",
           "re10k_ablation_no_probabilistic_sampling", "re10k_ablation_no_depth_encoding", "re10k_3_view")
IMAGE_SHAPE = (256, 256)
NUM_CONTEXT_VIEWS = 2   # every preset's but re10k_3_view's; see num_context_views
SEED = 111123   # config/main.yaml

# each experiment file's `model.encoder` overrides, applied to config/model/encoder/epipolar.yaml
_ENCODER_OVERRIDES = {
    "re10k_ablation_no_epipolar_transformer": lambda c: replace(c, use_epipolar_transformer=False),
    "re10k_ablation_no_probabilistic_sampling": lambda c: replace(c, num_monocular_samples=1, gaussians_per_pixel=1),
    "re10k_ablation_no_depth_encoding": lambda c: replace(
        c, epipolar_transformer=replace(c.epipolar_transformer, num_octaves=0)),
}
_CONTEXT_VIEWS = {"re10k_3_view": 3}


def _check(preset: str) -> None:
    if preset not in PRESETS:
        raise ValueError(f"unknown preset {preset!r}; expected one of {PRESETS}")


def num_context_views(preset: str) -> int:
    _check(preset)
    return _CONTEXT_VIEWS.get(preset, NUM_CONTEXT_VIEWS)


def encoder_cfg(preset: str) -> EncoderEpipolarCfg:
    _check(preset)
    cfg = EncoderEpipolarCfg(
        name="epipolar", d_feature=128, num_monocular_samples=32, num_surfaces=1, predict_opacity=False,
        backbone=BackboneDinoCfg("dino", "dino_vitb8", 512), visualizer=None, near_disparity=3.0,
        gaussian_adapter=GaussianAdapterCfg(0.5, 15.0, 4), apply_bounds_shim=True,
        epipolar_transformer=EpipolarTransformerCfg(ImageSelfAttentionCfg(4, 10, 2, 4, 128, 128, 256),
                                                    10, 2, 4, 32, 128, 256, 4),
        opacity_mapping=OpacityMappingCfg(0.0, 0.0, 1), gaussians_per_pixel=3, use_epipolar_transformer=True,
        use_transmittance=False)
    override = _ENCODER_OVERRIDES.get(preset)
    return cfg if override is None else override(cfg)


def dataset_cfg(root: Path | str, index_path: Path | str, image_shape: tuple[int, int] = IMAGE_SHAPE,
                preset: str = "re10k") -> DatasetRE10kCfg:
    vs = ViewSamplerEvaluationCfg("evaluation", Path(index_path), num_context_views(preset))
    return DatasetRE10kCfg(image_shape=list(image_shape), background_color=[0.0, 0.0, 0.0],
                           cameras_are_circular=False, overfit_to_scene=None, view_sampler=vs, name="re10k",
                           roots=[Path(root)], baseline_epsilon=1e-3, max_fov=100.0, make_baseline_1=True,
                           augment=True)


def make_test_dataset(cfg: DatasetRE10kCfg) -> DatasetRE10k:
    return DatasetRE10k(cfg, "test", get_view_sampler(cfg.view_sampler, "test", False, False, None))


def build_model(preset: str, dataset: DatasetRE10kCfg) -> tuple[EncoderEpipolar, DecoderSplattingCUDA]:
    """A randomly initialised encoder (no backbone weights are read: a checkpoint holds them all) and the decoder.
    The dataset's view sampler must draw the preset's number of context views (ValueError)."""
    views = num_context_views(preset)
    if dataset.view_sampler.num_context_views != views:
        raise ValueError(f"preset {preset!r} encodes {views} context views, but the dataset's view sampler draws "
                         f"{dataset.view_sampler.num_context_views}")
    encoder = EncoderEpipolar(encoder_cfg(preset), num_context_views=views)
    return encoder, DecoderSplattingCUDA(DecoderSplattingCUDACfg("splatting_cuda"), dataset)
