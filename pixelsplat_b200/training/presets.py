"""The reference's training configurations as Python values, on top of the evaluation presets (same encoder, same
dataset, here with the bounded view sampler):

    config/main.yaml                      seed 111123, optimizer lr 1.5e-4 / warm_up_steps 2000, gradient_clip_val
                                          0.5, train loader 16 workers / seed 1234, checkpoint every 5000 steps,
                                          val loader batch 1 / 1 worker / seed 3456, val_check_interval 250
    config/experiment/{re10k,acid}.yaml   batch 7, max_steps 300_001, losses [mse, lpips]
    config/experiment/re10k_depth_loss.yaml   max_steps 350_001, losses [mse, lpips, depth], depth sigma_image 12 and
                                          second derivative, train.depth_mode depth
    config/experiment/re10k_ablation_*.yaml   as re10k, with the encoder of the evaluation preset of the same name
    config/experiment/re10k_3_view.yaml   batch 3, 3 context views, context gap 50..90 -> 90..384 over 150_000 steps
    config/loss/{mse,lpips,depth}.yaml    weights 1.0 / 0.05 (apply_after_step 150_000) / 0.25
    config/dataset/view_sampler/bounded.yaml + view_sampler_dataset_specific_config/bounded_re10k.yaml
                                          2 context views, 4 targets, context gap 25 -> 45 over 150_000 steps
"""
from __future__ import annotations

from dataclasses import dataclass, replace
from pathlib import Path

from ..data import DatasetRE10k, DatasetRE10kCfg, StepTracker, ViewSamplerBoundedCfg, get_view_sampler
from ..evaluation import presets as ev
from ..loss import (LossDepth, LossDepthCfg, LossDepthCfgWrapper, LossLpips, LossLpipsCfg, LossLpipsCfgWrapper, LossMse,
                    LossMseCfg, LossMseCfgWrapper)

PRESETS = ("re10k", "acid", "re10k_depth_loss", "re10k_ablation_no_epipolar_transformer",
           "re10k_ablation_no_probabilistic_sampling", "re10k_ablation_no_depth_encoding", "re10k_3_view")
SEED = ev.SEED                  # torch.manual_seed(SEED + rank)
LOADER_SEED = 1234              # the train loader's generator: LOADER_SEED + rank
VAL_SEED = 3456                 # the validation loader's generator and the validation step's RNG: VAL_SEED + rank
VAL_EVERY = 250                 # the reference's trainer.val_check_interval


@dataclass(frozen=True)
class TrainPreset:
    model: str                  # the evaluation preset that builds the encoder
    batch_size: int
    num_workers: int
    max_steps: int
    checkpoint_every: int
    lr: float
    warm_up_steps: int
    max_norm: float
    losses: tuple[str, ...]
    mse_weight: float
    lpips_weight: float
    lpips_apply_after_step: int
    depth_weight: float
    depth_sigma_image: float | None
    depth_use_second_derivative: bool
    depth_mode: str | None
    view_sampler: ViewSamplerBoundedCfg


_BOUNDED_RE10K = ViewSamplerBoundedCfg(
    name="bounded", num_context_views=2, num_target_views=4, min_distance_between_context_views=45,
    max_distance_between_context_views=45, min_distance_to_context_views=0, warm_up_steps=150_000,
    initial_min_distance_between_context_views=25, initial_max_distance_between_context_views=25)

_RE10K = TrainPreset(model="re10k", batch_size=7, num_workers=16, max_steps=300_001, checkpoint_every=5000, lr=1.5e-4,
                     warm_up_steps=2000, max_norm=0.5, losses=("mse", "lpips"), mse_weight=1.0, lpips_weight=0.05,
                     lpips_apply_after_step=150_000, depth_weight=0.25, depth_sigma_image=None,
                     depth_use_second_derivative=False, depth_mode=None, view_sampler=_BOUNDED_RE10K)

TRAIN_PRESETS = {
    "re10k": _RE10K,
    "acid": replace(_RE10K, model="acid"),
    "re10k_depth_loss": replace(_RE10K, max_steps=350_001, losses=("mse", "lpips", "depth"), depth_sigma_image=12.0,
                                depth_use_second_derivative=True, depth_mode="depth"),
    **{name: replace(_RE10K, model=name) for name in ("re10k_ablation_no_epipolar_transformer",
                                                        "re10k_ablation_no_probabilistic_sampling",
                                                        "re10k_ablation_no_depth_encoding")},
    # twice the context gap, with a third view in between
    "re10k_3_view": replace(_RE10K, model="re10k_3_view", batch_size=3, view_sampler=replace(
        _BOUNDED_RE10K, num_context_views=3, min_distance_between_context_views=90,
        max_distance_between_context_views=384, initial_min_distance_between_context_views=50,
        initial_max_distance_between_context_views=90)),
}


def train_preset(name: str) -> TrainPreset:
    if name not in TRAIN_PRESETS:
        raise ValueError(f"unknown preset {name!r}; expected one of {PRESETS}")
    return TRAIN_PRESETS[name]


def dataset_cfg(preset: TrainPreset, root: Path | str, overfit_to_scene: str | None = None,
                image_shape: tuple[int, int] = ev.IMAGE_SHAPE) -> DatasetRE10kCfg:
    # the evaluation preset's dataset with the bounded sampler in place of the index-driven one (no index is read)
    return replace(ev.dataset_cfg(root, Path(), image_shape), view_sampler=preset.view_sampler,
                   overfit_to_scene=overfit_to_scene)


def make_train_dataset(cfg: DatasetRE10kCfg, step_tracker: StepTracker | None) -> DatasetRE10k:
    sampler = get_view_sampler(cfg.view_sampler, "train", cfg.overfit_to_scene is not None,
                               cfg.cameras_are_circular, step_tracker)
    return DatasetRE10k(cfg, "train", sampler)


def make_val_dataset(cfg: DatasetRE10kCfg, step_tracker: StepTracker | None) -> DatasetRE10k:
    """The reference's validation data: stage "val" reads the test split, shuffles chunks and examples, never flips,
    and samples views with the training's bounded sampler and warm-up."""
    sampler = get_view_sampler(cfg.view_sampler, "val", cfg.overfit_to_scene is not None,
                               cfg.cameras_are_circular, step_tracker)
    return DatasetRE10k(cfg, "val", sampler)


def make_losses(preset: TrainPreset, lpips=None) -> list:
    """The preset's loss modules in its order.  `lpips` is an `Lpips` module for LossLpips (default:
    `Lpips.from_files()`, the weights on disk)."""
    made = {"mse": lambda: LossMse(LossMseCfgWrapper(LossMseCfg(preset.mse_weight))),
            "lpips": lambda: LossLpips(LossLpipsCfgWrapper(LossLpipsCfg(preset.lpips_weight,
                                                                        preset.lpips_apply_after_step)), lpips=lpips),
            "depth": lambda: LossDepth(LossDepthCfgWrapper(LossDepthCfg(
                preset.depth_weight, preset.depth_sigma_image, preset.depth_use_second_derivative)))}
    return [made[name]() for name in preset.losses]
