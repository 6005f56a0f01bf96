"""The two view samplers the reference's experiment configs use (src/dataset/view_sampler/), restated so that a
seeded loader draws from torch's RNG in the reference's order: `ViewSamplerBounded` (random context gap with a
warm-up schedule) and `ViewSamplerEvaluation` (fixed indices from an evaluation index JSON)."""
from __future__ import annotations

import json
from dataclasses import dataclass
from pathlib import Path
from typing import Literal

import torch
from torch import Tensor

Stage = Literal["train", "val", "test"]


class StepTracker:
    """The training step, shared with DataLoader workers (a shared-memory int64), like the reference's
    StepTracker: the bounded sampler's warm-up reads it in the workers."""

    def __init__(self) -> None:
        self.step = torch.tensor(0, dtype=torch.int64).share_memory_()

    def set_step(self, step: int) -> None:
        self.step.fill_(step)

    def get_step(self) -> int:
        return int(self.step.item())


class ViewSampler:
    def __init__(self, cfg, stage: Stage, is_overfitting: bool, cameras_are_circular: bool,
                 step_tracker: StepTracker | None) -> None:
        self.cfg = cfg
        self.stage = stage
        self.is_overfitting = is_overfitting
        self.cameras_are_circular = cameras_are_circular
        self.step_tracker = step_tracker

    @property
    def global_step(self) -> int:
        return 0 if self.step_tracker is None else self.step_tracker.get_step()


@dataclass
class ViewSamplerBoundedCfg:
    name: Literal["bounded"]
    num_context_views: int
    num_target_views: int
    min_distance_between_context_views: int
    max_distance_between_context_views: int
    min_distance_to_context_views: int
    warm_up_steps: int
    initial_min_distance_between_context_views: int
    initial_max_distance_between_context_views: int


class ViewSamplerBounded(ViewSampler):
    def schedule(self, initial: int, final: int) -> int:
        fraction = self.global_step / self.cfg.warm_up_steps
        return min(initial + int((final - initial) * fraction), final)

    def sample(self, scene: str, extrinsics: Tensor, intrinsics: Tensor,
               device: torch.device = torch.device("cpu")) -> tuple[Tensor, Tensor]:
        """(context indices, target indices); ValueError when the scene has too few frames."""
        num_views = extrinsics.shape[0]
        cfg = self.cfg
        if self.stage == "test":
            max_gap = min_gap = cfg.max_distance_between_context_views
        elif cfg.warm_up_steps > 0:
            max_gap = self.schedule(cfg.initial_max_distance_between_context_views,
                                    cfg.max_distance_between_context_views)
            min_gap = self.schedule(cfg.initial_min_distance_between_context_views,
                                    cfg.min_distance_between_context_views)
        else:
            max_gap = cfg.max_distance_between_context_views
            min_gap = cfg.min_distance_between_context_views

        if not self.cameras_are_circular:
            max_gap = min(num_views - 1, max_gap)
        min_gap = max(2 * cfg.min_distance_to_context_views, min_gap)
        if max_gap < min_gap:
            raise ValueError("Example does not have enough frames!")
        context_gap = torch.randint(min_gap, max_gap + 1, size=tuple(), device=device).item()

        left = torch.randint(num_views if self.cameras_are_circular else num_views - context_gap,
                             size=tuple(), device=device).item()
        if self.stage == "test":
            left = left * 0
        right = left + context_gap
        if self.is_overfitting:
            left *= 0
            right *= 0
            right += max_gap

        if self.stage == "test":
            index_target = torch.arange(left, right + 1, device=device)
        else:
            index_target = torch.randint(left + cfg.min_distance_to_context_views,
                                         right + 1 - cfg.min_distance_to_context_views,
                                         size=(cfg.num_target_views,), device=device)
        if self.cameras_are_circular:
            index_target %= num_views
            right %= num_views

        extra_views = []
        if cfg.num_context_views > 2:
            num_extra_views = cfg.num_context_views - 2
            while len(set(extra_views)) != num_extra_views:
                extra_views = torch.randint(left + 1, right, (num_extra_views,)).tolist()
        return torch.tensor((left, *extra_views, right)), index_target

    @property
    def num_context_views(self) -> int:
        return self.cfg.num_context_views

    @property
    def num_target_views(self) -> int:
        return self.cfg.num_target_views


@dataclass
class ViewSamplerEvaluationCfg:
    name: Literal["evaluation"]
    index_path: Path
    num_context_views: int


@dataclass
class IndexEntry:
    context: tuple[int, ...]
    target: tuple[int, ...]


def add_third_context_index(indices: Tensor) -> Tensor:
    """Two context indices -> (left, middle, right), for 3-view models evaluated on a 2-view index."""
    left, right = indices.unbind(dim=-1)
    return torch.stack((left, (left + right) // 2, right), dim=-1)


class ViewSamplerEvaluation(ViewSampler):
    def __init__(self, cfg: ViewSamplerEvaluationCfg, stage: Stage, is_overfitting: bool,
                 cameras_are_circular: bool, step_tracker: StepTracker | None) -> None:
        super().__init__(cfg, stage, is_overfitting, cameras_are_circular, step_tracker)
        with Path(cfg.index_path).open("r") as f:
            self.index = {k: None if v is None else IndexEntry(tuple(v["context"]), tuple(v["target"]))
                          for k, v in json.load(f).items()}

    def sample(self, scene: str, extrinsics: Tensor, intrinsics: Tensor,
               device: torch.device = torch.device("cpu")) -> tuple[Tensor, Tensor]:
        entry = self.index.get(scene)
        if entry is None:
            raise ValueError(f"No indices available for scene {scene}.")
        context_indices = torch.tensor(entry.context, dtype=torch.int64, device=device)
        target_indices = torch.tensor(entry.target, dtype=torch.int64, device=device)
        v = self.cfg.num_context_views
        if v > len(context_indices) and v == 3:
            context_indices = add_third_context_index(context_indices)
        return context_indices, target_indices

    @property
    def num_context_views(self) -> int:
        return 0

    @property
    def num_target_views(self) -> int:
        return 0


VIEW_SAMPLERS = {"bounded": ViewSamplerBounded, "evaluation": ViewSamplerEvaluation}
ViewSamplerCfg = ViewSamplerBoundedCfg | ViewSamplerEvaluationCfg


def get_view_sampler(cfg: ViewSamplerCfg, stage: Stage, overfit: bool, cameras_are_circular: bool,
                     step_tracker: StepTracker | None) -> ViewSampler:
    if cfg.name not in VIEW_SAMPLERS:
        raise ValueError(f"view sampler {cfg.name!r} is not available (bounded, evaluation)")
    return VIEW_SAMPLERS[cfg.name](cfg, stage, overfit, cameras_are_circular, step_tracker)
