"""The reference's evaluation-index generator (src/evaluation/evaluation_index_generator.py and
src/scripts/generate_evaluation_index.py): for each test scene, a context pair whose two views overlap enough and a
few target frames between them, drawn from one seeded CPU generator that runs through the scenes in loader order.

Per scene of v frames on an h x w ray grid: for each context frame c of `randperm(v)`, walk away from c in both
directions from c +- min_distance; a frame k is a candidate when min(overlap_a, overlap_b) lies in [min_overlap,
max_overlap], where overlap_a is the share of k's rays that project into c's image and overlap_b the share of c's
rays that project into k's image (project_rays without near / far); a walk stops at the first overlap below
min_overlap or past max_distance.  The first c with a candidate gives the entry: a candidate drawn with randint,
then num_target_views distinct frames between the pair (redrawn until distinct).  No such c gives None.

The overlaps come from one `ps_view_overlap` launch per context frame tried, which counts every candidate the two
walks can reach at once (csrc/epipolar_geometry.cu); the counts are copied to the host once, and the walk, its
float32 comparisons and its random draws are replayed there exactly as the reference runs them.  Previews
(save_previews) are not provided.
"""
from __future__ import annotations

import ctypes
import json
from dataclasses import asdict, dataclass
from pathlib import Path
from typing import Callable, Iterable

import numpy as np
import torch
from torch import Tensor

from .. import _lib
from ..data.crop_shim import crop_shim_intrinsics
from ..data.dataset_re10k import IMAGE_SHAPE, DatasetRE10k
from ..data.view_sampler import IndexEntry


@dataclass
class EvaluationIndexGeneratorCfg:
    """config/generate_evaluation_index.yaml's index_generator, without save_previews."""
    num_target_views: int = 3
    min_distance: int = 45
    max_distance: int = 135
    min_overlap: float = 0.6
    max_overlap: float = 1.0
    output_path: Path = Path("outputs/evaluation_index_re10k")
    seed: int = 123

    def __post_init__(self) -> None:
        if self.num_target_views < 1 or self.min_distance < 0 or self.max_distance < 0:
            raise ValueError("num_target_views must be >= 1 and min_distance / max_distance >= 0")
        # a pair spans at least min_distance + 1 frames; fewer than num_target_views would redraw the targets forever
        if self.min_distance + 1 < self.num_target_views:
            raise ValueError(f"min_distance + 1 ({self.min_distance + 1}) frames cannot hold num_target_views "
                             f"({self.num_target_views}) distinct targets")


# (context, first, count) -> int counts [count, 2]: (rays of k in c's image, rays of c in k's image), k = first + i
CountsFn = Callable[[int, int, int], np.ndarray]


def view_overlap_counts(extrinsics: Tensor, intrinsics: Tensor, h: int, w: int, context: int, first: int,
                        count: int) -> Tensor:
    """ps_view_overlap on one scene's CUDA float32 cameras (c2w [v, 4, 4], normalised intrinsics [v, 3, 3]):
    int32 counts [count, 2] on the device, enqueued on the current stream."""
    if not (extrinsics.is_cuda and intrinsics.is_cuda):
        raise ValueError("view_overlap_counts: the cameras must be CUDA tensors")
    e = extrinsics.detach().to(torch.float32).contiguous()
    k = intrinsics.detach().to(torch.float32).contiguous()
    v = e.shape[0]
    if e.shape != (v, 4, 4) or k.shape != (v, 3, 3):
        raise ValueError(f"view_overlap_counts: expected [v, 4, 4] and [v, 3, 3], got {tuple(e.shape)}, "
                         f"{tuple(k.shape)}")
    out = torch.empty((count, 2), dtype=torch.int32, device=e.device)
    stream = torch.cuda.current_stream(e.device)
    rc = _lib.on_device(e.device, _lib.lib.ps_view_overlap, v, h, w, ctypes.c_void_p(e.data_ptr()),
                        ctypes.c_void_p(k.data_ptr()), context, first, count, ctypes.c_void_p(out.data_ptr()),
                        ctypes.c_void_p(stream.cuda_stream))
    _lib.check(rc, "ps_view_overlap")
    return out


def candidate_range(context: int, v: int, cfg: EvaluationIndexGeneratorCfg) -> tuple[int, int] | None:
    """(first, count) of the contiguous frame range that covers every frame the two walks from `context` can
    reach, or None when neither walk has a first frame inside the scene."""
    reach = max(cfg.min_distance, cfg.max_distance + 1)     # a walk evaluates the frame past max_distance, then stops
    ks = []
    for step in (1, -1):
        if 0 <= context + step * cfg.min_distance < v:
            ks += [context + step * cfg.min_distance, context + step * reach]
    if not ks:
        return None
    first, last = max(0, min(ks)), min(v - 1, max(ks))
    return first, last - first + 1


def in_overlap_range(overlap: np.float32, cfg: EvaluationIndexGeneratorCfg) -> bool:
    """`min_overlap <= overlap <= max_overlap` as torch evaluates it for a 0-d float32 tensor: in float32."""
    return bool(np.float32(cfg.min_overlap) <= overlap <= np.float32(cfg.max_overlap))


def walk_context(context: int, v: int, counts: np.ndarray, first: int, rays: int, cfg: EvaluationIndexGeneratorCfg,
                 generator: torch.Generator) -> IndexEntry | None:
    """The reference's walk from one context frame over the candidates' counts (counts[k - first] for frame k),
    and its draws when a candidate is found."""
    n = np.float32(rays)
    valid = []
    for step in (1, -1):
        k = context + step * cfg.min_distance
        while 0 <= k < v:
            a, b = counts[k - first]
            overlap_a, overlap_b = np.float32(a) / n, np.float32(b) / n      # .float().mean() of the 0 / 1 mask
            overlap = overlap_b if overlap_b < overlap_a else overlap_a      # min(overlap_a, overlap_b)
            if in_overlap_range(overlap, cfg):
                valid.append(k)
            if overlap < np.float32(cfg.min_overlap) or abs(k - context) > cfg.max_distance:
                break
            k += step
    if not valid:
        return None
    chosen = valid[int(torch.randint(0, len(valid), size=tuple(), generator=generator))]
    left, right = min(chosen, context), max(chosen, context)
    while True:
        targets = torch.randint(left, right + 1, (cfg.num_target_views,), generator=generator)
        if (targets.unique(return_counts=True)[1] == 1).all():
            break
    return IndexEntry(context=(left, right), target=tuple(sorted(targets.tolist())))


def scene_entry(v: int, h: int, w: int, cfg: EvaluationIndexGeneratorCfg, generator: torch.Generator,
                counts_fn: CountsFn) -> IndexEntry | None:
    """One scene's entry: the context frames in randperm order until one has a candidate.  counts_fn gives the
    overlap counts of the range `candidate_range` returns."""
    for context in torch.randperm(v, generator=generator).tolist():
        span = candidate_range(context, v, cfg)
        if span is None:
            continue
        entry = walk_context(context, v, counts_fn(context, *span), span[0], h * w, cfg, generator)
        if entry is not None:
            return entry
    return None


def generate_scene_entry(extrinsics: Tensor, intrinsics: Tensor, h: int, w: int, cfg: EvaluationIndexGeneratorCfg,
                         generator: torch.Generator) -> IndexEntry | None:
    """EvaluationIndexGenerator.test_step for one scene: cameras on a CUDA device (c2w [v, 4, 4], normalised
    intrinsics [v, 3, 3]), the h x w image shape, and the CPU generator shared by every scene.  One kernel launch
    and one device-to-host copy per context frame tried."""
    def counts(context: int, first: int, count: int) -> np.ndarray:
        return view_overlap_counts(extrinsics, intrinsics, h, w, context, first, count).cpu().numpy()
    return scene_entry(extrinsics.shape[0], h, w, cfg, generator, counts)


def camera_loader(dataset_root: Path | str, num_workers: int = 8) -> torch.utils.data.DataLoader:
    """The reference's test loader (batch size 1, num_workers 8 in config/generate_evaluation_index.yaml) over the
    test split in camera mode.  Worker i reads chunks i, i + n, ... and the loader takes one scene from each worker
    in turn, so the scene order, and with it the index, depends on num_workers."""
    from dataclasses import replace

    from .presets import dataset_cfg
    cfg = replace(dataset_cfg(dataset_root, "unused"), view_sampler=None)
    return torch.utils.data.DataLoader(DatasetRE10k(cfg, "test", None, cameras_only=True), batch_size=1,
                                       num_workers=num_workers)


def generate_index(scenes: Iterable[dict], h: int, w: int, cfg: EvaluationIndexGeneratorCfg,
                   device: torch.device | str) -> dict[str, IndexEntry | None]:
    """Every scene's entry, in the order `scenes` yields them (`camera_loader`); the intrinsics get the crop shim to
    h x w, as the reference's loader gives them, and the generator is seeded once with cfg.seed."""
    generator = torch.Generator()
    generator.manual_seed(cfg.seed)
    index: dict[str, IndexEntry | None] = {}
    for batch in scenes:
        (scene,) = batch["scene"]
        intrinsics = crop_shim_intrinsics(batch["intrinsics"][0], IMAGE_SHAPE[:2], (h, w))
        index[scene] = generate_scene_entry(batch["extrinsics"][0].to(device), intrinsics.to(device), h, w, cfg,
                                            generator)
    return index


def index_json(index: dict[str, IndexEntry | None]) -> dict:
    return {k: None if v is None else asdict(v) for k, v in index.items()}


def video_index_json(index: dict[str, IndexEntry | None]) -> dict:
    """generate_video_evaluation_index.py: the same context pairs, with every frame between them as a target."""
    out = {}
    for scene, entry in index.items():
        if entry is None:
            out[scene] = None
            continue
        a, b = entry.context
        out[scene] = {"context": [a, b], "target": list(range(a, b + 1))}
    return out


def save_index(index: dict[str, IndexEntry | None], output_path: Path, video: bool = False) -> list[Path]:
    """<output_path>/evaluation_index.json in the reference's json.dump layout, and with `video`
    <output_path>/evaluation_index_video.json."""
    output_path = Path(output_path)
    output_path.mkdir(exist_ok=True, parents=True)
    written = [output_path / "evaluation_index.json"]
    with written[0].open("w") as f:
        json.dump(index_json(index), f)
    if video:
        written.append(output_path / "evaluation_index_video.json")
        with written[1].open("w") as f:
            json.dump(video_index_json(index), f)
    return written
