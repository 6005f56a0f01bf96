"""The reference's metric computer (MetricComputer.test_step, src/evaluation/metric_computer.py, as its
src/scripts/compute_metrics.py runs it): the saved frames of several methods scored against a test split.

Per scene, each method's `<path>/<scene>/color/{index:06}.png` for every target index is decoded on the host,
uploaded as uint8 and scored by `frame_metrics` (the frame pass of csrc/eval_images.cu in frame mode, then SSIM and
LPIPS on the planes).  A scene whose directory or any frame is missing for any method is skipped, as in the
reference.  The result is each `lpips_<key>`, `ssim_<key>` and `psnr_<key>` averaged over the scored scenes.
The reference's side-by-side images and animations are not made.
"""
from __future__ import annotations

import json
from dataclasses import dataclass, field
from pathlib import Path
from typing import Iterable, Optional, Sequence

import torch
from torch import nn

from ..data import device_shim
from .evaluator import mean_over_scenes
from .image_io import load_frames
from .metrics import frame_metrics_chunked


@dataclass
class Method:
    name: str
    key: str
    path: Path


@dataclass
class MetricsResult:
    mean: dict[str, float]                                   # over the scored scenes
    scenes: dict[str, dict[str, float]] = field(default_factory=dict)
    skipped: list[str] = field(default_factory=list)


def scene_frame_paths(methods: Sequence[Method], scene: str, indices: Iterable[int]) -> Optional[dict[str, list[Path]]]:
    """{method key: its frame paths for `indices`}, or None when the scene is to be skipped: a method has no
    directory for it, or lacks one of the frames."""
    indices = [int(i) for i in indices]
    out = {}
    for m in methods:
        if not (Path(m.path) / scene).exists():
            return None
    for m in methods:
        paths = [Path(m.path) / scene / "color" / f"{i:0>6}.png" for i in indices]
        if not all(p.is_file() for p in paths):
            return None
        out[m.key] = paths
    return out


def scene_metric_keys(methods: Sequence[Method]) -> list[str]:
    return [f"{metric}_{m.key}" for m in methods for metric in ("lpips", "ssim", "psnr")]


def preview_table(running: dict[str, float], methods: Sequence[Method]) -> str:
    """The reference's running preview: one row per method, PSNR (dB), LPIPS and SSIM to three decimals."""
    rows = [("Method", "PSNR (dB)", "LPIPS", "SSIM")]
    rows += [(m.key, *(f"{running[f'{metric}_{m.key}']:.3f}" for metric in ("psnr", "lpips", "ssim")))
             for m in methods]
    widths = [max(len(r[i]) for r in rows) for i in range(4)]
    lines = ["  ".join(c.ljust(wd) for c, wd in zip(r, widths)).rstrip() for r in rows]
    lines.insert(1, "  ".join("-" * wd for wd in widths))
    return "\n".join(lines)


@torch.no_grad()
def compute_metrics(methods: Sequence[Method], loader: Iterable[dict], lpips: nn.Module | None = None,
                    image_shape: tuple[int, int] = (256, 256), output_path: Path | str | None = None,
                    device: torch.device | str | None = None, log=print) -> MetricsResult:
    """Scores every method's frames on each batch (batch size 1) of a test DataLoader.  `lpips` defaults to
    `Lpips.from_files()`.  Writes the means as JSON to `output_path` when given."""
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    result = MetricsResult({})
    for batch in loader:
        (scene,) = batch["scene"]
        assert batch["context"]["image"].shape[0] == 1
        paths = scene_frame_paths(methods, scene, batch["target"]["index"][0])
        if paths is None:
            if log is not None:
                log(f'Skipping "{scene}".')
            result.skipped.append(scene)
            continue
        gt = device_shim(batch, image_shape, device)["target"]["image"][0]
        metrics = {}
        for m in methods:
            per_view = frame_metrics_chunked(gt, load_frames(paths[m.key], device), lpips)
            metrics.update({f"{k}_{m.key}": float(per_view[k].mean()) for k in ("lpips", "ssim", "psnr")})
        result.scenes[scene] = metrics
        result.mean = mean_over_scenes(result.scenes.values())
        if log is not None:
            log(preview_table(result.mean, methods))
    if output_path is not None:
        output_path = Path(output_path)
        output_path.parent.mkdir(exist_ok=True, parents=True)
        output_path.write_text(json.dumps(result.mean))
    return result
