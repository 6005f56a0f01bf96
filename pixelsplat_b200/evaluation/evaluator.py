"""The reference's test step (ModelWrapper.test_step, src/model/model_wrapper.py) and the scoring its metric
computer then does on the written PNGs, in one pass over a test split.

Per scene: the encoder's data shim, the encoder (deterministic=False unless asked, as in the reference), the targets
rendered in chunks of 32, and the 8-bit frame pass (csrc/eval_images.cu) on each chunk.  The metrics are those of
the 8-bit frames, exactly what the reference measures on its PNGs; the frames are written as
`<output>/<scene>/color/{index:06}.png` (and the context views as `context/{index:06}.png`) when an output path is
given.  `run` keeps the mean over scenes and writes `benchmark.json` and `peak_memory.json` in the reference's
layout.

Timing differs from the reference's Benchmarker on purpose: that one reads the host clock around the encoder and
the render loop, which, with asynchronous CUDA launches, measures launch time rather than GPU time.  Here CUDA events
bracket the same work and are read once the scene has finished.
"""
from __future__ import annotations

import json
from collections import defaultdict
from contextlib import contextmanager
from dataclasses import dataclass, field
from pathlib import Path
from typing import Iterable, Optional

import torch
from torch import Tensor, nn

from ..data import device_shim
from .image_io import quantise, save_frame
from .metrics import CHUNK, frame_metrics_chunked

METRICS = ("psnr", "ssim", "lpips")


class Benchmarker:
    """The reference's Benchmarker (src/misc/benchmarker.py) with CUDA-event times: `time(tag, num_calls)` brackets
    work on the current stream; `collect()` waits for the events and appends seconds per call, `num_calls` times."""

    def __init__(self) -> None:
        self.execution_times: dict[str, list[float]] = defaultdict(list)
        self._pending: list = []

    @contextmanager
    def time(self, tag: str, num_calls: int = 1):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        try:
            yield
        finally:
            end.record()
            self._pending.append((tag, num_calls, start, end))

    def collect(self) -> None:
        for tag, num_calls, start, end in self._pending:
            end.synchronize()
            seconds = start.elapsed_time(end) / 1000.0
            self.execution_times[tag].extend([seconds / num_calls] * num_calls)
        self._pending.clear()

    def dump(self, path: Path) -> None:
        self.collect()
        path.parent.mkdir(exist_ok=True, parents=True)
        path.write_text(json.dumps(dict(self.execution_times)))

    @staticmethod
    def dump_memory(path: Path, device=None) -> None:
        path.parent.mkdir(exist_ok=True, parents=True)
        path.write_text(json.dumps(torch.cuda.memory_stats(device)["allocated_bytes.all.peak"]))


@dataclass
class SceneResult:
    scene: str
    context_index: list[int]
    target_index: list[int]
    metrics: dict[str, float]            # the scene's mean of each metric over its targets
    per_view: dict[str, Tensor]          # float32 [v] per metric
    frames: Optional[Tensor] = None      # uint8 [v, h, w, 3] on the device, the bytes written as PNGs


@dataclass
class EvaluationResult:
    mean: dict[str, float]               # the mean over scenes
    scenes: list[SceneResult] = field(default_factory=list)


def mean_over_scenes(per_scene: Iterable[dict[str, float]]) -> dict[str, float]:
    """Each key's mean over the scenes (Lightning's epoch mean of a per-step log_dict at batch size 1)."""
    per_scene = list(per_scene)
    if not per_scene:
        return {}
    return {k: sum(s[k] for s in per_scene) / len(per_scene) for k in per_scene[0]}


class Evaluator:
    """Runs `encoder` (an EncoderEpipolar with its weights loaded) and `decoder` (DecoderSplattingCUDA) over a test
    split.  `lpips` is an `Lpips` module (default: `Lpips.from_files()`); `output_path` None writes no file."""

    def __init__(self, encoder: nn.Module, decoder: nn.Module, output_path: Path | str | None = None,
                 lpips: nn.Module | None = None, deterministic: bool = False, global_step: int = 0,
                 write_frames: bool = True) -> None:
        self.encoder = encoder
        self.decoder = decoder
        self.output_path = None if output_path is None else Path(output_path)
        self.lpips = lpips
        self.deterministic = deterministic
        self.global_step = global_step
        self.write_frames = write_frames
        self.data_shim = encoder.get_data_shim()
        self.benchmarker = Benchmarker()

    @torch.no_grad()
    def test_step(self, batch: dict) -> SceneResult:
        """One scene of a device-resident test batch (what `device_shim` returns): render, quantise, score and
        optionally write its frames."""
        shape_in = tuple(batch["target"]["image"].shape)
        batch = self.data_shim(batch)
        b, v, _, h, w = batch["target"]["image"].shape
        assert b == 1
        if tuple(batch["target"]["image"].shape) != shape_in:
            raise ValueError(f"Evaluator: the data shim changed the targets from {shape_in} to "
                             f"{tuple(batch['target']['image'].shape)}; the reference's metric computer scores the "
                             "un-shimmed targets, so its numbers would differ. Use an image shape the shim keeps "
                             "(a multiple of 16, such as 256 x 256)")
        tgt = batch["target"]
        with self.benchmarker.time("encoder"):
            gaussians = self.encoder(batch["context"], self.global_step, deterministic=self.deterministic)
        with self.benchmarker.time("decoder", num_calls=v):
            color = torch.cat([self.decoder.forward(gaussians, tgt["extrinsics"][:1, i:i + CHUNK],
                                                    tgt["intrinsics"][:1, i:i + CHUNK], tgt["near"][:1, i:i + CHUNK],
                                                    tgt["far"][:1, i:i + CHUNK], (h, w)).color
                               for i in range(0, v, CHUNK)], dim=1)
        per_view = frame_metrics_chunked(tgt["image"][0], color[0], self.lpips, return_frames=True)
        frames = per_view.pop("frames")
        (scene,) = batch["scene"]
        result = SceneResult(scene, [int(i) for i in batch["context"]["index"][0]], [int(i) for i in tgt["index"][0]],
                             {k: float(per_view[k].mean()) for k in METRICS}, per_view, frames)
        if self.output_path is not None and self.write_frames:
            root = self.output_path / scene
            for index, frame in zip(result.target_index, frames.cpu().numpy()):
                save_frame(frame, root / "color" / f"{index:0>6}.png")
            for index, frame in zip(result.context_index, quantise(batch["context"]["image"][0]).cpu().numpy()):
                save_frame(frame, root / "context" / f"{index:0>6}.png")
        self.benchmarker.collect()
        return result

    def run(self, loader: Iterable[dict], image_shape: tuple[int, int] = (256, 256), seed: int = 111123,
            device: torch.device | str | None = None, keep_frames: bool = False, log=print) -> EvaluationResult:
        """Every batch of a test DataLoader (batch size 1) through `device_shim` and `test_step`, with torch's RNG
        seeded with `seed` first.  Returns the mean over scenes and the per-scene results (frames dropped unless
        `keep_frames`); writes `benchmark.json` and `peak_memory.json` under the output path, if any."""
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        torch.manual_seed(seed)
        torch.cuda.reset_peak_memory_stats(device)
        scenes = []
        for i, batch in enumerate(loader):
            if i % 100 == 0 and log is not None:
                log(f"Test step {i:0>6}.")
            r = self.test_step(device_shim(batch, image_shape, device))
            if not keep_frames:
                r.frames = None
            scenes.append(r)
        result = EvaluationResult(mean_over_scenes(s.metrics for s in scenes), scenes)
        if self.output_path is not None:
            self.benchmarker.dump(self.output_path / "benchmark.json")
            self.benchmarker.dump_memory(self.output_path / "peak_memory.json", device)
        return result
