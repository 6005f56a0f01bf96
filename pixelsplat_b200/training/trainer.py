"""The reference's training loop (ModelWrapper.training_step and configure_optimizers, src/model/model_wrapper.py, and
the Trainer set-up of src/main.py) without Lightning: one process per GPU, gradients averaged by
`parallel.GradientReducer`, clipping + Adam + warm-up by `optim.ClipAdam`.

A step:
    data shim -> encoder(batch["context"], global_step, False) -> decoder (depth_mode) -> losses, train PSNR
    reducer.zero_grad() / loss.backward() / reducer.finish() / optimizer.step()
    step_tracker.set_step(global_step)   (the bounded view sampler's warm-up reads it in the loader's workers)

With the loss list [mse] or [mse, depth] the MSE and the PSNR come from the compositor's fused epilogue
(`DecoderSplattingCUDA.forward_mse`, no image tensor); with LPIPS in the list the image is rendered.

The host reads device values in one place only, a log line; between log lines a step enqueues work and returns.

Validation (ModelWrapper.validation_step, run by Lightning every `val_check_interval` steps and once before the first
step): on rank 0, one held-out scene encoded twice, probabilistic and deterministic, rendered, scored with the float
PSNR / SSIM / LPIPS, and drawn as the reference's comparison image.  Its random numbers come from generators seeded
from (VAL_SEED + rank, global_step) inside `torch.random.fork_rng`, so the training stream is the same with
validation on or off, and a resumed run still continues the uninterrupted one bit for bit.
"""
from __future__ import annotations

import contextlib
import json
import time
from pathlib import Path
from typing import Iterable, Sequence

import torch
import torch.distributed as dist
from torch import Tensor, nn

from ..data import StepTracker, device_shim
from ..encoder.encoder_tail import EncoderEpipolarTail
from ..evaluation.checkpoint import load_checkpoint, read_checkpoint, save_checkpoint
from ..evaluation.image_io import comparison_layout, save_image
from ..loss import compute_psnr, compute_ssim, psnr_from_sse
from ..optim import ClipAdam
from ..parallel import GradientReducer, env_rank_world
from ..video import VALIDATION_VIDEOS, render_video, write_mp4
from .presets import VAL_SEED

PHASES = ("forward", "backward", "allreduce", "optimizer")
VAL_PHASES = ("trunk", "tail_probabilistic", "render_probabilistic", "tail_deterministic", "render_deterministic",
              "metrics")
VAL_TAGS = ("probabilistic", "deterministic")
VAL_METRICS = tuple(f"{m}_{tag}" for tag in VAL_TAGS for m in ("psnr", "ssim", "lpips"))


@contextlib.contextmanager
def validation_rng(rank: int, global_step: int, device: torch.device | None = None):
    """Forks torch's CPU generator and, when given, `device`'s generator, and seeds both from (VAL_SEED + rank,
    global_step); on exit both are back where they were.  No other generator is touched."""
    with torch.random.fork_rng(devices=[] if device is None else [device]):
        seed = ((VAL_SEED + rank) << 32) + global_step
        torch.default_generator.manual_seed(seed)
        if device is not None:
            with torch.cuda.device(device):
                torch.cuda.manual_seed(seed)
        yield


def _module_modes(modules: Sequence[nn.Module]) -> list[tuple[nn.Module, bool]]:
    return [(m, m.training) for module in modules for m in module.modules()]


class Trainer:
    """`encoder` and `decoder` on their CUDA device, `losses` the reference's loss modules (LossMse, LossLpips,
    LossDepth) in order.  `fused_mse` None picks the fused epilogue whenever the loss list allows it.  `lpips` is the
    `Lpips` module the validation step scores with (default: the LossLpips loss's module, when the list has one)."""

    def __init__(self, encoder: nn.Module, decoder: nn.Module, losses: Sequence[nn.Module],
                 depth_mode: str | None = None, lr: float = 1.5e-4, warm_up_steps: int = 2000,
                 max_norm: float = 0.5, step_tracker: StepTracker | None = None,
                 image_shape: tuple[int, int] = (256, 256), fused_mse: bool | None = None,
                 bucket_bytes: int = 8 << 20, lpips: nn.Module | None = None) -> None:
        self.encoder, self.decoder, self.losses = encoder, decoder, nn.ModuleList(losses)
        self.depth_mode, self.step_tracker, self.image_shape = depth_mode, step_tracker, tuple(image_shape)
        self.device = next(encoder.parameters()).device
        self.losses.to(self.device)
        if lpips is None:
            lpips = next((l.lpips for l in self.losses if l.name == "lpips"), None)
        self.lpips = None if lpips is None else lpips.to(self.device)
        self.rank, self.world, _ = env_rank_world()
        names = [l.name for l in self.losses]
        can_fuse = names in (["mse"], ["mse", "depth"])
        if fused_mse and not can_fuse:
            raise ValueError(f"Trainer: the fused MSE epilogue serves the loss lists [mse] and [mse, depth], not {names}")
        self.fused_mse = can_fuse if fused_mse is None else fused_mse
        if "depth" in names and depth_mode is None:
            raise ValueError("Trainer: LossDepth needs a depth_mode")
        if self.world > 1 and dist.is_initialized():      # one set of initial weights, rank 0's (as DDP does)
            for t in encoder.state_dict().values():
                dist.broadcast(t, src=0)
        self.data_shim = encoder.get_data_shim()
        params = list(encoder.parameters())
        self.reducer = GradientReducer(params, bucket_bytes)
        self.optimizer = ClipAdam(params, self.reducer, lr=lr, warm_up_steps=warm_up_steps, max_norm=max_norm)
        self.global_step = 0
        self.epoch = 0
        self._last = None                    # the last step's device scalars and phase events

    # ---- one step ---------------------------------------------------------------------------------------------
    def training_step(self, batch: dict) -> dict:
        """One optimisation step on a device-resident batch (what `device_shim` returns).  Returns the step's device
        scalars (each loss, `total`, `psnr`, `grad_norm`) without reading them."""
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(PHASES) + 1)]
        ev[0].record()
        batch = self.data_shim(batch)
        tgt = batch["target"]
        h, w = tgt["image"].shape[-2:]
        self.encoder.train()
        self.losses.train()
        self.reducer.zero_grad()
        gaussians = self.encoder(batch["context"], self.global_step, False)
        args = (gaussians, tgt["extrinsics"], tgt["intrinsics"], tgt["near"], tgt["far"], (h, w))
        values = {}
        if self.fused_mse:
            output, sse, sse_clipped = self.decoder.forward_mse(*args, tgt["image"], want_color=False,
                                                                depth_mode=self.depth_mode)
            psnr = psnr_from_sse(sse_clipped, (h, w)).mean()
        else:
            output = self.decoder.forward(*args, depth_mode=self.depth_mode)
            psnr = compute_psnr(tgt["image"].flatten(0, 1), output.color.flatten(0, 1)).mean()
        total = 0
        for loss_fn in self.losses:
            if self.fused_mse and loss_fn.name == "mse":
                loss = loss_fn.from_sse(sse, (h, w))
            else:
                loss = loss_fn(output, batch, gaussians, self.global_step)
            values[loss_fn.name] = loss.detach()
            total = total + loss
        ev[1].record()
        total.backward()
        ev[2].record()
        self.reducer.finish()
        ev[3].record()
        self.optimizer.step()
        ev[4].record()
        values.update(total=total.detach(), psnr=psnr, grad_norm=self.optimizer.grad_norm)
        if self.step_tracker is not None:
            self.step_tracker.set_step(self.global_step)
        self.global_step += 1
        self._last = (values, ev)
        return values

    def read_last(self) -> dict:
        """The last step's values on the host (one synchronising copy) and its phase times in milliseconds."""
        values, ev = self._last
        keys = list(values)
        # grad_norm is overwritten by the next step; it is read here, before one is enqueued
        host = torch.stack([values[k].float().reshape(()) for k in keys]).tolist()
        out = dict(zip(keys, host))
        out["phase_ms"] = {p: ev[i].elapsed_time(ev[i + 1]) for i, p in enumerate(PHASES)}
        return out

    # ---- validation -------------------------------------------------------------------------------------------
    def validation_step(self, batch: dict, videos: Sequence[str] = ()) -> dict:
        """The reference's validation step on a device-resident batch of one scene (what `device_shim` returns): the
        data shim, then the encoder's trunk once and its tail twice, probabilistic and then deterministic (the
        reference's order; with two context views the trunk draws no random numbers, so the draws are the ones two
        full encoder passes make; with three it draws the view embeddings' permutation once and both tails see it),
        each encoding rendered at the targets.  Runs without autograd, with the encoder, the losses and the LPIPS
        module in eval mode (BatchNorm reads its running statistics and does not update them), and restores their
        modes afterwards; inside `validation_rng`, so the training's generators do not move.

        The metrics are the means over the targets of `compute_psnr`, `compute_ssim` and LPIPS of the float renders,
        as the reference logs them, not of 8-bit frames as the evaluator scores them.  Returns `step`, `scene`,
        `context_index`, the six metrics (`psnr_probabilistic`, ..., `lpips_deterministic`) as host floats, `ms` and
        `phase_ms` (CUDA events), and `images`: the shimmed `context` and `target` views and the two renders, each
        [v, 3, h, w] on the device.

        `videos` names videos of `pixelsplat_b200.video` to render afterwards from the same trunk and in the same
        generators, as the reference's validation step does: `videos` in the result maps each name to uint8 frames
        [T, H, W, 3] on the host, leaving out those the number of context views rules out."""
        if self.lpips is None:
            raise ValueError("Trainer.validation_step: no Lpips module to score with; pass lpips= or train with "
                             "LossLpips")
        modes = _module_modes([self.encoder, self.losses, self.lpips])
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(VAL_PHASES) + 1)]
        try:
            with torch.no_grad(), validation_rng(self.rank, self.global_step, self.device):
                self.encoder.eval()
                self.losses.eval()
                self.lpips.eval()
                ev[0].record()
                batch = self.data_shim(batch)
                ctx, tgt = batch["context"], batch["target"]
                b, _, _, h, w = tgt["image"].shape
                if b != 1:
                    raise ValueError(f"Trainer.validation_step: expected one scene, got a batch of {b}")
                features, _ = self.encoder.trunk(ctx)
                ev[1].record()
                color = {}
                for i, tag in enumerate(VAL_TAGS):
                    gaussians = EncoderEpipolarTail.forward(self.encoder, features, ctx, self.global_step,
                                                            tag == "deterministic")
                    ev[2 + 2 * i].record()
                    color[tag] = self.decoder.forward(gaussians, tgt["extrinsics"], tgt["intrinsics"], tgt["near"],
                                                      tgt["far"], (h, w)).color[0]
                    ev[3 + 2 * i].record()
                gt = tgt["image"][0]
                values = []
                for tag in VAL_TAGS:
                    values += [compute_psnr(gt, color[tag]).mean(), compute_ssim(gt, color[tag]).mean(),
                               self.lpips(gt, color[tag], normalize=True)[:, 0, 0, 0].mean()]
                ev[-1].record()
                host = torch.stack([v.float() for v in values]).tolist()
                rendered = {}
                for name in videos:
                    frames = render_video(self.encoder, self.decoder, ctx, tgt, name, self.global_step, features)
                    if frames is not None:
                        rendered[name] = frames
        finally:
            for m, mode in modes:
                m.training = mode
        (scene,) = batch["scene"]
        out = {"step": self.global_step, "scene": scene, "context_index": [int(i) for i in ctx["index"][0]],
               **dict(zip(VAL_METRICS, host)), "ms": ev[0].elapsed_time(ev[-1]),
               "phase_ms": {p: ev[i].elapsed_time(ev[i + 1]) for i, p in enumerate(VAL_PHASES)}}
        out["images"] = {"context": ctx["image"][0], "target": gt, **color}
        if videos:
            out["videos"] = rendered
        return out

    # ---- checkpoints ------------------------------------------------------------------------------------------
    def save(self, path: Path | str) -> Path:
        rng = {"torch": torch.get_rng_state(), "cuda": torch.cuda.get_rng_state(self.device)}
        return save_checkpoint(path, self.encoder, self.global_step, self.epoch, self.optimizer.state_dict(),
                               self.optimizer.scheduler_state_dict(), rng)

    def resume(self, path: Path | str) -> None:
        """Weights, optimiser state (moments, step, learning rate), the step counter, the step tracker and, when the
        checkpoint holds them, torch's CPU and CUDA generator states.  The data loader's position is not restored
        (an iterable dataset has none to restore; Lightning does not either)."""
        self.global_step = load_checkpoint(path, self.encoder)
        ckpt = read_checkpoint(path)
        self.epoch = int(ckpt.get("epoch", 0))
        if not ckpt.get("optimizer_states"):
            raise ValueError(f"Trainer.resume: {path} holds no optimiser state")
        self.optimizer.load_state_dict(ckpt["optimizer_states"][0])
        if self.optimizer.steps != self.global_step:
            raise ValueError(f"Trainer.resume: {path} is at step {self.global_step} but its optimiser at "
                             f"{self.optimizer.steps}")
        if self.step_tracker is not None:
            self.step_tracker.set_step(max(self.global_step - 1, 0))
        if "rng_state" in ckpt:
            torch.set_rng_state(ckpt["rng_state"]["torch"])
            torch.cuda.set_rng_state(ckpt["rng_state"]["cuda"], self.device)

    def checkpoint_path(self, output: Path) -> Path:
        return Path(output) / "checkpoints" / f"epoch={self.epoch}-step={self.global_step}.ckpt"

    # ---- the loop ---------------------------------------------------------------------------------------------
    def fit(self, batches: Iterable[dict], max_steps: int, output: Path | str | None = None,
            checkpoint_every: int = 5000, log_every: int = 10, log=print, validation: Iterable[dict] | None = None,
            val_every: int = 0, val_videos: bool = False) -> list[dict]:
        """Steps over `batches` (a DataLoader over DatasetRE10k, or any iterable of its batches; it is restarted when
        exhausted, which counts an epoch) until `global_step == max_steps`.  Rank 0 writes a checkpoint every
        `checkpoint_every` steps and at the end, and one JSON line per `log_every` steps to `log` and
        `<output>/log.jsonl`.  Returns the log lines.

        With `validation` (batches of one scene, e.g. a DataLoader over the stage-"val" DatasetRE10k) and
        `val_every > 0`, rank 0 also runs `validation_step` before the first step (Lightning's sanity check) and after
        every step whose index is a multiple of `val_every`, after that step's checkpoint.  Each draws the next batch
        of one iterator over `validation`, restarted when exhausted, and writes one JSON line to
        `<output>/validation.jsonl` and the comparison image to `<output>/validation/comparison_{step:0>6}.png`.
        With `val_videos`, each validation also renders the reference's validation videos (rgb, and wobble with two
        context views) and writes `<output>/validation/video/{name}/{step:0>6}.mp4`."""
        output = None if output is None else Path(output)
        lines, log_file = [], None
        if output is not None and self.rank == 0:
            output.mkdir(parents=True, exist_ok=True)
            log_file = (output / "log.jsonl").open("a")
        validating = validation is not None and val_every > 0 and self.rank == 0
        val_iter = None

        def validate() -> None:
            nonlocal val_iter
            with validation_rng(self.rank, self.global_step, self.device):   # a loader without workers draws here
                batch = None if val_iter is None else next(val_iter, None)
                if batch is None:
                    val_iter = iter(validation)
                    batch = next(val_iter, None)
            if batch is None:
                raise ValueError("training: the validation loader yielded no batch")
            batch = device_shim(batch, self.image_shape, self.device)
            result = self.validation_step(batch, VALIDATION_VIDEOS) if val_videos else self.validation_step(batch)
            line = {k: v for k, v in result.items() if k not in ("images", "phase_ms", "videos")}
            if log is not None:
                log(f"validation step {line['step']}; scene = {[line['scene']]}; context = {[line['context_index']]}")
                log(json.dumps(line))
            if output is not None:
                images = result["images"]
                save_image(comparison_layout(images["context"], images["target"], images["probabilistic"],
                                             images["deterministic"]),
                           output / "validation" / f"comparison_{line['step']:0>6}.png")
                with (output / "validation.jsonl").open("a") as f:
                    f.write(json.dumps(line) + "\n")
                for name, frames in result.get("videos", {}).items():
                    write_mp4(frames.numpy(), output / "validation" / "video" / name / f"{line['step']:0>6}.mp4")

        try:
            if validating:
                validate()                                # Lightning's sanity check, on resume too
            scenes, t_last = 0, time.perf_counter()
            while self.global_step < max_steps:
                seen = 0
                for batch in batches:
                    seen += 1
                    batch = device_shim(batch, self.image_shape, self.device)
                    scenes += batch["target"]["image"].shape[0]
                    lr = self.optimizer.lr()
                    self.training_step(batch)
                    step = self.global_step
                    if step % log_every == 0 or step == max_steps:
                        line = {"step": step, "epoch": self.epoch, **self.read_last(), "lr": lr}
                        now = time.perf_counter()
                        line["scenes_per_s"] = self.world * scenes / (now - t_last)
                        scenes, t_last = 0, now
                        if not (line["total"] == line["total"] and abs(line["total"]) != float("inf")):
                            raise FloatingPointError(f"training: the total loss is {line['total']} at step {step}")
                        lines.append(line)
                        if self.rank == 0:
                            text = json.dumps(line)
                            if log is not None:
                                log(text)
                            if log_file is not None:
                                log_file.write(text + "\n")
                                log_file.flush()
                    if output is not None and self.rank == 0 and \
                            (step % checkpoint_every == 0 or step == max_steps):
                        self.save(self.checkpoint_path(output))
                    if validating and step % val_every == 0:
                        t_val = time.perf_counter()
                        validate()
                        t_last += time.perf_counter() - t_val     # scenes_per_s stays the training's rate
                    if step >= max_steps:
                        break
                if seen == 0:
                    raise ValueError("training: the data loader yielded no batch (the view sampler skips a scene with too few "
                                     "frames for its context gap)")
                if self.global_step < max_steps:
                    self.epoch += 1
        finally:
            if log_file is not None:
                log_file.close()
        return lines
