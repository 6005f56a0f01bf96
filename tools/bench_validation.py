#!/usr/bin/env python
"""Times the training's validation step against the training step it interrupts, CUDA events, median per call:
  shared    `Trainer.validation_step` as it runs: the encoder's trunk (backbone, projection, epipolar transformer)
            once, the tail and the render twice (probabilistic, deterministic), the float PSNR / SSIM / LPIPS of both,
            on one seeded synthetic scene at 256 x 256 with 2 context views and 4 targets (the bounded sampler's
            shape), the re10k preset encoder with random weights and LPIPS with seeded weights (the times do not
            depend on the weights);
  two-pass  the same step with two full encoder passes (the reference's route) on the same scene;
  train     one `Trainer.training_step` of the re10k preset (MSE + LPIPS, LPIPS inactive before step 150 000 as
            at the start of a run) at batch 7, 4 targets per scene.
The three are measured in alternation in one process.  Reports the trunk's saving and the validation's share of
the training time at --val-every 250 (one validation per 250 steps), with the card and its power limit, as one JSON
line.  Nothing is written.

    python tools/bench_validation.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import lpips_oracle as lo  # noqa: E402
from pixelsplat_b200 import synthetic  # noqa: E402
from pixelsplat_b200.evaluation.presets import build_model  # noqa: E402
from pixelsplat_b200.loss import compute_psnr, compute_ssim  # noqa: E402
from pixelsplat_b200.lpips import Lpips  # noqa: E402
from pixelsplat_b200.training import Trainer  # noqa: E402
from pixelsplat_b200.training import presets as tp  # noqa: E402
from pixelsplat_b200.training.trainer import VAL_PHASES, validation_rng  # noqa: E402
from tools.bench_depth import gpu_identity  # noqa: E402

DEV = torch.device("cuda", 0)
SHAPE = (256, 256)
TARGETS = 4


def batch(scenes: int, seed: int) -> dict:
    """A device-resident batch as `device_shim` returns it: 2 context views one unit apart, TARGETS target cameras
    around them, uniform random images.  near / far are replaced by the encoder's bounds shim."""
    g = torch.Generator().manual_seed(seed)
    ctx_e = torch.eye(4).repeat(scenes, 2, 1, 1)
    ctx_e[:, 1, 0, 3] = 1.0
    tgt_e = torch.stack([synthetic.target_cameras(TARGETS, seed=seed * 100 + s) for s in range(scenes)])

    def views(extrinsics, n):
        intrinsics = synthetic.intrinsics_re10k(n)[None].repeat(scenes, 1, 1, 1)
        return {"extrinsics": extrinsics.to(DEV), "intrinsics": intrinsics.to(DEV),
                "near": torch.full((scenes, n), 1.0, device=DEV), "far": torch.full((scenes, n), 100.0, device=DEV),
                "index": torch.arange(n).repeat(scenes, 1).to(DEV),
                "image": torch.rand(scenes, n, 3, *SHAPE, generator=g).to(DEV)}
    return {"context": views(ctx_e, 2), "target": views(tgt_e, TARGETS),
            "scene": [f"synthetic{s}" for s in range(scenes)]}


def events(n: int) -> list:
    return [torch.cuda.Event(enable_timing=True) for _ in range(n)]


def two_pass(t: Trainer, b: dict) -> list:
    """The reference's validation step: two full encoder passes, each rendered, then the same six metrics."""
    ev = events(4)
    with torch.no_grad(), validation_rng(0, t.global_step, DEV):
        t.encoder.eval()
        ev[0].record()
        b = t.data_shim(b)
        ctx, tgt = b["context"], b["target"]
        gt, color = tgt["image"][0], []
        for i, deterministic in enumerate((False, True)):
            gaussians = t.encoder(ctx, t.global_step, deterministic=deterministic)
            color.append(t.decoder.forward(gaussians, tgt["extrinsics"], tgt["intrinsics"], tgt["near"], tgt["far"],
                                           SHAPE).color[0])
            ev[1 + i].record()
        values = []
        for c in color:
            values += [compute_psnr(gt, c).mean(), compute_ssim(gt, c).mean(),
                       t.lpips(gt, c, normalize=True)[:, 0, 0, 0].mean()]
        torch.stack(values).tolist()
        ev[3].record()
    ev[3].synchronize()
    return ev


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--train-batch", type=int, default=7)
    ap.add_argument("--val-every", type=int, default=tp.VAL_EVERY)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_validation: no CUDA device; the times need an H100")
    torch.cuda.set_device(DEV)
    torch.manual_seed(0)
    preset = tp.train_preset("re10k")
    encoder, decoder = build_model(preset.model, tp.dataset_cfg(preset, "/nonexistent"))
    lpips = Lpips()
    lpips.load_state_dict(lo.random_state_dict(0))
    t = Trainer(encoder.to(DEV), decoder.to(DEV), tp.make_losses(preset, lpips), lr=preset.lr,
                warm_up_steps=preset.warm_up_steps, max_norm=preset.max_norm)
    val_batch, train_batch = batch(1, 1), batch(args.train_batch, 2)

    shared, twopass, train = [], [], []
    for i in range(args.warmup + args.steps):
        r = t.validation_step(val_batch)
        ev = two_pass(t, val_batch)
        t.training_step(train_batch)
        line = t.read_last()
        if i >= args.warmup:
            shared.append({"total": r["ms"], **r["phase_ms"]})
            twopass.append({"total": ev[0].elapsed_time(ev[3]),
                            "encoder_render_probabilistic": ev[0].elapsed_time(ev[1]),
                            "encoder_render_deterministic": ev[1].elapsed_time(ev[2]),
                            "metrics": ev[2].elapsed_time(ev[3])})
            train.append(sum(line["phase_ms"].values()))
    med = lambda rows, k: statistics.median(row[k] for row in rows)
    res = {f"shared_{k}_ms": med(shared, k) for k in ("total", *VAL_PHASES)}
    res.update({f"two_pass_{k}_ms": med(twopass, k) for k in twopass[0]})
    res[f"train_step_batch{args.train_batch}_ms"] = train_ms = statistics.median(train)
    res["trunk_saving_ms"] = res["two_pass_total_ms"] - res["shared_total_ms"]
    for name in ("shared", "two_pass"):
        val_ms = res[f"{name}_total_ms"]
        res[f"{name}_overhead_at_val_every_{args.val_every}_pct"] = 100 * val_ms / (args.val_every * train_ms)
    res.update({"steps": args.steps, "warmup": args.warmup, **gpu_identity(0)})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
