"""Command line of the training.

    python -m pixelsplat_b200.training --dataset-root datasets/re10k --preset re10k --output outputs/train/re10k

trains the preset's model on the dataset's train split as the reference's `python -m src.main +experiment=re10k`
does, writes `<output>/checkpoints/epoch=E-step=N.ckpt` (Lightning's layout: `python -m pixelsplat_b200.evaluation
--checkpoint` reads them) and one JSON line per `--log-every` steps to stdout and `<output>/log.jsonl`.

`--val-every 250` adds the reference's validation (its `val_check_interval` is 250; the default 0 trains without
it): on rank 0, before the first step and after every 250th, one scene of the test split encoded probabilistically
and deterministically, scored with the float PSNR / SSIM / LPIPS of its renders (`<output>/validation.jsonl`) and
drawn as context | ground truth | probabilistic | deterministic (`<output>/validation/comparison_{step:0>6}.png`).
It needs `<dataset-root>/test/` and the LPIPS weights.  Validation draws from its own seeded generators, so the
training's numbers are the same with it on or off.  `--val-videos` adds the reference's validation videos to each
validation: `<output>/validation/video/rgb/{step:0>6}.mp4` and, with two context views, `.../wobble/...`.

On several GPUs, one process per GPU:

    python -m torch.distributed.run --nproc-per-node 8 -m pixelsplat_b200.training ...

Nothing is downloaded.  `--backbone-weights VIT.pth RESNET.pth` starts the backbone from DINO's released files;
without it the whole encoder starts from a random initialisation.  LPIPS reads torchvision's VGG16 file and the lpips
package's lin weights from disk (`--lpips-vgg` / `--lpips-lin`, or where those packages keep them).
"""
from __future__ import annotations

import argparse
import os
import sys
from pathlib import Path

import torch


def _non_negative(text: str) -> int:
    value = int(text)
    if value < 0:
        raise argparse.ArgumentTypeError(f"expected a step count >= 0, got {value}")
    return value


def parse(argv: list[str]) -> argparse.Namespace:
    from .presets import PRESETS, VAL_EVERY
    p = argparse.ArgumentParser(prog="python -m pixelsplat_b200.training",
                                description="Train pixelSplat on RE10k / ACID chunks.")
    p.add_argument("--dataset-root", type=Path, required=True, help="dataset root holding train/index.json")
    p.add_argument("--preset", choices=PRESETS, default="re10k")
    p.add_argument("--output", type=Path, required=True, help="where checkpoints/ and log.jsonl go")
    p.add_argument("--batch-size", type=int, default=None, help="scenes per GPU (default: the preset's batch size)")
    p.add_argument("--max-steps", type=int, default=None, help="default: the preset's")
    p.add_argument("--checkpoint-every", type=int, default=None, help="steps (default: the preset's 5000)")
    p.add_argument("--log-every", type=int, default=10)
    p.add_argument("--val-every", type=_non_negative, default=0, metavar="N",
                   help=f"validate on one scene of <dataset-root>/test before the first step and every N steps (the "
                        f"reference's val_check_interval is {VAL_EVERY}); writes <output>/validation.jsonl and "
                        f"<output>/validation/*.png.  0 (default): no validation")
    p.add_argument("--val-videos", action="store_true",
                   help="with --val-every: also render the rgb and wobble videos of each validation scene to "
                        "<output>/validation/video/{rgb,wobble}/{step:0>6}.mp4")
    p.add_argument("--resume", type=Path, default=None, help="a checkpoint of this command or of the reference")
    p.add_argument("--backbone-weights", type=Path, nargs=2, default=None, metavar=("VIT", "RESNET"),
                   help="DINO's released ViT and ResNet-50 files")
    p.add_argument("--lpips-vgg", type=Path, default=None, help="torchvision's vgg16-397923af.pth")
    p.add_argument("--lpips-lin", type=Path, default=None, help="the lpips package's weights/v0.1/vgg.pth")
    p.add_argument("--num-workers", type=int, default=None, help="DataLoader workers (default: the preset's 16)")
    p.add_argument("--overfit-to-scene", type=str, default=None, help="train on this one scene only")
    p.add_argument("--deterministic", action="store_true",
                   help="torch.use_deterministic_algorithms(True, warn_only=True): every kernel of this package and "
                        "the optimiser sum in a fixed order; torch warns about the one op left without a "
                        "deterministic backward, the backbone's F.interpolate")
    args = p.parse_args(argv)
    if args.val_videos and args.val_every == 0:
        p.error("--val-videos renders the videos of each validation; it needs --val-every N > 0")
    return args


def _worker_init_fn(worker_id: int) -> None:
    import random

    import numpy as np
    seed = int(torch.utils.data.get_worker_info().seed) % (2 ** 32 - 1)
    random.seed(seed)
    np.random.seed(seed)


def main(argv: list[str] | None = None) -> list[dict]:
    args = parse(sys.argv[1:] if argv is None else argv)
    validating = args.val_every > 0
    if validating and not (args.dataset_root / "test").is_dir():
        raise SystemExit(f"training: --val-every {args.val_every} validates on {args.dataset_root / 'test'}, which is "
                         "not a directory; pass --val-every 0 to train without validation")
    if args.deterministic:                         # cuBLAS needs its workspace setting before its first call
        os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
        torch.use_deterministic_algorithms(True, warn_only=True)
    from .. import parallel
    from ..data import StepTracker
    from ..encoder.backbone import BackboneDino
    from ..evaluation.presets import build_model
    from . import presets
    from .trainer import Trainer

    rank, world, local = parallel.init_distributed()
    device = torch.device("cuda", local)
    torch.cuda.set_device(device)
    preset = presets.train_preset(args.preset)
    torch.manual_seed(presets.SEED + rank)
    cfg = presets.dataset_cfg(preset, args.dataset_root, args.overfit_to_scene)
    encoder, decoder = build_model(preset.model, cfg)
    say = print if rank == 0 else (lambda *a, **k: None)
    if args.backbone_weights is not None:
        encoder.backbone = BackboneDino.from_files(encoder.cfg.backbone, 3, *args.backbone_weights)
        say(f"Backbone weights from {args.backbone_weights[0]} and {args.backbone_weights[1]}.")
    elif args.resume is None:
        say("No --backbone-weights: the encoder, backbone included, starts from a random initialisation.")
    lpips = None
    if "lpips" in preset.losses:
        from ..lpips import Lpips
        lpips = Lpips.from_files(args.lpips_vgg, args.lpips_lin)
    elif validating:
        from ..lpips import Lpips
        try:
            with torch.random.fork_rng(devices=[]):       # building the module draws its initial weights
                lpips = Lpips.from_files(args.lpips_vgg, args.lpips_lin)
        except Exception as e:
            raise SystemExit(f"training: --val-every {args.val_every} scores with LPIPS, whose weights cannot be "
                             f"read ({e}); pass --lpips-vgg and --lpips-lin, or --val-every 0 to train without "
                             "validation") from e
    step_tracker = StepTracker()
    trainer = Trainer(encoder.to(device), decoder.to(device), presets.make_losses(preset, lpips),
                      depth_mode=preset.depth_mode, lr=preset.lr, warm_up_steps=preset.warm_up_steps,
                      max_norm=preset.max_norm, step_tracker=step_tracker, image_shape=tuple(cfg.image_shape),
                      lpips=lpips)
    if args.resume is not None:
        trainer.resume(args.resume)
        say(f"Resumed {args.resume} at step {trainer.global_step}, lr {trainer.optimizer.lr():.3e}.")
    workers = preset.num_workers if args.num_workers is None else args.num_workers
    loader = torch.utils.data.DataLoader(
        presets.make_train_dataset(cfg, step_tracker), args.batch_size or preset.batch_size, num_workers=workers,
        generator=torch.Generator().manual_seed(presets.LOADER_SEED + rank), worker_init_fn=_worker_init_fn,
        persistent_workers=workers > 0, pin_memory=True)
    validation = None
    if validating and rank == 0:
        val_workers = min(1, workers)
        validation = torch.utils.data.DataLoader(
            presets.make_val_dataset(cfg, step_tracker), 1, num_workers=val_workers,
            generator=torch.Generator().manual_seed(presets.VAL_SEED + rank), worker_init_fn=_worker_init_fn,
            persistent_workers=val_workers > 0, pin_memory=True)
    try:
        return trainer.fit(loader, preset.max_steps if args.max_steps is None else args.max_steps, args.output,
                           preset.checkpoint_every if args.checkpoint_every is None else args.checkpoint_every,
                           args.log_every, log=say, validation=validation, val_every=args.val_every,
                           val_videos=args.val_videos)
    finally:
        if args.deterministic:
            torch.use_deterministic_algorithms(False)
        if world > 1 and torch.distributed.is_initialized():
            torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
