"""Command line of the evaluation.

    python -m pixelsplat_b200.evaluation --dataset-root datasets/re10k --index assets/evaluation_index_re10k.json \\
        --checkpoint checkpoints/re10k.ckpt --preset re10k --output outputs/test/re10k

runs the reference's test step over the test split: it prints the PSNR / SSIM / LPIPS table of the 8-bit frames
(the paper's numbers) and, with --output, writes the frames (unless --no-frames), benchmark.json,
peak_memory.json and metrics.json (the mean and each scene's metrics).

    python -m pixelsplat_b200.evaluation compute-metrics --dataset-root datasets/re10k \\
        --index assets/evaluation_index_re10k.json --method pixelSplat:ours:outputs/test/re10k \\
        --output-metrics outputs/metrics.json

is the reference's compute_metrics script: it scores saved frame directories of one or more methods.

Nothing is downloaded: the checkpoint holds every encoder weight, and LPIPS reads torchvision's VGG16 file and the
lpips package's lin weights from disk (--lpips-vgg / --lpips-lin, or where those packages keep them).
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch


def _common(p: argparse.ArgumentParser) -> None:
    p.add_argument("--dataset-root", type=Path, required=True, help="dataset root holding test/index.json")
    p.add_argument("--index", type=Path, required=True, help="evaluation index (scene -> context / target)")
    p.add_argument("--seed", type=int, default=None, help="torch seed (default: the reference's 111123)")
    p.add_argument("--num-workers", type=int, default=4, help="DataLoader workers (the reference's test loader: 4)")
    p.add_argument("--lpips-vgg", type=Path, default=None, help="torchvision's vgg16-397923af.pth")
    p.add_argument("--lpips-lin", type=Path, default=None, help="the lpips package's weights/v0.1/vgg.pth")


def _loader(args):
    from .presets import dataset_cfg, make_test_dataset
    cfg = dataset_cfg(args.dataset_root, args.index)
    return cfg, torch.utils.data.DataLoader(make_test_dataset(cfg), batch_size=1, num_workers=args.num_workers,
                                            pin_memory=True)


def _lpips(args, device):
    from ..lpips import Lpips
    return Lpips.from_files(args.lpips_vgg, args.lpips_lin).to(device).eval()


def evaluate(argv: list[str]) -> dict:
    p = argparse.ArgumentParser(prog="python -m pixelsplat_b200.evaluation",
                                description="Evaluate a pixelSplat checkpoint on the RE10k / ACID test split.")
    _common(p)
    p.add_argument("--checkpoint", type=Path, required=True, help="a pixelSplat Lightning checkpoint (.ckpt)")
    p.add_argument("--preset", choices=("re10k", "acid"), default="re10k")
    p.add_argument("--output", type=Path, default=None, help="where frames and the JSON files go")
    p.add_argument("--deterministic", action="store_true",
                   help="the encoder picks each ray's most likely depth instead of sampling one")
    p.add_argument("--no-frames", action="store_true", help="write no PNG (metrics and JSON files only)")
    p.add_argument("--global-step", type=int, default=0,
                   help="step given to the encoder (the presets' opacity mapping does not depend on it)")
    args = p.parse_args(argv)

    from .checkpoint import load_checkpoint
    from .evaluator import Evaluator
    from .presets import SEED, build_model
    device = torch.device("cuda", torch.cuda.current_device())
    cfg, loader = _loader(args)
    encoder, decoder = build_model(args.preset, cfg)
    step = load_checkpoint(args.checkpoint, encoder)
    print(f"Loaded {args.checkpoint} (trained for {step} steps).")
    evaluator = Evaluator(encoder.to(device).eval(), decoder.to(device), args.output, _lpips(args, device),
                          deterministic=args.deterministic, global_step=args.global_step,
                          write_frames=not args.no_frames)
    result = evaluator.run(loader, seed=SEED if args.seed is None else args.seed, device=device)
    print(f"{len(result.scenes)} scenes: " + ", ".join(f"{k} {v:.4f}" for k, v in result.mean.items()))
    out = {"mean": result.mean, "scenes": {s.scene: s.metrics for s in result.scenes}}
    if args.output is not None:
        (args.output / "metrics.json").write_text(json.dumps(out))
    return out


def compute_metrics(argv: list[str]) -> dict:
    p = argparse.ArgumentParser(prog="python -m pixelsplat_b200.evaluation compute-metrics",
                                description="Score saved frame directories against the test split.")
    _common(p)
    p.add_argument("--method", action="append", required=True, metavar="NAME:KEY:PATH",
                   help="a method's display name, metric key and frame directory (repeatable)")
    p.add_argument("--output-metrics", type=Path, default=None, help="JSON file for the mean metrics")
    args = p.parse_args(argv)

    from .metric_computer import Method, compute_metrics as run
    from .presets import SEED
    methods = []
    for spec in args.method:
        parts = spec.split(":", 2)
        if len(parts) != 3:
            p.error(f"--method {spec!r}: expected NAME:KEY:PATH")
        methods.append(Method(parts[0], parts[1], Path(parts[2])))
    device = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(SEED if args.seed is None else args.seed)
    _, loader = _loader(args)
    result = run(methods, loader, _lpips(args, device), output_path=args.output_metrics, device=device)
    return result.mean


def main(argv: list[str] | None = None) -> None:
    argv = sys.argv[1:] if argv is None else argv
    if argv and argv[0] == "compute-metrics":
        compute_metrics(argv[1:])
    else:
        evaluate(argv)


if __name__ == "__main__":
    main()
