"""Command line of the evaluation.

    python -m pixelsplat_b200.evaluation --dataset-root datasets/re10k --index assets/evaluation_index_re10k.json \\
        --checkpoint checkpoints/re10k.ckpt --preset re10k --output outputs/test/re10k

runs the reference's test step over the test split: it prints the PSNR / SSIM / LPIPS table of the 8-bit frames
(the paper's numbers) and, with --output, writes the frames (unless --no-frames), benchmark.json,
peak_memory.json and metrics.json (the mean and each scene's metrics).

With --refine-steps N (N >= 0), each scene's Gaussians are refined in memory on its context views before the targets
are rendered: the route export-ply --write-frame -> refine-ply --steps N -> render-ply takes through two PLY files
per scene, with the same frames, metrics and refine.json (written beside metrics.json).  --refine-steps 0 scores the
export round trip unrefined, the baseline a refined score is compared with.  refine-ply's options (--lr-*,
--densify-*, --min-opacity, --opacity-reset-every, --loss, --lambda-dssim, --lr-xyz-final, --lr-xyz-steps) apply, and
only with --refine-steps.  With --preset re10k_3_view the refinement uses all three context views.

    python -m pixelsplat_b200.evaluation compute-metrics --dataset-root datasets/re10k \\
        --index assets/evaluation_index_re10k.json --method pixelSplat:ours:outputs/test/re10k \\
        --output-metrics outputs/metrics.json

is the reference's compute_metrics script: it scores saved frame directories of one or more methods.

    python -m pixelsplat_b200.evaluation export-ply --dataset-root datasets/re10k \\
        --index assets/evaluation_index_re10k.json --checkpoint checkpoints/re10k.ckpt --preset re10k \\
        --output outputs/ply/re10k [--scene NAME ...] [--format viewer|reference]

encodes the test scenes as the test step does and writes each scene's Gaussians to <output>/<scene>.ply: by default
in the viewer format (pixelsplat_b200.ply_export.export_gaussians_ply), or as the reference's export_ply writes them.

With --write-frame, each viewer-format file gets <output>/<scene>.frame.json: the export frame (centre, scale and
rotation) that maps it back into the scene's world.

    python -m pixelsplat_b200.evaluation render-ply --ply outputs/ply/re10k --dataset-root datasets/re10k \
        --index assets/evaluation_index_re10k.json --output outputs/ply_render/re10k
    python -m pixelsplat_b200.evaluation render-ply --ply outputs/ply/re10k/SCENE.ply --spin 120 \
        --output outputs/spin.mp4 [--radius 2 --elevation 20 --resolution 256 256]

renders 3D Gaussian splatting PLY files (pixelsplat_b200.ply_import).  Scene mode renders each index scene's target
views from <ply>/<scene>.ply, put back into the scene's world by <scene>.frame.json, and writes the frames as the
evaluator does (so compute-metrics can score them as a --method) with metrics.json.  Spin mode writes an orbit of
one file about its +z axis as an mp4, colour beside turbo depth.

    python -m pixelsplat_b200.evaluation refine-ply --ply outputs/ply/re10k --dataset-root datasets/re10k \
        --index assets/evaluation_index_re10k.json --output outputs/ply_refined/re10k [--steps 100]

refines each index scene's <ply>/<scene>.ply (pixelsplat_b200.ply_refine) in its world against the scene's context
views only, and writes <output>/<scene>.ply, a copy of <scene>.frame.json and refine.json (each scene's context-view
MSE before and after).  --densify-until N adds 3DGS's densification, pruning and opacity reset before step N
(--densify-from, --densify-every, --densify-grad, --min-opacity, --opacity-reset-every, --densify-seed; 3DGS's
defaults), and refine.json's gaussians_before / gaussians_after.  --loss l1-dssim minimises 3DGS's
(1 - lambda) L1 + lambda D-SSIM summed over the context views instead of their MSE (--lambda-dssim, 3DGS's 0.2;
refine.json adds each scene's loss_before / loss_after), and --lr-xyz-final decays the position rate exponentially to
that value over --lr-xyz-steps steps (default: --steps), as 3DGS's schedule does.  render-ply --ply <output> then
scores the refined scenes on the held-out targets.

    python -m pixelsplat_b200.evaluation generate-index --dataset-root datasets/re10k \
        --output outputs/evaluation_index_re10k [--video]

is the reference's generate_evaluation_index script: it writes <output>/evaluation_index.json (a context pair and
target frames per test scene, or null), and with --video <output>/evaluation_index_video.json, where the targets are
every frame between the pair.

    python -m pixelsplat_b200.evaluation render-video --dataset-root datasets/re10k \
        --index assets/evaluation_index_re10k.json --checkpoint checkpoints/re10k.ckpt --preset re10k \
        --output outputs/video/re10k [--scene NAME ...] [--video rgb wobble interpolation_exagerrated]

renders the reference's validation videos of the test scenes (pixelsplat_b200.video) and writes
<output>/<scene>/<name>.mp4: by default rgb (context view 0 to view 1) and wobble; interpolation_exagerrated on
request.  With three context views, rgb ends at the index's first target and the other two are skipped.

--preset names the experiment the checkpoint was trained with: re10k, acid, re10k_depth_loss, the paper's ablations
re10k_ablation_no_epipolar_transformer / _no_probabilistic_sampling / _no_depth_encoding, or re10k_3_view (three
context views: the index's two and the frame halfway between them).

Nothing is downloaded: the checkpoint holds every encoder weight, and LPIPS reads torchvision's VGG16 file and the
lpips package's lin weights from disk (--lpips-vgg / --lpips-lin, or where those packages keep them).
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch


def _data(p: argparse.ArgumentParser) -> None:
    p.add_argument("--dataset-root", type=Path, required=True, help="dataset root holding test/index.json")
    p.add_argument("--index", type=Path, required=True, help="evaluation index (scene -> context / target)")
    p.add_argument("--seed", type=int, default=None, help="torch seed (default: the reference's 111123)")
    p.add_argument("--num-workers", type=int, default=4, help="DataLoader workers (the reference's test loader: 4)")


def _common(p: argparse.ArgumentParser) -> None:
    _data(p)
    p.add_argument("--lpips-vgg", type=Path, default=None, help="torchvision's vgg16-397923af.pth")
    p.add_argument("--lpips-lin", type=Path, default=None, help="the lpips package's weights/v0.1/vgg.pth")


def _loader(args, preset: str = "re10k"):
    from .presets import dataset_cfg, make_test_dataset
    cfg = dataset_cfg(args.dataset_root, args.index, preset=preset)
    return cfg, torch.utils.data.DataLoader(make_test_dataset(cfg), batch_size=1, num_workers=args.num_workers,
                                            pin_memory=True)


def _lpips(args, device):
    from ..lpips import Lpips
    return Lpips.from_files(args.lpips_vgg, args.lpips_lin).to(device).eval()


def load_preset_checkpoint(path: Path, encoder, preset: str) -> int:
    """`load_checkpoint`, with a hint when the checkpoint's weights do not fit the preset's encoder: a checkpoint of
    an ablation or of the three-view model loads only into the model of its own preset."""
    from .checkpoint import load_checkpoint
    try:
        return load_checkpoint(path, encoder)
    except RuntimeError as e:
        raise SystemExit(f"evaluation: {path} does not fit the encoder of --preset {preset}; check that --preset "
                         f"names the experiment the checkpoint was trained with ({e})") from e


def parse_evaluate(argv: list[str]) -> argparse.Namespace:
    from .presets import PRESETS
    p = argparse.ArgumentParser(prog="python -m pixelsplat_b200.evaluation",
                                description="Evaluate a pixelSplat checkpoint on the RE10k / ACID test split.")
    _common(p)
    p.add_argument("--checkpoint", type=Path, required=True, help="a pixelSplat Lightning checkpoint (.ckpt)")
    p.add_argument("--preset", choices=PRESETS, default="re10k",
                   help="the experiment the checkpoint was trained with (default: re10k)")
    p.add_argument("--output", type=Path, default=None, help="where frames and the JSON files go")
    p.add_argument("--deterministic", action="store_true",
                   help="the encoder picks each ray's most likely depth instead of sampling one")
    p.add_argument("--no-frames", action="store_true", help="write no PNG (metrics and JSON files only)")
    p.add_argument("--global-step", type=int, default=0,
                   help="step given to the encoder (the presets' opacity mapping does not depend on it)")
    p.add_argument("--refine-steps", type=_non_negative(int), default=None,
                   help="refine each scene's Gaussians on its context views with this many Adam steps before the "
                        "targets are rendered, in memory, as export-ply --write-frame, refine-ply and render-ply do "
                        "with files; 0 scores the export round trip unrefined, the baseline (default: off)")
    options = _add_refine_arguments(p, "--refine-steps")
    args = p.parse_args(argv)
    names = ["refine_steps"] + [a.dest for a in options]
    if args.refine_steps is None:
        # argparse's own matching (abbreviations, --opt=value) tells which refinement options were given
        for a in options:
            a.default = argparse.SUPPRESS
        given = vars(p.parse_known_args(argv)[0])
        stray = [a.option_strings[0] for a in options if a.dest in given]
        if stray:
            p.error(f"{', '.join(stray)} without --refine-steps: refinement is off unless --refine-steps is given")
        args.refine = None
    else:
        _refine_settings(p, args)
        args.refine = dict(steps=args.refine_steps, lr=args.lr, densify=args.densify, **_refine_options(args))
        names += ["lr", "densify"]
    for name in names:
        delattr(args, name)
    return args


def evaluate(argv: list[str]) -> dict:
    args = parse_evaluate(argv)
    from .evaluator import Evaluator
    from .presets import SEED, build_model
    device = torch.device("cuda", torch.cuda.current_device())
    cfg, loader = _loader(args, args.preset)
    encoder, decoder = build_model(args.preset, cfg)
    step = load_preset_checkpoint(args.checkpoint, encoder, args.preset)
    print(f"Loaded {args.checkpoint} (trained for {step} steps).")
    evaluator = Evaluator(encoder.to(device).eval(), decoder.to(device), args.output, _lpips(args, device),
                          deterministic=args.deterministic, global_step=args.global_step,
                          write_frames=not args.no_frames, refine=args.refine)
    result = evaluator.run(loader, seed=SEED if args.seed is None else args.seed, device=device)
    if args.refine is not None:
        for s in result.scenes:
            print(_refine_line(s.scene, s.refine))
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


def parse_export_ply(argv: list[str]) -> argparse.Namespace:
    from .presets import PRESETS
    p = argparse.ArgumentParser(prog="python -m pixelsplat_b200.evaluation export-ply",
                                description="Write the Gaussians of test scenes as 3D Gaussian splatting PLY files.")
    _data(p)
    p.add_argument("--checkpoint", type=Path, required=True, help="a pixelSplat Lightning checkpoint (.ckpt)")
    p.add_argument("--preset", choices=PRESETS, default="re10k",
                   help="the experiment the checkpoint was trained with (default: re10k)")
    p.add_argument("--output", type=Path, required=True, help="directory of the <scene>.ply files")
    p.add_argument("--scene", action="append", default=None, metavar="NAME",
                   help="export only this scene (repeatable; default: every test scene)")
    p.add_argument("--format", choices=("viewer", "reference"), default="viewer",
                   help="viewer: what the rasterizer renders, with SH up to degree 3 (default); reference: the "
                        "reference's export_ply (DC only, camera-frame rotations, raw opacity)")
    p.add_argument("--write-frame", action="store_true",
                   help="also write <output>/<scene>.frame.json: the export frame's centre, scale and rotation, which "
                        "render-ply needs to put the file back into the scene's world (viewer format only)")
    args = p.parse_args(argv)
    if args.write_frame and args.format != "viewer":
        p.error("--write-frame needs --format viewer")
    return args


def export_ply(argv: list[str]) -> list[Path]:
    """The test step's data path, seed and encoder call (Evaluator.run / test_step), then one file per scene.  With
    --scene, the scenes before the last named one are still encoded, so that each named scene's Gaussians are the
    ones the test step renders (the encoder samples depths from torch's generator)."""
    args = parse_export_ply(argv)
    from ..data import device_shim
    from ..ply_export import export_frame, export_gaussians_ply, export_ply as export_reference, write_frame_json
    from .presets import IMAGE_SHAPE, SEED, build_model
    device = torch.device("cuda", torch.cuda.current_device())
    cfg, loader = _loader(args, args.preset)
    encoder, _ = build_model(args.preset, cfg)
    step = load_preset_checkpoint(args.checkpoint, encoder, args.preset)
    print(f"Loaded {args.checkpoint} (trained for {step} steps).")
    encoder = encoder.to(device).eval()
    data_shim = encoder.get_data_shim()
    wanted = None if args.scene is None else set(args.scene)
    written: list[Path] = []
    torch.manual_seed(SEED if args.seed is None else args.seed)
    with torch.no_grad():
        for batch in loader:
            if wanted is not None and not wanted - {p.stem for p in written}:
                break
            batch = data_shim(device_shim(batch, IMAGE_SHAPE, device))
            dump = {} if args.format == "reference" else None
            gaussians = encoder(batch["context"], 0, deterministic=False, visualization_dump=dump)
            (scene,) = batch["scene"]
            if wanted is not None and scene not in wanted:
                continue
            path = args.output / f"{scene}.ply"
            extrinsics = batch["context"]["extrinsics"][0, 0]
            if args.format == "viewer":
                export_gaussians_ply(gaussians, extrinsics, path)
                if args.write_frame:
                    write_frame_json(export_frame(gaussians.means[0], extrinsics), path.with_suffix(".frame.json"))
            else:
                export_reference(extrinsics, gaussians.means[0], dump["scales"][0], dump["rotations"][0],
                                 gaussians.harmonics[0], gaussians.opacities[0], path)
            written.append(path)
    print(f"Wrote {len(written)} PLY files to {args.output}.")
    missing = sorted(wanted - {p.stem for p in written}) if wanted is not None else []
    if missing:
        raise SystemExit(f"evaluation export-ply: no test scene named {', '.join(missing)}")
    return written


def parse_render_video(argv: list[str]) -> argparse.Namespace:
    from ..video import VALIDATION_VIDEOS, VIDEOS
    from .presets import PRESETS
    p = argparse.ArgumentParser(prog="python -m pixelsplat_b200.evaluation render-video",
                                description="Render the interpolation and wobble videos of test scenes as MP4.")
    _data(p)
    p.add_argument("--checkpoint", type=Path, required=True, help="a pixelSplat Lightning checkpoint (.ckpt)")
    p.add_argument("--preset", choices=PRESETS, default="re10k",
                   help="the experiment the checkpoint was trained with (default: re10k)")
    p.add_argument("--output", type=Path, required=True, help="directory of the <scene>/<video>.mp4 files")
    p.add_argument("--scene", action="append", default=None, metavar="NAME",
                   help="render only this scene (repeatable; default: every test scene)")
    p.add_argument("--video", nargs="+", choices=tuple(VIDEOS), default=list(VALIDATION_VIDEOS),
                   help="videos to render (default: rgb wobble, the reference's validation videos)")
    args = p.parse_args(argv)
    args.video = list(dict.fromkeys(args.video))
    return args


def render_videos(argv: list[str]) -> list[Path]:
    """The test step's data path; torch's generators seeded from --seed before each scene, so a scene's frames do
    not depend on which scenes are rendered; one encoder trunk per scene and the videos in the order asked."""
    args = parse_render_video(argv)
    from ..data import device_shim
    from ..video import render_video, write_mp4
    from .presets import IMAGE_SHAPE, SEED, build_model
    device = torch.device("cuda", torch.cuda.current_device())
    cfg, loader = _loader(args, args.preset)
    encoder, decoder = build_model(args.preset, cfg)
    step = load_preset_checkpoint(args.checkpoint, encoder, args.preset)
    print(f"Loaded {args.checkpoint} (trained for {step} steps).")
    encoder, decoder = encoder.to(device).eval(), decoder.to(device)
    data_shim = encoder.get_data_shim()
    wanted = None if args.scene is None else set(args.scene)
    seed = SEED if args.seed is None else args.seed
    written: list[Path] = []
    seen: set[str] = set()
    with torch.no_grad():
        for batch in loader:
            (scene,) = batch["scene"]
            if wanted is not None and scene not in wanted:
                continue
            seen.add(scene)
            torch.manual_seed(seed)
            batch = data_shim(device_shim(batch, IMAGE_SHAPE, device))
            features, _ = encoder.trunk(batch["context"])
            for name in args.video:
                frames = render_video(encoder, decoder, batch["context"], batch["target"], name, 0, features)
                if frames is None:
                    print(f"{scene}: {name} needs two context views; skipped")
                    continue
                written.append(write_mp4(frames.numpy(), args.output / scene / f"{name}.mp4"))
            if wanted is not None and not wanted - seen:
                break
    print(f"Wrote {len(written)} videos to {args.output}.")
    missing = sorted(wanted - seen) if wanted is not None else []
    if missing:
        raise SystemExit(f"evaluation render-video: no test scene named {', '.join(missing)}")
    return written


def parse_render_ply(argv: list[str]) -> argparse.Namespace:
    p = argparse.ArgumentParser(prog="python -m pixelsplat_b200.evaluation render-ply",
                                description="Render 3D Gaussian splatting PLY files: the test scenes' target views "
                                            "from exported files, or a spin around one file.")
    p.add_argument("--ply", type=Path, required=True,
                   help="directory of <scene>.ply and <scene>.frame.json (scene mode), or one .ply file (--spin)")
    p.add_argument("--output", type=Path, required=True,
                   help="directory of <scene>/color/<index>.png and metrics.json, or the .mp4 file (--spin)")
    p.add_argument("--dataset-root", type=Path, default=None, help="dataset root holding test/index.json")
    p.add_argument("--index", type=Path, default=None, help="evaluation index (scene -> context / target)")
    p.add_argument("--num-workers", type=int, default=4, help="DataLoader workers (the reference's test loader: 4)")
    p.add_argument("--lpips-vgg", type=Path, default=None, help="torchvision's vgg16-397923af.pth")
    p.add_argument("--lpips-lin", type=Path, default=None, help="the lpips package's weights/v0.1/vgg.pth")
    p.add_argument("--spin", type=int, default=None, metavar="FRAMES",
                   help="render an orbit of FRAMES frames around the file's origin as an mp4 instead")
    p.add_argument("--radius", type=float, default=2.0, help="orbit radius, in the file's units (default: 2)")
    p.add_argument("--elevation", type=float, default=20.0, help="orbit elevation in degrees (default: 20)")
    p.add_argument("--resolution", type=int, nargs=2, default=[256, 256], metavar=("H", "W"),
                   help="spin frame size (default: 256 256)")
    args = p.parse_args(argv)
    if args.spin is None:
        if args.dataset_root is None or args.index is None:
            p.error("scene mode needs --dataset-root and --index (or --spin FRAMES for an orbit)")
    elif args.spin < 1 or args.radius <= 0 or min(args.resolution) < 1:
        p.error("--spin, --radius and --resolution must be positive")
    return args


def render_ply(argv: list[str]) -> dict:
    """Scene mode: every index scene's target views rendered from <ply>/<scene>.ply, imported into the scene's world
    through <scene>.frame.json, as the test step renders (chunks of CHUNK views, the 8-bit frame pass); frames in
    the evaluator's layout and the evaluator's metrics.json.  Spin mode: one file's orbit as an mp4."""
    args = parse_render_ply(argv)
    from types import SimpleNamespace
    from ..ply_import import load_gaussians_ply
    from ..decoder import DecoderSplattingCUDA, DecoderSplattingCUDACfg
    device = torch.device("cuda", torch.cuda.current_device())
    if args.spin is not None:
        from ..video import render_spin, write_mp4
        decoder = DecoderSplattingCUDA(DecoderSplattingCUDACfg("splatting_cuda"),
                                       SimpleNamespace(background_color=[0.0, 0.0, 0.0])).to(device)
        frames = render_spin(decoder, load_gaussians_ply(args.ply, device), args.spin, args.radius,
                             args.elevation, tuple(args.resolution))
        path = write_mp4(frames.numpy(), args.output)
        print(f"Wrote {len(frames)} frames to {path}.")
        return {"frames": len(frames)}

    from ..data import device_shim
    from .evaluator import METRICS, mean_over_scenes
    from .image_io import save_frame
    from .metrics import CHUNK, frame_metrics_chunked
    from .presets import IMAGE_SHAPE
    cfg, loader = _loader(args)
    decoder = DecoderSplattingCUDA(DecoderSplattingCUDACfg("splatting_cuda"), cfg).to(device)
    lpips = _lpips(args, device)
    scenes = {}
    with torch.no_grad():
        for batch in loader:
            (scene,) = batch["scene"]
            frame = args.ply / f"{scene}.frame.json"
            if not frame.exists():
                raise SystemExit(f"evaluation render-ply: {frame} is missing; export the scenes with "
                                 "`export-ply --write-frame` to render them in their world")
            gaussians = load_gaussians_ply(args.ply / f"{scene}.ply", device, frame=frame)
            tgt = device_shim(batch, IMAGE_SHAPE, device)["target"]
            v, (h, w) = tgt["image"].shape[1], tgt["image"].shape[-2:]
            color = torch.cat([decoder.forward(gaussians, tgt["extrinsics"][:1, i:i + CHUNK],
                                               tgt["intrinsics"][:1, i:i + CHUNK], tgt["near"][:1, i:i + CHUNK],
                                               tgt["far"][:1, i:i + CHUNK], (h, w)).color
                               for i in range(0, v, CHUNK)], dim=1)
            per_view = frame_metrics_chunked(tgt["image"][0], color[0], lpips, return_frames=True)
            frames = per_view.pop("frames").cpu().numpy()
            for index, f in zip(tgt["index"][0].tolist(), frames):
                save_frame(f, args.output / scene / "color" / f"{index:0>6}.png")
            scenes[scene] = {k: float(per_view[k].mean()) for k in METRICS}
    out = {"mean": mean_over_scenes(scenes.values()), "scenes": scenes}
    print(f"{len(scenes)} scenes: " + ", ".join(f"{k} {v:.4f}" for k, v in out["mean"].items()))
    args.output.mkdir(parents=True, exist_ok=True)
    (args.output / "metrics.json").write_text(json.dumps(out))
    return out


def _non_negative(kind):
    def parse(text: str):
        value = kind(text)
        if not value >= 0:
            raise argparse.ArgumentTypeError(f"{text} is negative")
        return value
    return parse


def _positive(kind):
    def parse(text: str):
        value = kind(text)
        if not value > 0:
            raise argparse.ArgumentTypeError(f"{text} is not positive")
        return value
    return parse


def _unit_interval(text: str) -> float:
    value = float(text)
    if not 0 <= value <= 1:
        raise argparse.ArgumentTypeError(f"{text} is not in [0, 1]")
    return value


def _add_refine_arguments(p: argparse.ArgumentParser, steps_flag: str) -> list[argparse.Action]:
    """The refinement options refine-ply and evaluate share: learning rates, densification, loss and the position
    rate's decay (`steps_flag` is the command's flag for the number of steps).  Returns their actions."""
    from ..ply_refine import DEFAULT_LR, GROUPS, DensifyConfig
    actions = []
    for g in GROUPS:
        actions.append(p.add_argument(f"--lr-{g.replace('_', '-')}", dest=f"lr_{g}", type=_non_negative(float),
                                      default=DEFAULT_LR[g],
                                      help=f"learning rate of the {g} properties (default: 3DGS's {DEFAULT_LR[g]:g})"))
    d = DensifyConfig()
    actions += [
        p.add_argument("--densify-until", type=_non_negative(int), default=0,
                       help="densify, prune and reset opacities before this step, as 3DGS does (default: 0, off; "
                            f"3DGS: {d.until_step})"),
        p.add_argument("--densify-from", type=_non_negative(int), default=d.from_step,
                       help=f"densify after this step (default: 3DGS's {d.from_step})"),
        p.add_argument("--densify-every", type=int, default=d.every,
                       help=f"steps between densifications (default: 3DGS's {d.every})"),
        p.add_argument("--densify-grad", type=_non_negative(float), default=d.grad_threshold,
                       help=f"mean screen-space gradient norm that selects a Gaussian (default: 3DGS's "
                            f"{d.grad_threshold:g}, calibrated for its L1 + D-SSIM loss; with --loss mse the "
                            "gradients are smaller and it has not been tuned)"),
        p.add_argument("--min-opacity", type=_non_negative(float), default=d.min_opacity,
                       help=f"prune Gaussians below this opacity (default: 3DGS's {d.min_opacity:g})"),
        p.add_argument("--opacity-reset-every", type=_non_negative(int), default=d.opacity_reset_every,
                       help=f"steps between opacity resets, 0 for none (default: 3DGS's {d.opacity_reset_every})"),
        p.add_argument("--densify-seed", type=_non_negative(int), default=d.seed,
                       help=f"seed of the split copies' draws (default: {d.seed})"),
        p.add_argument("--loss", choices=("mse", "l1-dssim"), default="mse",
                       help="mse: the MSE over the context views (default); l1-dssim: 3DGS's (1 - lambda) L1 + "
                            "lambda D-SSIM, summed over the context views"),
        p.add_argument("--lambda-dssim", type=_unit_interval, default=0.2,
                       help="D-SSIM weight of --loss l1-dssim (default: 3DGS's 0.2)"),
        p.add_argument("--lr-xyz-final", type=_positive(float), default=None,
                       help="decay the position rate exponentially from --lr-xyz to this rate (default: off, a "
                            "constant rate; 3DGS: 1.6e-6)"),
        p.add_argument("--lr-xyz-steps", type=_positive(int), default=None,
                       help=f"steps of the position rate's decay (default: {steps_flag}; 3DGS: 30000)")]
    return actions


def _refine_settings(p: argparse.ArgumentParser, args: argparse.Namespace) -> None:
    """The checks and derived values of `_add_refine_arguments`' options, in place: `loss` as refine_records names
    it, `lr` (every group's rate) and `densify` (a DensifyConfig, or None with --densify-until 0)."""
    from ..ply_refine import GROUPS, DensifyConfig
    args.loss = args.loss.replace("-", "_")
    if args.lr_xyz_steps is not None and args.lr_xyz_final is None:
        p.error("--lr-xyz-steps needs --lr-xyz-final")
    if args.lr_xyz_final is not None and not args.lr_xyz > 0:
        p.error("--lr-xyz-final needs --lr-xyz > 0")
    args.lr = {g: getattr(args, f"lr_{g}") for g in GROUPS}
    args.densify = None
    if args.densify_until > 0:
        try:
            args.densify = DensifyConfig(from_step=args.densify_from, until_step=args.densify_until,
                                         every=args.densify_every, grad_threshold=args.densify_grad,
                                         min_opacity=args.min_opacity, opacity_reset_every=args.opacity_reset_every,
                                         seed=args.densify_seed)
        except ValueError as e:
            p.error(str(e))


def parse_refine_ply(argv: list[str]) -> argparse.Namespace:
    p = argparse.ArgumentParser(prog="python -m pixelsplat_b200.evaluation refine-ply",
                                description="Refine exported 3D Gaussian splatting PLY files on each test scene's "
                                            "context views.")
    p.add_argument("--ply", type=Path, required=True, help="directory of <scene>.ply and <scene>.frame.json")
    p.add_argument("--dataset-root", type=Path, required=True, help="dataset root holding test/index.json")
    p.add_argument("--index", type=Path, required=True, help="evaluation index (scene -> context / target)")
    p.add_argument("--output", type=Path, required=True,
                   help="directory of the refined <scene>.ply, <scene>.frame.json and refine.json")
    p.add_argument("--scene", action="append", default=None, metavar="NAME",
                   help="refine only this scene (repeatable; default: every index scene)")
    p.add_argument("--steps", type=_non_negative(int), default=100, help="Adam steps per scene (default: 100)")
    p.add_argument("--num-workers", type=int, default=4, help="DataLoader workers (the reference's test loader: 4)")
    _add_refine_arguments(p, "--steps")
    args = p.parse_args(argv)
    _refine_settings(p, args)
    return args


def _refine_options(args) -> dict:
    """The refinement's loss and schedule arguments of `ply_refine.refine_records`."""
    return dict(loss=args.loss, lambda_dssim=args.lambda_dssim, lr_xyz_final=args.lr_xyz_final,
                lr_xyz_steps=args.lr_xyz_steps)


def _refine_scene_report(args, result) -> dict:
    """One scene's entry of refine.json (`ply_refine.scene_report`) for the parsed refinement options."""
    from ..ply_refine import scene_report
    return scene_report(result, args.steps, args.loss, args.densify)


def _refine_report(args, scenes: dict) -> dict:
    """refine.json (`ply_refine.refine_report`) for the parsed refinement options."""
    from ..ply_refine import refine_report
    return refine_report(scenes, args.steps, args.lr, args.densify, **_refine_options(args))


def _refine_line(scene: str, r: dict) -> str:
    """A scene's refine.json entry as one line of output."""
    line = f"{scene}: context MSE {r['mse_before']:.6f} -> {r['mse_after']:.6f} in {r['steps']} steps"
    if "loss_before" in r:
        line += f", L1 + D-SSIM {r['loss_before']:.6f} -> {r['loss_after']:.6f}"
    if "gaussians_before" in r:
        line += f", {r['gaussians_before']} -> {r['gaussians_after']} Gaussians"
    return line


def refine_ply(argv: list[str]) -> dict:
    """Every index scene's <ply>/<scene>.ply refined in its world (<scene>.frame.json) on the scene's context views,
    loaded as render-ply loads its targets; the targets stay held out."""
    args = parse_refine_ply(argv)
    import shutil
    from ..data import device_shim
    from ..ply_import import read_frame_json, read_ply_body
    from ..ply_refine import refine_ply as refine, refine_records
    from .presets import IMAGE_SHAPE
    device = torch.device("cuda", torch.cuda.current_device())
    cfg, loader = _loader(args)
    background = torch.tensor(cfg.background_color, dtype=torch.float32, device=device)
    wanted = None if args.scene is None else set(args.scene)
    scenes = {}
    for batch in loader:
        (scene,) = batch["scene"]
        if wanted is not None and scene not in wanted:
            continue
        frame = args.ply / f"{scene}.frame.json"
        if not frame.exists():
            raise SystemExit(f"evaluation refine-ply: {frame} is missing; export the scenes with "
                             "`export-ply --write-frame` to refine them in their world")
        ctx = device_shim(batch, IMAGE_SHAPE, device)["context"]
        result = refine(args.ply / f"{scene}.ply", frame, extrinsics=ctx["extrinsics"][0],
                        intrinsics=ctx["intrinsics"][0], near=ctx["near"][0], far=ctx["far"][0],
                        images=ctx["image"][0], background_color=background, steps=args.steps,
                        out_path=args.output / f"{scene}.ply", lr=args.lr, device=device, densify=args.densify,
                        **_refine_options(args))
        shutil.copyfile(frame, args.output / f"{scene}.frame.json")
        if result is None:   # --steps 0: the file is copied; its MSE is one render
            layout, records = read_ply_body(args.ply / f"{scene}.ply", device)
            result = refine_records(records, layout.properties, layout.sh_degree,
                                    frame=read_frame_json(frame, device), extrinsics=ctx["extrinsics"][0],
                                    intrinsics=ctx["intrinsics"][0], near=ctx["near"][0], far=ctx["far"][0],
                                    images=ctx["image"][0], background_color=background, steps=0,
                                    **_refine_options(args))
        scenes[scene] = _refine_scene_report(args, result)
        print(_refine_line(scene, scenes[scene]))
    missing = sorted(wanted - set(scenes)) if wanted is not None else []
    if missing:
        raise SystemExit(f"evaluation refine-ply: no index scene named {', '.join(missing)}")
    out = _refine_report(args, scenes)
    args.output.mkdir(parents=True, exist_ok=True)
    (args.output / "refine.json").write_text(json.dumps(out, indent=1) + "\n")
    return out


def parse_generate_index(argv: list[str]) -> argparse.Namespace:
    from .index_generator import EvaluationIndexGeneratorCfg
    d = EvaluationIndexGeneratorCfg()
    p = argparse.ArgumentParser(prog="python -m pixelsplat_b200.evaluation generate-index",
                                description="Pick a context pair and target frames for every test scene.")
    p.add_argument("--dataset-root", type=Path, required=True, help="dataset root holding test/index.json")
    p.add_argument("--output", type=Path, required=True, help="directory of evaluation_index.json")
    p.add_argument("--num-target-views", type=int, default=d.num_target_views, help="target frames per scene")
    p.add_argument("--min-overlap", type=float, default=d.min_overlap, help="least overlap of a context pair")
    p.add_argument("--max-overlap", type=float, default=d.max_overlap, help="largest overlap of a context pair")
    p.add_argument("--min-distance", type=int, default=d.min_distance, help="least frame gap of a context pair")
    p.add_argument("--max-distance", type=int, default=d.max_distance,
                   help="frame gap past which a walk stops (the first frame past it is still a candidate)")
    p.add_argument("--seed", type=int, default=d.seed, help="seed of the generator that draws every choice")
    p.add_argument("--num-workers", type=int, default=8,
                   help="DataLoader workers (the reference's: 8).  The scene order, and so the index, depends on it: "
                        "keep 8 to reproduce the reference's index")
    p.add_argument("--video", action="store_true",
                   help="also write evaluation_index_video.json (every frame between the pair is a target)")
    args = p.parse_args(argv)
    if args.num_workers < 0:
        p.error("--num-workers must be >= 0")
    try:
        args.cfg = EvaluationIndexGeneratorCfg(args.num_target_views, args.min_distance, args.max_distance,
                                               args.min_overlap, args.max_overlap, args.output, args.seed)
    except ValueError as e:
        p.error(str(e))
    return args


def generate_index(argv: list[str]) -> list[Path]:
    args = parse_generate_index(argv)
    from . import index_generator as ig
    from .presets import IMAGE_SHAPE
    device = torch.device("cuda", torch.cuda.current_device())
    index = ig.generate_index(ig.camera_loader(args.dataset_root, args.num_workers), *IMAGE_SHAPE, args.cfg, device)
    written = ig.save_index(index, args.output, video=args.video)
    found = sum(v is not None for v in index.values())
    print(f"{len(index)} scenes, {found} with a context pair: wrote " + ", ".join(str(p) for p in written))
    return written


def main(argv: list[str] | None = None) -> None:
    argv = sys.argv[1:] if argv is None else argv
    if argv and argv[0] == "generate-index":
        generate_index(argv[1:])
    elif argv and argv[0] == "compute-metrics":
        compute_metrics(argv[1:])
    elif argv and argv[0] == "export-ply":
        export_ply(argv[1:])
    elif argv and argv[0] == "render-video":
        render_videos(argv[1:])
    elif argv and argv[0] == "render-ply":
        render_ply(argv[1:])
    elif argv and argv[0] == "refine-ply":
        refine_ply(argv[1:])
    else:
        evaluate(argv)


if __name__ == "__main__":
    main()
