#!/usr/bin/env python
"""Training and encoding cost of the paper's model, its three ablations and the three-view model, CUDA events:
for each preset at its training batch size (7 scenes; 3 for re10k_3_view), on seeded synthetic 256 x 256 scenes
with the preset's context views and 4 targets, the preset's encoder with random weights and its losses (MSE + LPIPS
with seeded weights, LPIPS inactive before step 150 000 as at the start of a run):
  train_step_ms      median `Trainer.training_step` time over --steps steps after --warmup;
  peak_train_gib     torch.cuda.max_memory_allocated over one training step (weights and optimiser state included);
  encode_scene_ms    median time of one evaluation scene's encoder pass (eval mode, no autograd, batch 1).
Prints one JSON line per preset and a last one with the card and its power limit.  Nothing is written.

    python tools/bench_presets.py [--steps 20] [--warmup 3]
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
from pixelsplat_b200.evaluation.presets import build_model, num_context_views  # noqa: E402
from pixelsplat_b200.lpips import Lpips  # noqa: E402
from pixelsplat_b200.training import Trainer  # noqa: E402
from pixelsplat_b200.training import presets as tp  # noqa: E402
from tools.bench_depth import gpu_identity  # noqa: E402

DEV = torch.device("cuda", 0)
SHAPE = (256, 256)
TARGETS = 4
PRESETS = ("re10k", "re10k_ablation_no_epipolar_transformer", "re10k_ablation_no_probabilistic_sampling",
           "re10k_ablation_no_depth_encoding", "re10k_3_view")


def batch(scenes: int, views: int, seed: int) -> dict:
    """A device-resident batch as `device_shim` returns it: `views` context cameras spread over one unit along x,
    TARGETS target cameras around them, uniform random images.  near / far are replaced by the bounds shim."""
    g = torch.Generator().manual_seed(seed)
    ctx_e = torch.eye(4).repeat(scenes, views, 1, 1)
    ctx_e[:, :, 0, 3] = torch.linspace(0.0, 1.0, views)
    tgt_e = torch.stack([synthetic.target_cameras(TARGETS, seed=seed * 100 + s) for s in range(scenes)])

    def view_set(extrinsics, n):
        intrinsics = synthetic.intrinsics_re10k(n)[None].repeat(scenes, 1, 1, 1)
        return {"extrinsics": extrinsics.to(DEV), "intrinsics": intrinsics.to(DEV),
                "near": torch.full((scenes, n), 1.0, device=DEV), "far": torch.full((scenes, n), 100.0, device=DEV),
                "index": torch.arange(n).repeat(scenes, 1).to(DEV),
                "image": torch.rand(scenes, n, 3, *SHAPE, generator=g).to(DEV)}
    return {"context": view_set(ctx_e, views), "target": view_set(tgt_e, TARGETS),
            "scene": [f"synthetic{s}" for s in range(scenes)]}


def measure(name: str, steps: int, warmup: int) -> dict:
    preset = tp.train_preset(name)
    views = num_context_views(preset.model)
    torch.manual_seed(0)
    encoder, decoder = build_model(preset.model, tp.dataset_cfg(preset, "/nonexistent"))
    lpips = Lpips()
    lpips.load_state_dict(lo.random_state_dict(0))
    t = Trainer(encoder.to(DEV), decoder.to(DEV), tp.make_losses(preset, lpips), lr=preset.lr,
                warm_up_steps=preset.warm_up_steps, max_norm=preset.max_norm)
    train_batch, scene = batch(preset.batch_size, views, 2), batch(1, views, 1)

    train, peak = [], 0
    for i in range(warmup + steps):
        if i == warmup:
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(DEV)
        t.training_step(train_batch)
        line = t.read_last()
        if i == warmup:
            peak = torch.cuda.max_memory_allocated(DEV)
        if i >= warmup:
            train.append(sum(line["phase_ms"].values()))

    encode = []
    shim = t.data_shim
    t.encoder.eval()
    with torch.no_grad():
        ctx = shim(scene)["context"]
        for i in range(warmup + steps):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            t.encoder(ctx, 0, deterministic=False)
            ev[1].record()
            ev[1].synchronize()
            if i >= warmup:
                encode.append(ev[0].elapsed_time(ev[1]))
    out = {"preset": name, "context_views": views, "batch": preset.batch_size,
           "train_step_ms": statistics.median(train), "peak_train_gib": peak / 2 ** 30,
           "encode_scene_ms": statistics.median(encode)}
    del t, encoder, decoder
    torch.cuda.empty_cache()
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_presets: no CUDA device; the times need an H100")
    torch.cuda.set_device(DEV)
    for name in PRESETS:
        print(json.dumps(measure(name, args.steps, args.warmup)), flush=True)
    print(json.dumps({"steps": args.steps, "warmup": args.warmup,
                      "total_memory_gib": torch.cuda.get_device_properties(0).total_memory / 2 ** 30,
                      **gpu_identity(0)}))


if __name__ == "__main__":
    main()
