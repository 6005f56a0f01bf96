#!/usr/bin/env python
"""Times the evaluation's per-scene work on the GPU, CUDA events, median per call:
  scene      one synthetic re10k-shaped test scene at 256 x 256, 2 context views and 3 targets (the RE10k / ACID
             evaluation index) or 100 targets (the video index's shape), split into the encoder (EncoderEpipolar,
             re10k preset, random weights, deterministic=False), the render (32 targets per decoder call), the
             8-bit frame pass (csrc/eval_images.cu: frames, planes and squared error), SSIM and LPIPS (seeded
             weights; the time does not depend on them);
  frame pass the kernel against the same work in torch (clip, mul, to(uint8), float, div, squared error, and the
             HWC frame copy) on [32, 3, 256, 256].
Prints one JSON line with the card and its power limit.  Nothing is written.

    python tools/bench_eval.py [--steps 20] [--warmup 3]
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
from pixelsplat_b200.evaluation import frame_pass  # noqa: E402
from pixelsplat_b200.evaluation.metrics import CHUNK  # noqa: E402
from pixelsplat_b200.evaluation.presets import build_model, dataset_cfg  # noqa: E402
from pixelsplat_b200.loss import compute_ssim  # noqa: E402
from pixelsplat_b200.lpips import Lpips  # noqa: E402
from tools.bench_depth import gpu_identity  # noqa: E402

DEV = "cuda"
SHAPE = (256, 256)


def timed(fn, steps: int, warmup: int) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def example(targets: int) -> dict:
    """A re10k-shaped scene: two context views with the synthetic rig's cameras, `targets` target cameras."""
    g = torch.Generator().manual_seed(targets)
    sc = synthetic.scene_re10k_like(seed=0, target_views=targets)
    ctx = synthetic.scene_re10k_like(seed=1, target_views=2)

    def views(s, n):
        return {"extrinsics": s.extrinsics[None].to(DEV), "intrinsics": s.intrinsics[None].to(DEV),
                "near": s.near[None].to(DEV), "far": s.far[None].to(DEV),
                "image": torch.rand(1, n, 3, *SHAPE, generator=g).to(DEV)}
    return {"context": views(ctx, 2), "target": views(sc, targets)}


@torch.no_grad()
def scene_times(targets: int, encoder, decoder, lpips, steps: int, warmup: int) -> dict:
    b = example(targets)
    ctx, tgt = b["context"], b["target"]
    gt = tgt["image"][0]
    gaussians = encoder(ctx, 0, deterministic=False)

    def render():
        return torch.cat([decoder(gaussians, tgt["extrinsics"][:, i:i + CHUNK], tgt["intrinsics"][:, i:i + CHUNK],
                                  tgt["near"][:, i:i + CHUNK], tgt["far"][:, i:i + CHUNK], SHAPE).color[0]
                          for i in range(0, targets, CHUNK)])
    color = render()
    planes = frame_pass(color, target=gt).planes
    out = {"encoder_ms": timed(lambda: encoder(ctx, 0, deterministic=False), steps, warmup),
           "render_ms": timed(render, steps, warmup),
           "frame_pass_ms": timed(lambda: frame_pass(color, target=gt), steps, warmup),
           "ssim_ms": timed(lambda: compute_ssim(gt, planes), steps, warmup),
           "lpips_ms": timed(lambda: torch.cat([lpips(gt[i:i + CHUNK], planes[i:i + CHUNK], normalize=True)
                                                for i in range(0, targets, CHUNK)]), steps, warmup)}
    out["total_ms"] = sum(out.values())
    return {f"t{targets}_{k}": v for k, v in out.items()}


def frame_pass_vs_torch(steps: int, warmup: int) -> dict:
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(32, 3, *SHAPE, generator=g) * 1.2 - 0.1).to(DEV)
    t = torch.rand(32, 3, *SHAPE, generator=g).to(DEV)

    def torch_route():
        u = (x.clip(min=0, max=1) * 255).to(torch.uint8)
        frames = u.permute(0, 2, 3, 1).contiguous()
        planes = u.float() / 255
        return frames, planes, ((planes - t.clip(min=0, max=1)) ** 2).sum(dim=(1, 2, 3))
    kernel_ms = timed(lambda: frame_pass(x, target=t), steps, warmup)
    torch_ms = timed(torch_route, steps, warmup)
    n = x.numel()
    bytes_moved = n * (4 + 4 + 4 + 1)          # render and target read, planes and frames written
    return {"fp32x32_kernel_ms": kernel_ms, "fp32x32_torch_ms": torch_ms, "fp32x32_bytes": bytes_moved,
            "fp32x32_kernel_GBps": bytes_moved / (kernel_ms * 1e-3) / 1e9}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval: no CUDA device; the times need an H100")
    torch.manual_seed(0)
    encoder, decoder = build_model("re10k", dataset_cfg("/nonexistent", "/nonexistent"))
    encoder, decoder = encoder.to(DEV).eval(), decoder.to(DEV)
    lpips = Lpips()
    lpips.load_state_dict(lo.random_state_dict(0))
    lpips = lpips.to(DEV).eval()
    res = {**frame_pass_vs_torch(args.steps, args.warmup)}
    for targets in (3, 100):
        res.update(scene_times(targets, encoder, decoder, lpips, args.steps, args.warmup))
    res.update(gpu_identity(0))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
