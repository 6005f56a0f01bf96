#!/usr/bin/env python
"""Times SSIM two ways at the shapes it is used at:
  gpu        pixelsplat_b200.loss.ssim (csrc/ssim.cu), forward and forward + backward, CUDA events;
  reference  the reference's compute_ssim route (/root/reference/src/evaluation/metrics.py:36-52): a device-to-host
             copy, then one CPU call per image; the CPU call is oracle/ssim_oracle.py's numpy restatement in float32
             (skimage is not available), timed on this machine's host with the host clock.
Shapes: [32, 3, 256, 256] (one test_step chunk) and [4, 3, 256, 256] (one scene's target views in training).
GPU: warm-up, then three alternating rounds (forward, forward + backward) of --steps calls each, median per call.
Prints one JSON line per shape with both times, the algorithmic bytes and FLOPs, the achieved GB/s, the card and its
power limit.  Nothing is written.

    python tools/bench_ssim.py [--steps 200] [--warmup 20] [--ref-images 4]
"""
import argparse
import json
import os
import statistics
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tools.bench_depth import gpu_identity  # noqa: E402

# Algorithmic work per pixel of the separable 11-tap filter (no halo recompute): the forward filters 5 maps (x, y,
# x^2, y^2, xy) twice, 11 FMA each, plus ~20 flops for the products and S; the backward recomputes that, forms the
# chain rule's 4 maps (~40 flops) and filters them twice, and writes both gradients (~8 flops).
FWD_FLOPS_PER_PX = 5 * 2 * 11 * 2 + 20
BWD_FLOPS_PER_PX = FWD_FLOPS_PER_PX + 40 + 4 * 2 * 11 * 2 + 8


def work(shape) -> dict:
    b, c, h, w = shape
    px = b * c * h * w
    return {"fwd_bytes": 2 * 4 * px + 4 * b * c, "fwdbwd_bytes": 2 * 4 * px + 4 * b * c + 2 * 4 * px + 2 * 4 * px,
            "fwd_flops": FWD_FLOPS_PER_PX * px, "fwdbwd_flops": (FWD_FLOPS_PER_PX + BWD_FLOPS_PER_PX) * px}


def time_gpu(shape, steps, warmup) -> dict:
    from pixelsplat_b200.loss import ssim
    g = torch.Generator().manual_seed(0)
    x = torch.rand(shape, generator=g).cuda()
    y = (x.cpu() + 0.1 * torch.randn(shape, generator=g)).cuda().requires_grad_(True)

    def fwd():
        with torch.no_grad():
            ssim(x, y)

    def fwdbwd():
        torch.autograd.grad(ssim(x, y).sum(), y)

    for f in (fwd, fwdbwd):
        for _ in range(warmup):
            f()
    torch.cuda.synchronize()
    ms = {"fwd": [], "fwdbwd": []}
    for _ in range(3):
        for name, f in (("fwd", fwd), ("fwdbwd", fwdbwd)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(steps):
                f()
            b.record()
            torch.cuda.synchronize()
            ms[name].append(a.elapsed_time(b) / steps)
    return {k: statistics.median(v) for k, v in ms.items()} | {"rounds_ms": ms}


def time_reference(shape, n_images) -> dict:
    """Device-to-host copy of the whole batch, then the numpy restatement per image (float32, as the reference's
    float32 arrays are); the per-image time is measured on n_images images and scaled to the batch."""
    from oracle import ssim_oracle as so
    import numpy as np
    g = torch.Generator().manual_seed(1)
    x = torch.rand(shape, generator=g).cuda()
    y = (x.cpu() + 0.1 * torch.randn(shape, generator=g)).cuda()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    xh, yh = x.cpu().numpy(), y.cpu().numpy()
    copy_s = time.perf_counter() - t0
    n = min(n_images, shape[0])
    t0 = time.perf_counter()
    for i in range(n):
        so.ssim_planes_numpy(xh[i], yh[i], np.float32).mean()
    per_image_s = (time.perf_counter() - t0) / n
    return {"d2h_ms": copy_s * 1e3, "per_image_ms": per_image_s * 1e3,
            "batch_ms": (copy_s + per_image_s * shape[0]) * 1e3, "images_timed": n}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--ref-images", type=int, default=4, help="images timed on the CPU route per shape")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ssim.py needs a CUDA device: pixelsplat_b200 has no CPU path")
    ident = gpu_identity(0)
    for shape in ((32, 3, 256, 256), (4, 3, 256, 256)):
        gpu = time_gpu(shape, args.steps, args.warmup)
        ref = time_reference(shape, args.ref_images)
        wk = work(shape)
        line = {"metric": "ssim", "shape": list(shape), "gpu_fwd_ms": gpu["fwd"], "gpu_fwdbwd_ms": gpu["fwdbwd"],
                "fwd_GBps": wk["fwd_bytes"] / (gpu["fwd"] * 1e-3) / 1e9,
                "fwdbwd_GBps": wk["fwdbwd_bytes"] / (gpu["fwdbwd"] * 1e-3) / 1e9,
                "fwd_TFLOPs": wk["fwd_flops"] / (gpu["fwd"] * 1e-3) / 1e12,
                "fwdbwd_TFLOPs": wk["fwdbwd_flops"] / (gpu["fwdbwd"] * 1e-3) / 1e12,
                "reference_route_ms": ref["batch_ms"], "reference_d2h_ms": ref["d2h_ms"],
                "reference_per_image_ms": ref["per_image_ms"], "speedup_fwd": ref["batch_ms"] / gpu["fwd"],
                "host_cpu": {"cpu_count": os.cpu_count(), "threads": 1,
                             "note": "numpy elementwise ops, one thread; images_timed=%d" % ref["images_timed"]},
                "rounds_ms": gpu["rounds_ms"], **wk,
                "how": "gpu: eager calls, 3 alternating rounds of --steps calls, CUDA events, median per call; "
                       "reference: D2H copy + numpy float32 restatement per image, host clock"}
        line.update(ident)
        print(json.dumps(line))


if __name__ == "__main__":
    main()
