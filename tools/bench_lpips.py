#!/usr/bin/env python
"""Times LPIPS (pixelsplat_b200.lpips, VGG16 trunk in torch/cuDNN, distance head fused in csrc/lpips.cu) at the
shapes it is used at:
  [28, 3, 256, 256]  training: LossLpips of 7 scenes x 4 target views (prediction requires grad, target does not);
  [32, 3, 256, 256]  the test metric (compute_lpips of one chunk, no grad).
Per shape:
  head     the fused head against the torch head (oracle/lpips_oracle.head in float32, the lpips package's form), on
           the same relu1_2 .. relu5_3 features, forward and forward + backward (gradient of the prediction side),
           in alternating rounds of --steps calls, CUDA events, median per call; achieved GB/s against the
           algorithmic bytes (forward: both sides read once; backward: both read once more, one side written);
  whole    the whole LossLpips forward + backward (training) or the metric forward, and the trunk alone, so the head's
           share is visible;
  kernels  per-kernel CUDA times of a few whole calls under torch.profiler (a separate run);
  memory   peak allocated bytes of one call of each head and of the whole call.
Weights are seeded random tensors (the timings do not depend on their values); TF32 is left as torch has it.
Prints one JSON line per shape with the card and its power limit.  Nothing is written.

    python tools/bench_lpips.py [--steps 50] [--warmup 10]
"""
import argparse
import json
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import lpips_oracle as lo  # noqa: E402
from tools.bench_depth import gpu_identity  # noqa: E402


def map_floats(h, w):
    """Sum of C H W over relu1_2 .. relu5_3 for an h x w input (7 995 392 at 256 x 256)."""
    total = 0
    for c in lo.CHANNELS:
        total += c * h * w
        h, w = h // 2, w // 2
    return total


def timed(fns: dict, steps: int, rounds: int = 3) -> dict:
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for name, f in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(steps):
                f()
            b.record()
            torch.cuda.synchronize()
            ms[name].append(a.elapsed_time(b) / steps)
    return {k: statistics.median(v) for k, v in ms.items()} | {"rounds_ms": ms}


def peak_bytes(f) -> int:
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    f()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def kernel_times(f, iters: int = 3) -> list:
    from torch.profiler import ProfilerActivity, profile
    f()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            f()
        torch.cuda.synchronize()
    rows = []
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if t > 0:
            rows.append({"kernel": e.key[:90], "calls_per_iter": e.count / iters, "us_per_iter": t / iters})
    rows.sort(key=lambda r: -r["us_per_iter"])
    return rows[:12]


def bench_shape(shape, train: bool, steps: int, warmup: int) -> dict:
    from pixelsplat_b200.loss import LossLpips, LossLpipsCfg, LossLpipsCfgWrapper
    from pixelsplat_b200.lpips import Lpips, lpips_head
    dev = "cuda"
    model = Lpips()
    model.load_state_dict(lo.random_state_dict(0))
    model = model.to(dev).eval()
    g = torch.Generator().manual_seed(1)
    n, _, h, w = shape
    target = torch.rand(shape, generator=g).to(dev)
    pred = (target.cpu() + 0.05 * torch.randn(shape, generator=g)).clamp(0, 1).to(dev)
    with torch.no_grad():
        f0 = [t.contiguous() for t in model.features(pred, True)]
        f1 = [t.contiguous() for t in model.features(target, True)]
    weights = model.lin_weights()
    f0g = [t.clone().requires_grad_(True) for t in f0]

    def fused_fwd():
        with torch.no_grad():
            lpips_head(f0, f1, weights)

    def torch_fwd():
        with torch.no_grad():
            lo.head(f0, f1, weights)

    def fused_fwdbwd():
        torch.autograd.grad(lpips_head(f0g, f1, weights).sum(), f0g)

    def torch_fwdbwd():
        torch.autograd.grad(lo.head(f0g, f1, weights).sum(), f0g)

    heads = {"fused_fwd": fused_fwd, "torch_fwd": torch_fwd}
    if train:
        heads |= {"fused_fwdbwd": fused_fwdbwd, "torch_fwdbwd": torch_fwdbwd}
    # the two heads agree on these features
    agree = float(((lpips_head(f0, f1, weights).double() - lo.head(f0, f1, weights).double()).abs()
                   / lo.head([t.double() for t in f0], [t.double() for t in f1],
                             [t.double() for t in weights]).abs()).max())

    loss = LossLpips(LossLpipsCfgWrapper(LossLpipsCfg(0.05, 0)), lpips=model).to(dev)
    loss.train()                                               # the training loss runs with dropout, as upstream
    pred5 = pred.view(n // 4 if n % 4 == 0 else 1, -1, *shape[1:])
    tgt5 = target.view(pred5.shape)
    batch = {"target": {"image": tgt5}}
    predg = pred5.clone().requires_grad_(True)
    P = type("P", (), {})
    pr = P()
    pr.color = predg

    def whole():
        if train:
            torch.autograd.grad(loss(pr, batch, None, 1), predg)
        else:
            with torch.no_grad():
                model(target, pred, normalize=True)

    predt = pred.clone().requires_grad_(True)

    def trunk():
        if train:
            feats = model.features(predt, True)
            with torch.no_grad():
                model.features(target, True)
            torch.autograd.grad(feats, predt, [torch.ones_like(t) for t in feats])
        else:
            with torch.no_grad():
                model.features(target, True)
                model.features(pred, True)

    allf = heads | {"whole": whole, "trunk": trunk}
    for f in allf.values():
        for _ in range(warmup):
            f()
    torch.cuda.synchronize()
    t = timed(allf, steps)
    floats = n * map_floats(h, w)
    fwd_bytes = 2 * 4 * floats + 4 * n
    bwd_bytes = 2 * 4 * floats + 4 * floats             # read both sides again, write the prediction side
    line = {"metric": "lpips", "shape": list(shape), "mode": "training (LossLpips, dropout on)" if train else
            "metric (eval, no grad)", "head_fused_fwd_ms": t["fused_fwd"], "head_torch_fwd_ms": t["torch_fwd"],
            "head_fwd_speedup": t["torch_fwd"] / t["fused_fwd"],
            "head_fused_fwd_GBps": fwd_bytes / (t["fused_fwd"] * 1e-3) / 1e9,
            "whole_ms": t["whole"], "trunk_ms": t["trunk"],
            "head_share_of_whole": (t["fused_fwdbwd"] if train else t["fused_fwd"]) / t["whole"],
            "fwd_bytes": fwd_bytes, "fwdbwd_bytes": fwd_bytes + bwd_bytes, "map_floats_per_image": map_floats(h, w),
            "fused_vs_torch_head_max_rel": agree, "rounds_ms": t["rounds_ms"],
            "peak_bytes": {k: peak_bytes(f) for k, f in allf.items()},
            "kernels_whole": kernel_times(whole)}
    if train:
        line |= {"head_fused_fwdbwd_ms": t["fused_fwdbwd"], "head_torch_fwdbwd_ms": t["torch_fwdbwd"],
                 "head_fwdbwd_speedup": t["torch_fwdbwd"] / t["fused_fwdbwd"],
                 "head_fused_fwdbwd_GBps": (fwd_bytes + bwd_bytes) / (t["fused_fwdbwd"] * 1e-3) / 1e9}
    line["how"] = ("eager calls, 3 alternating rounds of --steps calls each, CUDA events, median per call; per-kernel "
                   "times from torch.profiler in a separate run; cuDNN settings as torch has them "
                   f"(allow_tf32={torch.backends.cudnn.allow_tf32})")
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lpips.py needs a CUDA device: pixelsplat_b200 has no CPU path")
    ident = gpu_identity(0)
    for shape, train in (((28, 3, 256, 256), True), ((32, 3, 256, 256), False)):
        line = bench_shape(shape, train, args.steps, args.warmup)
        line.update(ident)
        print(json.dumps(line))


if __name__ == "__main__":
    main()
